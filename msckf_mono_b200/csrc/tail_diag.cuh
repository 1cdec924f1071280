// msckf_mono_b200/csrc/tail_diag.cuh -- the 32 x 32 diagonal block of the tail's blocked factorisation (round 2).
//
// Round 1 factorised a diagonal block with one warp per matrix, a shuffle + shared-memory round trip per pivot and a second
// pair of warps building the inverses one pivot behind (the S'' warp polling Gamma's keep / drop decision through a
// volatile flag): per-pivot communication made it half of the kernel.  What shaped this version (%globaltimer stamps
// inside the functions, scripts/tail_profile.py):
//   * per-pivot communication is what costs: the block is itself blocked by panels, the diagonal micro-block of a panel is
//     factorised REDUNDANTLY in registers by every thread of the warps that need it -- static indices, right-looking, so the
//     dependent chain of a pivot is rsqrt -> multiply -> one FMA (scripts/fp64_latency.cu measures it) -- and the keep / drop
//     decision of each pivot (Gamma's pivot against thr x its original diagonal, the rank cap; S'' follows) is evaluated by
//     every thread from the same numbers; two CTA barriers per panel;
//   * code that runs once per call is bound by instruction fetch once the body exceeds the instruction caches (a first
//     version with a fully unrolled 32-step inverse was ~3 200 instructions and slower than the rolled code): every loop
//     here is rolled except the micro-block itself;
//   * the inverses of the factors ride along the panels as 32 extra rows (rows of the identity, solved like panel rows):
//     no separate inverse stage.  Only the inverses leave the block -- the panels below it are X = rows x Linv^T.
// Two entry points: tf_factor_block (Gamma and S'' together on one CTA, 4-column panels: the 8-CTA cluster form) and
// tf_factor_one (one matrix per CTA, 8-column panels, Gamma's flags handed to the S'' CTA through DSMEM: the 9-CTA form).
#pragma once
#include "common.cuh"

namespace mb {

constexpr int kFB = 32;        // block size of the fused form
constexpr int kFLD = kFB + 2;  // row stride of the 32 x 32 shared blocks: even (16-byte loads), conflict-free per quarter warp

struct TfRank { int g, a; };

// 1 / sqrt(p), p > 0 finite: hardware seed (MUFU.RSQ64H, ~2^-22) + two Newton steps in fp64
__device__ __forceinline__ double tf_rsqrt_pos(double p) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(p));
  const double hp = 0.5 * p;
  y = y * (1.5 - hp * y * y);
  y = y * (1.5 - hp * y * y);
  return y;
}

__device__ __noinline__ TfRank tf_factor_block(double* __restrict__ DG, double* __restrict__ DA, double* __restrict__ LIG,
                                               double* __restrict__ LIA, double* __restrict__ idg, double* __restrict__ ida,
                                               const double* __restrict__ d0, int kb, int nb, double thr, int rank_cap, bool full,
                                               TfRank rk, int tid, int nthreads, double* __restrict__ TA /*[32][kFLD] scratch*/,
                                               double* __restrict__ TG /*[32][kFLD] scratch*/, double* __restrict__ pivr,
                                               unsigned long long* dprof = nullptr) {
  constexpr int LD = kFLD, PW = 4;
  int dpi = 0;
  auto dstamp = [&]() {
    if (dprof && tid == 0 && dpi < 14) dprof[dpi++] = globaltimer();
  };
  dstamp();
  const int half = (tid >> 5) & 1, lane = tid & 31;
  const bool extra = tid >= 64;  // warps 2, 3: the rows of the identity that turn into the inverses (see below)
  // The inverses ride along as 32 EXTRA ROWS per matrix: solving  Y L^T = I  row by row is exactly what the panel algorithm
  // does to the rows below the block (micro-solve against the diagonal micro-block, then the trailing update), and
  // Y = L^-T, i.e. extra row i, column j holds Linv[j][i] -- stored transposed, straight into LIA / LIG.  Row i of the identity
  // is zero left of column i, so it only joins from the panel that contains column i.  This replaces a separate inverse
  // stage (7 CTA barriers per block in the first version of this file).
  for (int e = tid; e < kFB * LD; e += nthreads) {
    const int k = e / LD, c = e % LD;
    LIA[e] = (k == c) ? 1.0 : 0.0;
    LIG[e] = (k == c) ? 1.0 : 0.0;
  }
  __syncthreads();
#pragma unroll 1
  for (int c0 = 0; c0 < kFB; c0 += PW) {
    if (c0 >= nb) {  // columns beyond the matrix: dropped indices
      if (tid < PW) { ida[c0 + tid] = 0.0; idg[c0 + tid] = 0.0; }
      continue;
    }
    if (tid < 128) {
    // (1) the two 4 x 4 diagonal micro-blocks, redundantly in every thread of warps 0..3 (the row solvers of (2) need them
    // in registers; all eight warps doing it would make the half-rate FP64 pipe, not the pivot chain, the limit)
    double Gm[PW][PW], Am[PW][PW], ivg[PW], iva[PW], pvs[PW];
#pragma unroll
    for (int a = 0; a < PW; ++a)
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        Am[a][b] = DA[(c0 + a) * LD + c0 + b];
        Gm[a][b] = full ? 0.0 : DG[(c0 + a) * LD + c0 + b];
      }
#pragma unroll
    for (int j = 0; j < PW; ++j) {
      const double dk0 = d0[kb + c0 + j];
      const double pg = Gm[j][j], pa = Am[j][j];
      bool drop;
      if (full) drop = (c0 + j >= nb) || !(dk0 > 0.0) || rk.a >= rank_cap;
      else drop = (c0 + j >= nb) || !(dk0 > 0.0) || !(pg > thr * dk0) || rk.g >= rank_cap;
      if (!drop) rk.g++;
      pvs[j] = full ? 1.0 : pg;
      const double ig = (drop || full) ? 0.0 : tf_rsqrt_pos(pg);
      const bool dropa = drop || !(pa > 0.0);
      if (!dropa) rk.a++;
      const double ia = dropa ? 0.0 : tf_rsqrt_pos(pa);
      ivg[j] = ig; iva[j] = ia;
#pragma unroll
      for (int a = j + 1; a < PW; ++a) { Gm[a][j] *= ig; Am[a][j] *= ia; }
#pragma unroll
      for (int b = j + 1; b < PW; ++b)
#pragma unroll
        for (int a = b; a < PW; ++a) { Gm[a][b] -= Gm[a][j] * Gm[b][j]; Am[a][b] -= Am[a][j] * Am[b][j]; }
    }
    if (tid < PW) {
      double vg = 0.0, va = 0.0;
#pragma unroll
      for (int j = 0; j < PW; ++j) if (j == tid) { vg = ivg[j]; va = iva[j]; }
      idg[c0 + tid] = vg; ida[c0 + tid] = va;
    }
    if (tid == 127) {  // diagnostics (msckf_b200_rank_pivots): Gamma's pivots as they were compared -- plain stores, off the chain
#pragma unroll
      for (int j = 0; j < PW; ++j) if (c0 + j < nb) pivr[kb + c0 + j] = pvs[j];
    }
    // (2) one row of the panel per thread (rows c0 .. nb-1; warp 0: S'', warp 1: Gamma), solved in registers; a row inside the
    // micro-block reproduces the factor's own row (entries right of its diagonal are masked)
    const int rrow = c0 + lane;
    if (!extra && rrow < nb && !(half == 1 && full)) {
      double* D = half ? DG : DA;
      double x[PW];
#pragma unroll
      for (int j = 0; j < PW; ++j) x[j] = (c0 + j <= rrow) ? D[rrow * LD + c0 + j] : 0.0;
#pragma unroll
      for (int j = 0; j < PW; ++j) {
        x[j] *= half ? ivg[j] : iva[j];
        if (c0 + j > rrow) x[j] = 0.0;
#pragma unroll
        for (int jj = j + 1; jj < PW; ++jj) x[jj] -= x[j] * (half ? Gm[jj][j] : Am[jj][j]);
      }
#pragma unroll
      for (int j = 0; j < PW; ++j) if (c0 + j <= rrow) D[rrow * LD + c0 + j] = x[j];
    }
    if (extra && lane < c0 + PW && lane < nb && !(half == 1 && full)) {  // extra row `lane` of the identity, active from its own column on
      double* LI = half ? LIG : LIA;
      double x[PW];
#pragma unroll
      for (int j = 0; j < PW; ++j) x[j] = LI[(c0 + j) * LD + lane];
#pragma unroll
      for (int j = 0; j < PW; ++j) {
        x[j] *= half ? ivg[j] : iva[j];
#pragma unroll
        for (int jj = j + 1; jj < PW; ++jj) x[jj] -= x[j] * (half ? Gm[jj][j] : Am[jj][j]);
      }
#pragma unroll
      for (int j = 0; j < PW; ++j) LI[(c0 + j) * LD + lane] = x[j];
    }
    }
    __syncthreads();
    // (3) trailing update inside the block: rows / columns c0+4 .. nb-1, lower triangle, both matrices -- and of the extra rows:
    // rhs[i][j] -= sum_k Y[i][c0+k] L[j][c0+k] for the active rows i < q0, columns j >= q0.  Threads as a 16 x 16 grid (no
    // index divisions on this path: every instruction here is on the critical chain of the whole kernel).
    const int q0 = c0 + PW, nr = nb - q0;
    if (nr > 0) {
      const int ty = tid >> 4, tx = tid & 15;
#pragma unroll 1
      for (int i = q0 + ty; i < nb; i += 16) {
        const double2 a01 = *reinterpret_cast<const double2*>(DA + i * LD + c0), a23 = *reinterpret_cast<const double2*>(DA + i * LD + c0 + 2);
        const double2 g01 = *reinterpret_cast<const double2*>(DG + i * LD + c0), g23 = *reinterpret_cast<const double2*>(DG + i * LD + c0 + 2);
#pragma unroll 1
        for (int j = q0 + tx; j <= i; j += 16) {
          const double2 b01 = *reinterpret_cast<const double2*>(DA + j * LD + c0), b23 = *reinterpret_cast<const double2*>(DA + j * LD + c0 + 2);
          DA[i * LD + j] -= (a01.x * b01.x + a01.y * b01.y) + (a23.x * b23.x + a23.y * b23.y);
          if (!full) {
            const double2 h01 = *reinterpret_cast<const double2*>(DG + j * LD + c0), h23 = *reinterpret_cast<const double2*>(DG + j * LD + c0 + 2);
            DG[i * LD + j] -= (g01.x * h01.x + g01.y * h01.y) + (g23.x * h23.x + g23.y * h23.y);
          }
        }
      }
      const int nact = min(q0, nb);
#pragma unroll 1
      for (int j = q0 + ty; j < nb; j += 16) {
        const double2 b01 = *reinterpret_cast<const double2*>(DA + j * LD + c0), b23 = *reinterpret_cast<const double2*>(DA + j * LD + c0 + 2);
        const double2 h01 = *reinterpret_cast<const double2*>(DG + j * LD + c0), h23 = *reinterpret_cast<const double2*>(DG + j * LD + c0 + 2);
#pragma unroll 1
        for (int i = tx; i < nact; i += 16) {
          LIA[j * LD + i] -= (LIA[c0 * LD + i] * b01.x + LIA[(c0 + 1) * LD + i] * b01.y) + (LIA[(c0 + 2) * LD + i] * b23.x + LIA[(c0 + 3) * LD + i] * b23.y);
          if (!full) LIG[j * LD + i] -= (LIG[c0 * LD + i] * h01.x + LIG[(c0 + 1) * LD + i] * h01.y) + (LIG[(c0 + 2) * LD + i] * h23.x + LIG[(c0 + 3) * LD + i] * h23.y);
        }
      }
    }
    __syncthreads();
  }
  dstamp();  // factors + inverses done
  // rows / columns of dropped or out-of-range pivots of the inverses are zero by construction (1 / L_kk := 0)
  return rk;
}

// ---- the same factorisation for ONE matrix per CTA (k_tail_fused<S, 2>: Gamma's and S''s chains of diagonal blocks run on
// two CTAs of the cluster, side by side).  S'' must follow Gamma's keep / drop decisions: the Gamma CTA publishes the flags of
// a panel as ONE 32-bit word -- (block tag << 8) | drop bits -- with an atomic exchange into the S'' CTA's shared memory
// through DSMEM (a single word: no fence, nothing else to order).  The S'' CTA does not wait for it: it factorises its micro-block
// assuming "nothing dropped" (its own non-positive pivots aside), then looks at the word, and only if Gamma did drop
// something (the panel that meets the null space of H_o) repeats the micro-block with the real flags.  Gamma never waits.
//   role 0: S'', following the flags   role 1: Gamma, deciding and publishing   role 2: S'' alone (m <= n: no Gamma)
struct TfLink {
  volatile unsigned* words;  // [32 / PW] role 0: local; role 1: the partner's (mapped) array
  int* timed_out;            // role 0: set when the partner's word never arrived (reported as a failed update, never silent)
};

__device__ __noinline__ int tf_factor_one(double* __restrict__ D, double* __restrict__ LI, double* __restrict__ idv,
                                          const double* __restrict__ d0, int kb, int nb, double thr, int rank_cap, int role, int rk,
                                          int tid, int nthreads, unsigned tag /* > 0, grows with every block */, TfLink lk,
                                          double* __restrict__ pivr, unsigned long long* dprof = nullptr) {
  constexpr int LD = kFLD, PW = 8, PH = PW / 2;  // 8-column panels: four per block, half the barriers of tf_factor_block's 4
  auto dstamp = [&](int slot) {  // fixed slots: 0 entry | 1 + 4 p + {0: micro + rows, 1: barrier, 2: trailing, 3: barrier} for panels p < 3 | 13 end
    if (dprof && tid == 0) dprof[slot] = globaltimer();
  };
  dstamp(0);
  const int lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < kFB * LD; e += nthreads) LI[e] = (e / LD == e % LD) ? 1.0 : 0.0;  // the extra rows (see tf_factor_block)
  __syncthreads();
#pragma unroll 1
  for (int c0 = 0; c0 < kFB; c0 += PW) {
    if (c0 >= nb) {  // columns beyond the matrix: dropped indices (both CTAs skip them: nothing to publish)
      if (tid < PW) idv[c0 + tid] = 0.0;
      continue;
    }
    if (tid < 64) {
      double Mm[PW][PW], iv[PW], pvs[PW];
      unsigned bits = 0u;  // Gamma's drop flags of this panel (role 0: assumed clear on the first pass)
      int rk1 = rk;
#pragma unroll 1
      for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
        for (int a = 0; a < PW; ++a)
#pragma unroll
          for (int b = 0; b <= a; ++b) Mm[a][b] = D[(c0 + a) * LD + c0 + b];
        rk1 = rk;
        unsigned mine = 0u;
#pragma unroll
        for (int j = 0; j < PW; ++j) {
          const double dk0 = d0[kb + c0 + j];
          const double p = Mm[j][j];
          bool drop;
          if (role == 1) {
            drop = (c0 + j >= nb) || !(dk0 > 0.0) || !(p > thr * dk0) || rk1 >= rank_cap;
            if (drop) mine |= 1u << j;
          } else if (role == 2) {
            drop = (c0 + j >= nb) || !(dk0 > 0.0) || rk1 >= rank_cap || !(p > 0.0);
          } else {
            drop = ((bits >> j) & 1u) != 0u || !(p > 0.0);
          }
          if (!drop) rk1++;
          pvs[j] = (role == 2) ? 1.0 : p;
          const double i_ = drop ? 0.0 : tf_rsqrt_pos(p);
          iv[j] = i_;
#pragma unroll
          for (int a = j + 1; a < PW; ++a) Mm[a][j] *= i_;
#pragma unroll
          for (int b = j + 1; b < PW; ++b)
#pragma unroll
            for (int a = b; a < PW; ++a) Mm[a][b] -= Mm[a][j] * Mm[b][j];
        }
        // publish / poll the panel's word with atomics (one word is the whole message; atomics keep the exchange well-defined
        // for the memory model and for racecheck); one lane per warp polls, the warp gets the word by shuffle
        if (role == 1 && tid == 0) atomicExch(const_cast<unsigned*>(lk.words) + c0 / PW, (tag << 8) | mine);
        if (role != 0 || pass == 1) break;
        unsigned w = 0u;
        if (lane == 0) {
          unsigned* wp = const_cast<unsigned*>(lk.words) + c0 / PW;
          w = atomicOr(wp, 0u);
          for (int spin = 0; (w >> 8) != tag && spin < (1 << 22); ++spin) w = atomicOr(wp, 0u);  // (bounded: a lost partner must not hang the device)
        }
        w = __shfl_sync(0xffffffffu, w, 0);
        if ((w >> 8) != tag) { if (tid == 0) *lk.timed_out = 1; w = 0xffu; }  // lost partner: drop the panel and flag the update
        if ((w & 0xffu) == 0u) break;  // nothing dropped by Gamma: the speculative pass stands
        bits = w & 0xffu;
      }
      rk = rk1;
      if (tid < PW) {
        double v = 0.0;
#pragma unroll
        for (int j = 0; j < PW; ++j) if (j == tid) v = iv[j];
        idv[c0 + tid] = v;
      }
      if (role != 0 && tid == 63) {  // diagnostics (msckf_b200_rank_pivots): the pivots as they were compared -- plain stores
#pragma unroll
        for (int j = 0; j < PW; ++j) if (c0 + j < nb) pivr[kb + c0 + j] = pvs[j];
      }
      // one row per lane: warp 0 the panel rows c0 .. nb-1, warp 1 the extra rows 0 .. c0+3 (the inverse, transposed)
      const int rrow = c0 + lane;
      if (warp == 0 && rrow < nb) {
        double x[PW];
#pragma unroll
        for (int j = 0; j < PW; ++j) x[j] = (c0 + j <= rrow) ? D[rrow * LD + c0 + j] : 0.0;
#pragma unroll
        for (int j = 0; j < PW; ++j) {
          x[j] *= iv[j];
          if (c0 + j > rrow) x[j] = 0.0;
#pragma unroll
          for (int jj = j + 1; jj < PW; ++jj) x[jj] -= x[j] * Mm[jj][j];
        }
#pragma unroll
        for (int j = 0; j < PW; ++j) if (c0 + j <= rrow) D[rrow * LD + c0 + j] = x[j];
      }
      if (warp == 1 && lane < c0 + PW && lane < nb) {
        double x[PW];
#pragma unroll
        for (int j = 0; j < PW; ++j) x[j] = LI[(c0 + j) * LD + lane];
#pragma unroll
        for (int j = 0; j < PW; ++j) {
          x[j] *= iv[j];
#pragma unroll
          for (int jj = j + 1; jj < PW; ++jj) x[jj] -= x[j] * Mm[jj][j];
        }
#pragma unroll
        for (int j = 0; j < PW; ++j) LI[(c0 + j) * LD + lane] = x[j];
      }
    }
    if (c0 < 3 * PW) dstamp(1 + 4 * (c0 / PW));
    __syncthreads();
    if (c0 < 3 * PW) dstamp(2 + 4 * (c0 / PW));
    // trailing update inside the block (rows / columns c0+4 .. nb-1, lower triangle) and of the extra rows; the 256 threads
    // are split between the two: 128 as an 8 x 16 grid on the block, 128 on the extra rows
    const int q0 = c0 + PW, nr = nb - q0;
    if (nr > 0) {
      const int h = tid >> 7, t7 = tid & 127, ty = t7 >> 4, tx = t7 & 15;
      if (h == 0) {
#pragma unroll 1
        for (int i = q0 + ty; i < nb; i += 8) {
          double2 av[PH];
#pragma unroll
          for (int u = 0; u < PH; ++u) av[u] = *reinterpret_cast<const double2*>(D + i * LD + c0 + 2 * u);
#pragma unroll 1
          for (int j = q0 + tx; j <= i; j += 16) {
            double acc[PH];
#pragma unroll
            for (int u = 0; u < PH; ++u) {
              const double2 bv = *reinterpret_cast<const double2*>(D + j * LD + c0 + 2 * u);
              acc[u] = av[u].x * bv.x + av[u].y * bv.y;
            }
            double t = acc[0];
#pragma unroll
            for (int u = 1; u < PH; ++u) t += acc[u];
            D[i * LD + j] -= t;
          }
        }
      } else {
        const int nact = min(q0, nb);
#pragma unroll 1
        for (int j = q0 + ty; j < nb; j += 8) {
          double2 bv[PH];
#pragma unroll
          for (int u = 0; u < PH; ++u) bv[u] = *reinterpret_cast<const double2*>(D + j * LD + c0 + 2 * u);
#pragma unroll 1
          for (int i = tx; i < nact; i += 16) {
            double acc[PH];
#pragma unroll
            for (int u = 0; u < PH; ++u) acc[u] = LI[(c0 + 2 * u) * LD + i] * bv[u].x + LI[(c0 + 2 * u + 1) * LD + i] * bv[u].y;
            double t = acc[0];
#pragma unroll
            for (int u = 1; u < PH; ++u) t += acc[u];
            LI[j * LD + i] -= t;
          }
        }
      }
    }
    if (c0 < 3 * PW) dstamp(3 + 4 * (c0 / PW));
    __syncthreads();
    if (c0 < 3 * PW) dstamp(4 + 4 * (c0 / PW));
  }
  dstamp(13);
  return rk;
}

}  // namespace mb
