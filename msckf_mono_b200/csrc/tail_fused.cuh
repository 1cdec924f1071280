// msckf_mono_b200/csrc/tail_fused.cuh
// The serial part of the EKF tail for windows up to 34 clones as ONE thread-block-cluster kernel:
//     Gamma (Gram matrix of the basis)  -> rank decision      }  rank-revealing Cholesky of Gamma (G) and S'' (A),
//     S'' = L L^T over the kept indices                        }  blocked by 32, A following G's decisions
//     W = L^-1 [T''P | r'']   fused into the factorisation: every worker CTA keeps its share of the right-hand-side columns
//                             as rows in shared memory and treats them as extra panel rows
// followed by  P <- P - W^T W, dx = W^T y and the state injection (k_syrk, all SMs)   (msckf.h:1373-1418).
// Two forms: k_tail_fused<S, 2> -- a cluster of 9 CTAs (non-portable size, used where the device accepts it): CTA 0 runs S''s
// chain of diagonal blocks, CTA 1 Gamma's, CTAs 2..8 are the workers; k_tail_fused<S, 1> -- a cluster of 8: CTA 0 runs both
// chains (tf_factor_block), CTAs 1..7 are the workers.
//
// What bounds this kernel is latency, not the FP64 pipe (scripts/fp64_rate.cu measures its rate): a chain of n dependent
// pivots (scripts/fp64_latency.cu measures one step) plus what surrounds them, and instruction fetch -- the kernel is
// ~100 KB of SASS, far more than the instruction caches hold, so every phase of every block iteration starts cold.
// Measured (ncu source view, %globaltimer stamps: scripts/tail_profile.py) and acted upon:
//   * the diagonal block (tail_diag.cuh): blocked by panels (8 columns in the two-chain form, 4 in the one-chain form), the
//     diagonal micro-block factorised redundantly in registers by the threads that solve the panel rows, keep / drop decisions
//     evaluated by all of them from the same numbers; the inverses ride along as 32 extra rows; loops rolled except the
//     micro-block (a fully unrolled 32-step-inverse version was fetch-bound);
//   * the two chains only meet in the keep / drop flags: one 32-bit word per panel through DSMEM, S'' speculates "nothing
//     dropped" and repeats a micro-block only when Gamma did drop (tf_factor_one);
//   * the chain CTAs run ONE BLOCK AHEAD of the workers: they solve the 32 panel rows of the next diagonal block themselves
//     with the inverses they still hold, form that block and factorise it while the workers solve the panel, exchange it and
//     run the trailing update (split cluster barrier: arrive early, wait late; published inverses double-buffered);
//   * the panel below a diagonal block is X = A_panel L_kk^-T: with L_kk^-1 at hand a small GEMM shared by all 8 warps
//     instead of a 32-step substitution per row; panel rows are dealt to the workers (no redundant solves) and exchanged
//     through L2 (a scratch panel every worker reads back after the cluster barrier: faster than pushing it into 8 shared
//     memories through DSMEM);
//   * shared-memory bank conflicts: tiles are dealt so that the lanes of a warp read neighbouring columns.
// Two cluster barriers (release/acquire at cluster scope) per block order the phases.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"
#include "tail_cluster.cuh"
#include "tail_diag.cuh"

namespace mb {


__host__ __device__ inline size_t tail_fused_smem_bytes(int n) {
  const size_t ldt = (size_t)((n + 3) & ~3);
  // DG, DA, LIG, LIA, WB, DT [32][34] | PT_A, PT_G, Ws [32][ldt] | XT [32][32] | d0 [n] | idg, ida [32]
  return sizeof(double) * (6 * (size_t)kFB * kFLD + 3 * (size_t)kFB * ldt + (size_t)kFB * kFB + ((n + 1) & ~1) + 2 * kFB) + 64;
}

__device__ __forceinline__ void tf_ld8(const double* p, double (&v)[8]) {
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const double2 t = *reinterpret_cast<const double2*>(p + 2 * u);
    v[2 * u] = t.x; v[2 * u + 1] = t.y;
  }
}
__device__ __forceinline__ void tf_ld4(const double* p, double (&v)[4]) {
  const double2 t = *reinterpret_cast<const double2*>(p), u = *reinterpret_cast<const double2*>(p + 2);
  v[0] = t.x; v[1] = t.y; v[2] = u.x; v[3] = u.y;
}

// diagonal block -> shared [32][34]: lower triangle including the diagonal (zeros elsewhere)
__device__ __forceinline__ void tf_load_diag(double* D, const double* A, int ld, int kb, int nb, int tid) {
  for (int e = tid; e < kFB * kFLD; e += kTailThreads) {
    const int i = e / kFLD, j = e % kFLD;
    double v = 0.0;
    if (i < nb && j <= i) v = A[(size_t)(kb + i) * ld + kb + j];
    D[e] = v;
  }
}

// NCH = number of CTAs that run chains of diagonal blocks: 1 (cluster of 8: CTA 0 factorises Gamma's and S''s blocks together)
// or 2 (cluster of 9: CTA 0 S'', CTA 1 Gamma, side by side -- tf_factor_one; the other seven CTAs are the workers either way).
template <class S, int NCH>
__global__ void __launch_bounds__(kTailThreads) k_tail_fused(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& ua = args[blockIdx.z];
  if (ua.n_tracks == 0 || ua.tail_kind != 0) return;  // (uniform over the cluster)
  const int n = ua.n, ld = ua.ld;
  double* __restrict__ G = ua.T2;        // T'' on entry: patched into Gamma in place
  double* __restrict__ A = ua.S2;
  const double thr = ua.rank_thr;
  int* __restrict__ rank_out = ua.rank_out;
  const int* __restrict__ m_in = ua.m_out;
  const double* __restrict__ TP = ua.TP;
  const double* __restrict__ r2 = ua.r2;
  double* __restrict__ Wm = ua.W;
  double* __restrict__ yv = ua.y;
  double* __restrict__ dx_out = ua.dx;
  double* __restrict__ scratch = ua.G;   // >= 64 * (34 + ldt) doubles
  unsigned long long* __restrict__ prof = ua.prof;  // optional phase timestamps
  namespace cg = cooperative_groups;
  constexpr int NB = kFB, LD = kFLD;
  // [2 slots][2][32][34] inverses of the diagonal blocks' factors (A, G): CTA 0 runs one block ahead of the others, so the
  // slot of block k + 1 is written while slot k may still be read
  auto Lsc_of = [&](int blk) { return scratch + (size_t)(blk & 1) * 2 * NB * LD; };
  double* Psc = scratch + 4 * NB * LD;        // [2][32][ldt] the current panels, transposed (A, G)
  cg::cluster_group cluster = cg::this_cluster();
  const int crank = (int)cluster.block_rank();
  const int C = (int)cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int prof_i = 0;
  auto stamp = [&]() {
    if (prof && blockIdx.x == 0 && tid == 0 && prof_i < 39) prof[prof_i++] = globaltimer();
  };
  stamp();
  int wprof_i = 0;
  auto wstamp = [&]() {  // the same for the first worker CTA (slots 20..39)
    if (prof && (int)blockIdx.x == NCH && blockIdx.z == 0 && tid == 0 && wprof_i < 19) prof[20 + wprof_i++] = globaltimer();
  };
  extern __shared__ __align__(16) double sm[];
  const int ldt = (n + 3) & ~3;              // row stride of the transposed panels (16-byte aligned rows)
  double* DG = sm;                           // [32][34] diagonal block of G (CTA 0); then this CTA's panel rows of G; then X_G^T
  double* DA = DG + NB * LD;                 // [32][34] same for A
  double* LIG = DA + NB * LD;                // [32][34] inverse of the factor of G's block
  double* LIA = LIG + NB * LD;               // [32][34] same for A
  double* WB = LIA + NB * LD;                // [32][34] the current block of this CTA's W rows
  double* DT = WB + NB * LD;                 // [32][34] scratch of the diagonal block's inverse (CTA 0)
  double* PT_A = DT + NB * LD;               // [32][ldt] panel of A, transposed
  double* PT_G = PT_A + (size_t)NB * ldt;    // [32][ldt] panel of G, transposed
  double* Ws = PT_G + (size_t)NB * ldt;      // [32][ldt] row c = RHS column col0 + c of the substitution
  double* XT = Ws + (size_t)NB * ldt;        // [32][32]  solved block of the W rows, transposed
  double* d0 = XT + NB * NB;                 // [n] original diagonal of Gamma (CTA 0)
  double* idg = d0 + ((n + 1) & ~1);         // [32] 1 / diag of the block's factor of G (0 = dropped)
  double* ida = idg + NB;                    // [32] same for A
  __shared__ int s_rankA, s_rankG;
  __shared__ int s_timeout;             // NCH = 2, CTA 0: the Gamma CTA's flags did not arrive within the polling bound
  __shared__ unsigned s_words[NB / 4];  // NCH = 2, CTA 0: Gamma's drop flags, one word per panel of the block (written by CTA 1)
  const int m = *m_in;
  const bool full = m <= n;  // all rows explicit and orthonormal: Gamma = I_m, nothing to decide, G untouched
  const int rank_cap = min(m, n);
  const int gtid = crank * kTailThreads + tid, gthreads = C * kTailThreads;

  if (m == 0) {  // nothing accepted: the reference returns before touching the state (msckf.h:401-403, :1328)
    for (int a = gtid; a < n; a += gthreads) dx_out[a] = 0.0;
    if (gtid == 0) *rank_out = 0;
    return;
  }
  const int ncol = n + 1;
  const int NWK = C - NCH, widx = crank - NCH;  // workers: the CTAs behind the chain CTAs
  const int per = (ncol + NWK - 1) / NWK;    // RHS columns per worker (<= 32); the chain CTAs take none
  const int col0 = widx * per, cw = (crank < NCH) ? 0 : max(0, min(per, ncol - col0));
  const int ncw4 = (cw + 3) / 4;
  // ---------------------------------------------------------------- Gamma = [[I_h, H_h], [H_h^T, Lambda]]: T'' already
  // holds H_h (rows < 15) and Lambda; only the lower triangle is read below, so patching the first 15 columns suffices
  if (!full) {
    for (int e = gtid; e < n * kImuDim; e += gthreads) {
      const int a = e / kImuDim, b = e % kImuDim;
      G[(size_t)a * ld + b] = (a < kImuDim) ? ((a == b) ? 1.0 : 0.0) : G[(size_t)b * ld + a];
    }
  }
  if (tid < NB / 4) s_words[tid] = 0u;
  if (tid == 0) s_timeout = 0;
  // split barrier: the chain CTAs only wait for everybody's part of the Gamma patch, not for the workers' staging of the
  // right-hand sides (strided loads that nobody needs before the first panel)
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  if (crank >= NCH) {
    for (int e = tid; e < NB * n; e += kTailThreads) {  // consecutive threads -> consecutive k: conflict-free stores
      const int c = e / n, k = e % n, col = col0 + c;
      double v = 0.0;
      if (c < cw) v = (col < n) ? TP[(size_t)k * ld + col] : r2[k];
      Ws[(size_t)c * ldt + k] = v;
    }
    for (int e = tid; e < NB * (ldt - n); e += kTailThreads) Ws[(size_t)(e / (ldt - n)) * ldt + n + e % (ldt - n)] = 0.0;
  }
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  stamp();  // Gamma patched, right-hand sides staged
  if (crank < NCH) {
    for (int k = tid; k < n; k += kTailThreads) {
      d0[k] = full ? (k < m ? 1.0 : 0.0) : G[(size_t)k * ld + k];
      if (crank == 0) ua.pivr[n + k] = d0[k];  // (diagnostics: the denominators of msckf_b200_rank_pivots)
    }
    if (tid == 0) { s_rankA = 0; s_rankG = 0; }
  }
  __syncthreads();
  // ---------------------------------------------------------------- blocked rank-revealing Cholesky (G decides, A follows)
  // The chain CTAs factorise the diagonal blocks: NCH = 1: CTA 0 both matrices (tf_factor_block, tail_diag.cuh: G decides
  // keep / drop per pivot, A follows); NCH = 2: CTA 0 S'' and CTA 1 Gamma (tf_factor_one: Gamma's flags reach CTA 0 through
  // DSMEM).  A block (lower triangle incl. the diagonal) is in shared memory when `factor` is called; the inverses end up
  // in shared memory and in the L2 scratch for the workers.  Block 0 is factorised up front; block kb + 1 is factorised
  // WHILE the workers run the trailing update of block kb (it only needs the leading 32 x 32 tile of that update, which the
  // chain CTAs form themselves from the panel).
  // The NM matrices a chain CTA carries -- NCH = 1: S'' and Gamma (Gamma's loads and arithmetic skipped when m <= n);
  // NCH = 2: its own in DA / LIA / ida (CTA 0: S'', CTA 1: Gamma; the Gamma CTA idles when m <= n).  Matrix q is handed out
  // by a function of q over the restrict pointer Mch, not kept in an array of pointers: with an array the one-chain form
  // needs 6 more registers, without Mch the two-chain form spills.
  constexpr int NM = 3 - NCH;
  const bool chainG = (NCH == 2) && crank == 1;
  struct ChainMat { const double* M; double* D; double* LI; double* X; };  // in L2, its diagonal block, that block's inverse, X
  double* __restrict__ Mch = chainG ? G : A;
  auto cm = [&](int q) { return q == 0 ? ChainMat{Mch, DA, LIA, WB} : ChainMat{G, DG, LIG, DT}; };
  auto live = [&](int q) { return NCH == 2 || q == 0 || !full; };
  auto isG = [&](int q) { return NCH == 2 ? chainG : q == 1; };
  TfLink link;
  link.words = s_words;
  link.timed_out = &s_timeout;
  if (NCH == 2 && chainG) link.words = cluster.map_shared_rank(s_words, 0);  // the Gamma CTA writes into CTA 0's array
  auto factor = [&](int kb, int nb, bool stamps, double* Lsc) {
    if (stamps && tid == 0) prof[76] = globaltimer();
    if (NCH == 1) {
      TfRank rk;
      rk.g = s_rankG; rk.a = s_rankA;
      __syncthreads();
      rk = tf_factor_block(DG, DA, LIG, LIA, idg, ida, d0, kb, nb, thr, rank_cap, full, rk, tid, kTailThreads, WB, DT, ua.pivr, stamps ? prof + 60 : nullptr);
      if (tid == 0) { s_rankG = rk.g; s_rankA = rk.a; }
    } else {
      const int rk0 = chainG ? s_rankG : s_rankA;
      __syncthreads();
      const int role = full ? 2 : (chainG ? 1 : 0);
      const int rk1 = tf_factor_one(DA, LIA, ida, d0, kb, nb, thr, rank_cap, role, rk0, tid, kTailThreads, (unsigned)(kb / NB) + 1u, link, ua.pivr, stamps ? prof + 60 : nullptr);
      if (tid == 0) { if (chainG) s_rankG = rk1; else s_rankA = rk1; }
    }
    if (stamps && tid == 0) prof[77] = globaltimer();
    // the inverses go to the workers through L2 (a DSMEM push of 2 x 8.7 KB to 7 CTAs runs at ~20 B/clk: 3 us)
    for (int e = tid; e < NB * LD / 2; e += kTailThreads) {
#pragma unroll
      for (int q = 0; q < NM; ++q)
        if (live(q)) reinterpret_cast<double2*>(Lsc + (isG(q) ? NB * LD : 0))[e] = reinterpret_cast<const double2*>(cm(q).LI)[e];
    }
  };
  if (crank < NCH && !(chainG && full)) {
    const int nb0 = min(NB, n);
#pragma unroll
    for (int q = 0; q < NM; ++q)
      if (live(q)) tf_load_diag(cm(q).D, cm(q).M, ld, 0, nb0, tid);
    __syncthreads();
    factor(0, nb0, prof != nullptr && crank == 0, Lsc_of(0));
  }
  stamp();  // diagonal block 0 done
  for (int kb = 0; kb < n; kb += NB) {
    const int nb = min(NB, n - kb);
    const int r0 = kb + nb;
    const int nr = n - r0;
    cluster.sync();  // B1: inverses of block kb in L2; trailing update of block kb - 1 complete
    const int blk = kb / NB;
    const double* Lsc = Lsc_of(blk);
    if (crank < NCH) {
      // ---- the chain CTAs run ONE BLOCK AHEAD of the workers: while those solve the panel of block kb, exchange it and run the
      // trailing update, a chain CTA solves only the 32 panel rows of the NEXT diagonal block itself (X = rows * Linv^T with
      // the inverses it still holds), forms that block's leading tile and factorises it, for each of its matrices.  It has
      // nothing to contribute to the panel barrier (arrives at once, waits when done), so the workers never wait for it there.
      if (nr <= 0) break;
      asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");  // B2 of this block
      if (!(chainG && full)) {
        const int nb2 = min(NB, nr);
        // every global load of this step in flight before the first use: the block's 32 panel rows (column block kb) and the
        // old values of its leading tile -- one L2 round trip instead of one per loop iteration
        constexpr int NS = NB * NB / kTailThreads;                       // 4 staged entries per thread and matrix
        constexpr int NLd = (NB * LD + kTailThreads - 1) / kTailThreads;  // 5 leading-tile entries per thread and matrix
        double s_[NM][NS], o_[NM][NLd];
#pragma unroll
        for (int u = 0; u < NS; ++u) {
          const int e = tid + u * kTailThreads, l = e / NB, c = e % NB;
          const bool in = (l < nb2 && c < nb);
#pragma unroll
          for (int q = 0; q < NM; ++q) s_[q][u] = (in && live(q)) ? __ldcg(cm(q).M + (size_t)(r0 + l) * ld + kb + c) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < NLd; ++u) {
          const int e = tid + u * kTailThreads, i = e / LD, j = e % LD;
          const bool in = (e < NB * LD && i < nb2 && j <= i);
#pragma unroll
          for (int q = 0; q < NM; ++q) o_[q][u] = (in && live(q)) ? __ldcg(cm(q).M + (size_t)(r0 + i) * ld + r0 + j) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < NS; ++u) {
          const int e = tid + u * kTailThreads, l = e / NB, c = e % NB;
#pragma unroll
          for (int q = 0; q < NM; ++q) cm(q).D[l * LD + c] = s_[q][u];
        }
        __syncthreads();
#pragma unroll 1
        for (int e = tid; e < NB * NB; e += kTailThreads) {  // X = rows * Linv^T (rows of a dropped pivot of Linv are zero)
          const int l = e / NB, j = e % NB;
          double s[NM][4] = {};
#pragma unroll 2
          for (int c = 0; c < NB; c += 4) {
#pragma unroll
            for (int q = 0; q < NM; ++q) {
              if (!live(q)) continue;
              double a4[4], l4[4];
              tf_ld4(cm(q).D + l * LD + c, a4); tf_ld4(cm(q).LI + j * LD + c, l4);
#pragma unroll
              for (int t = 0; t < 4; ++t) s[q][t] += a4[t] * l4[t];
            }
          }
#pragma unroll
          for (int q = 0; q < NM; ++q) cm(q).X[l * LD + j] = (s[q][0] + s[q][1]) + (s[q][2] + s[q][3]);
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < NLd; ++u) {  // the next diagonal block = its leading tile of the trailing update
          const int e = tid + u * kTailThreads, i = e / LD, j = e % LD;
          if (e >= NB * LD) break;
          double v[NM] = {};
          if (i < nb2 && j <= i) {
            double s[NM][4] = {};
#pragma unroll 2
            for (int c = 0; c < NB; c += 4) {
#pragma unroll
              for (int q = 0; q < NM; ++q) {
                if (!live(q)) continue;
                double a4[4], b4[4];
                tf_ld4(cm(q).X + i * LD + c, a4); tf_ld4(cm(q).X + j * LD + c, b4);
#pragma unroll
                for (int t = 0; t < 4; ++t) s[q][t] += a4[t] * b4[t];
              }
            }
#pragma unroll
            for (int q = 0; q < NM; ++q) v[q] = o_[q][u] - ((s[q][0] + s[q][1]) + (s[q][2] + s[q][3]));
          }
#pragma unroll
          for (int q = 0; q < NM; ++q) cm(q).D[e] = v[q];
        }
        __syncthreads();
        stamp();  // next diagonal block formed (CTA 0)
        factor(r0, nb2, false, Lsc_of(blk + 1));
        stamp();  // next diagonal block factorised (CTA 0)
      }
      asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");   // B2
      continue;
    }
    wstamp();  // B1 passed
    // phase 2 (CTAs 1..7): the panel below the block, X = rows * Linv^T.  Rows are dealt to the CTAs in contiguous chunks (an
    // even number of rows each); lane = local row, warp w computes columns w, w + 8, w + 16, w + 24; the results go to a scratch
    // panel in L2 that every worker reads back after the barrier.  The W rows of this CTA are solved the same way (local).
    const int chunk = (((nr + NWK - 1) / NWK) + 1) & ~1;
    const int i0 = widx * chunk;
    const int nloc = max(0, min(chunk, nr - i0));
    {
      {  // the inverses of block kb: all loads in flight before the first store
        constexpr int NE = NB * LD / 2, NI = (NE + kTailThreads - 1) / kTailThreads;
        double2 va[NI], vg[NI];
#pragma unroll
        for (int u = 0; u < NI; ++u) {
          const int e = tid + u * kTailThreads;
          if (e < NE) { va[u] = __ldcg(reinterpret_cast<const double2*>(Lsc) + e); if (!full) vg[u] = __ldcg(reinterpret_cast<const double2*>(Lsc + NB * LD) + e); }
        }
#pragma unroll
        for (int u = 0; u < NI; ++u) {
          const int e = tid + u * kTailThreads;
          if (e < NE) { reinterpret_cast<double2*>(LIA)[e] = va[u]; if (!full) reinterpret_cast<double2*>(LIG)[e] = vg[u]; }
        }
      }
      for (int e = tid; e < NB * NB; e += kTailThreads) {
        const int l = e / NB, c = e % NB;
        const bool in = (l < nloc && c < nb);
        DA[l * LD + c] = in ? A[(size_t)(r0 + i0 + l) * ld + kb + c] : 0.0;
        if (!full) DG[l * LD + c] = in ? G[(size_t)(r0 + i0 + l) * ld + kb + c] : 0.0;
        WB[l * LD + c] = (c < nb) ? Ws[(size_t)l * ldt + kb + c] : 0.0;
      }
      __syncthreads();
      double xa[4] = {0.0, 0.0, 0.0, 0.0}, xg[4] = {0.0, 0.0, 0.0, 0.0}, xw[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 2
      for (int c0 = 0; c0 < NB; c0 += 4) {
        double a[4], g[4], w[4];
        tf_ld4(DA + lane * LD + c0, a);
        tf_ld4(WB + lane * LD + c0, w);
        if (!full) tf_ld4(DG + lane * LD + c0, g);
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = warp + 8 * jj;
          double l[4];
          tf_ld4(LIA + j * LD + c0, l);
          xa[jj] += (a[0] * l[0] + a[1] * l[1]) + (a[2] * l[2] + a[3] * l[3]);
          xw[jj] += (w[0] * l[0] + w[1] * l[1]) + (w[2] * l[2] + w[3] * l[3]);
          if (!full) {
            double h[4];
            tf_ld4(LIG + j * LD + c0, h);
            xg[jj] += (g[0] * h[0] + g[1] * h[1]) + (g[2] * h[2] + g[3] * h[3]);
          }
        }
      }
      __syncthreads();  // every warp is done reading the staged rows: DA / DG now take X^T ([j][l]) for the push
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = warp + 8 * jj;
        DA[j * LD + lane] = xa[jj];
        if (!full) DG[j * LD + lane] = xg[jj];
        if (j < nb) Ws[(size_t)lane * ldt + kb + j] = xw[jj];  // final
        XT[j * NB + lane] = (j < nb) ? xw[jj] : 0.0;
      }
      __syncthreads();
      // this CTA's rows of the solved panel -> global scratch (transposed); every CTA reads the whole panel after the barrier
      for (int e = tid; e < NB * nloc; e += kTailThreads) {
        const int j = e / nloc, l = e % nloc;
        Psc[(size_t)j * ldt + i0 + l] = DA[j * LD + l];
        if (!full) Psc[(size_t)(NB + j) * ldt + i0 + l] = DG[j * LD + l];
      }
    }
    wstamp();  // panel computed
    if (nr <= 0) break;  // last block: the W rows are complete
    cluster.sync();
    wstamp();  // B2 passed
    {
      const int nr2 = (nr + 1) >> 1;  // 16-byte loads; an odd last column picks up the (finite) neighbour, zeroed below
      const int tot = NB * nr2;
      for (int e0 = tid; e0 < tot; e0 += 4 * kTailThreads) {  // 4 (8) loads in flight per thread before the first store
        double2 va[4], vg[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = e0 + u * kTailThreads;
          if (e < tot) {
            const int j = e / nr2, l2 = 2 * (e % nr2);
            va[u] = __ldcg(reinterpret_cast<const double2*>(Psc + (size_t)j * ldt + l2));
            if (!full) vg[u] = __ldcg(reinterpret_cast<const double2*>(Psc + (size_t)(NB + j) * ldt + l2));
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = e0 + u * kTailThreads;
          if (e < tot) {
            const int j = e / nr2, l2 = 2 * (e % nr2);
            *reinterpret_cast<double2*>(PT_A + (size_t)j * ldt + l2) = va[u];
            if (!full) *reinterpret_cast<double2*>(PT_G + (size_t)j * ldt + l2) = vg[u];
          }
        }
      }
      __syncthreads();
      const int nrp = (nr + 3) & ~3;  // zero the tail of the padded rows so that partial tiles read zeros
      for (int e = tid; e < (nrp - nr) * NB; e += kTailThreads) {
        const size_t o = (size_t)(e / (nrp - nr)) * ldt + nr + e % (nrp - nr);
        PT_A[o] = 0.0;
        if (!full) PT_G[o] = 0.0;
      }
      __syncthreads();
    }
    wstamp();  // panel exchanged
    // phase 3.  CTA 0: the next diagonal block = leading 32 x 32 tile of the trailing update, formed from the panel
    // straight into shared memory, then factorised.  CTAs 1..7: the rest of the trailing update, 4x4 register tiles on
    // the transposed panels -- the lower-triangle tiles of A, then of G (rows >= 32 of the trailing matrix), dealt in
    // contiguous runs (neighbouring lanes read neighbouring columns: no bank conflicts); then their own W tiles.
    {
      const int nt = (nr + 3) / 4, ntile = nt * (nt + 1) / 2;
      constexpr int kLead = (NB / 4) * (NB / 4 + 1) / 2;  // tiles of the leading 32 x 32 block: CTA 0's
      const int nrest = max(0, ntile - kLead);
      const int nitems = full ? nrest : 2 * nrest;
      const int run = (nitems + NWK - 1) / NWK;
      const int first = widx * run;
      const int mine = max(0, min(run, nitems - first));
      const int nloc3 = mine + ncw4 * nt;
      for (int q = tid; q < nloc3; q += kTailThreads) {
        if (q < mine) {
          const int it = first + q;
          const bool isG = it >= nrest;
          int ti, tj;
          tri_tile_index((isG ? it - nrest : it) + kLead, ti, tj);
          tc_update_tile<NB>((isG ? G : A) + (size_t)r0 * ld + r0, isG ? PT_G : PT_A, ldt, ld, ti, tj, nr);
        } else {
          const int w = q - mine, ti = w % nt, c4 = w / nt;
          double acc[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
          tc_tile_4x4(XT, PT_A, NB, ldt, 4 * c4, 4 * ti, NB, acc);
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            double2* dst = reinterpret_cast<double2*>(Ws + (size_t)(4 * c4 + p) * ldt + r0 + 4 * ti);
            double2 v0 = dst[0], v1 = dst[1];
            v0.x -= acc[p][0]; v0.y -= acc[p][1]; v1.x -= acc[p][2]; v1.y -= acc[p][3];
            dst[0] = v0; dst[1] = v1;
          }
        }
      }
    }
    wstamp();  // trailing update + W tiles done
  }
  cluster.sync();
  if (gtid == 0) {
    *rank_out = s_rankA;
    if (NCH == 2 && s_timeout) ua.m_out[2] = 1;  // reported by msckf_b200_fetch as MSCKF_B200_ERR_NUMERIC
  }
  for (int e = tid; e < n * cw; e += kTailThreads) {
    const int row = e / cw, cc = e % cw, col = col0 + cc;
    const double v = Ws[(size_t)cc * ldt + row];
    if (col < n) Wm[(size_t)row * ld + col] = v; else yv[row] = v;
  }
  stamp();  // end
  if (prof && blockIdx.x == 0 && tid == 0) prof[prof_i] = 0ull;
}

}  // namespace mb
