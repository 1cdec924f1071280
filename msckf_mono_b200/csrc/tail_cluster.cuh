// msckf_mono_b200/csrc/tail_cluster.cuh
// The serial part of the EKF tail for LARGE windows (15 + 6M > ~220: the fused form of tail_fused.cuh does not fit the
// shared memory of a CTA any more) as ONE thread-block-cluster kernel (8 CTAs on 8 SMs of one GPC):
//     Gamma (Gram matrix of the basis)      -> rank decision        }  rank-revealing Cholesky of Gamma and S''
//     S'' = L L^T over the kept indices                              }  in lockstep, blocked by NB
//     W = L^-1 [T''P | r'']                                         (forward substitution as a second sweep, RHS columns
//                                                                    sharded over the cluster)
// followed by  P <- P - W^T W, dx = W^T y and the state injection (k_syrk, all SMs)   (msckf.h:1373-1418)
// The matrices stay in global memory (they are L2 resident: n <= 639, fp64); cluster barriers (release/acquire
// at cluster scope) order the phases.  Diagonal blocks: one warp of CTA 0; panel rows: solved redundantly by every CTA
// (one thread per row) into a transposed shared panel; trailing update: 4x4 register tiles dealt to the CTAs.
// This is the first-generation design; tail_fused.cuh documents what was measured on it and changed for the default
// path.  Also shared with tail_fused.cuh: the tile helpers below.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"

namespace mb {
namespace cg = cooperative_groups;

constexpr int kTailThreads = 256;

template <int NB>
__device__ __forceinline__ void tc_load_diag(double* D, const double* A, int ld, int kb, int nb, int tid) {
  for (int e = tid; e < NB * NB; e += kTailThreads) {
    const int i = e / NB, j = e % NB;
    double v = (i == j) ? 1.0 : 0.0;  // identity padding when nb < NB
    if (i < nb && j < nb) v = (j <= i) ? A[(size_t)(kb + i) * ld + kb + j] : 0.0;
    D[i * (NB + 1) + j] = v;
  }
}

// one panel row: x D^T = a with the row in registers; inv[] holds 1 / D_jj (0 for dropped columns); the solved row
// is written transposed into the shared panel PT (and optionally back to global)
template <int NB>
__device__ __forceinline__ void tc_panel_row(const double* Mx, int ld, int row, int kb, int nb, const double* D, const double* inv,
                                             double* PT, int ldt, int prow, double* Lw /*nullable: where the solved row goes*/) {
  constexpr int LD = NB + 1;
  double x[NB];
#pragma unroll
  for (int j = 0; j < NB; ++j) x[j] = (j < nb) ? Mx[(size_t)row * ld + kb + j] : 0.0;
#pragma unroll
  for (int j = 0; j < NB; ++j) {  // right-looking: the updates of the later entries are independent (full ILP)
    x[j] *= inv[j];
#pragma unroll
    for (int jj = j + 1; jj < NB; ++jj) x[jj] -= x[j] * D[jj * LD + j];
  }
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    PT[(size_t)j * ldt + prow] = x[j];
    if (Lw && j < nb) Lw[(size_t)row * ld + kb + j] = x[j];
  }
}

// C[4][4] += sum_j At[j][ra..ra+3] * Bt[j][rb..rb+3] over nk rows of the (transposed) operands, row strides lda / ldb
__device__ __forceinline__ void tc_tile_4x4(const double* At, const double* Bt, int lda, int ldb, int ra, int rb, int nk, double acc[4][4]) {
#pragma unroll 4
  for (int j = 0; j < nk; ++j) {
    const double2 a01 = *reinterpret_cast<const double2*>(At + (size_t)j * lda + ra);
    const double2 a23 = *reinterpret_cast<const double2*>(At + (size_t)j * lda + ra + 2);
    const double2 b01 = *reinterpret_cast<const double2*>(Bt + (size_t)j * ldb + rb);
    const double2 b23 = *reinterpret_cast<const double2*>(Bt + (size_t)j * ldb + rb + 2);
    const double a[4] = {a01.x, a01.y, a23.x, a23.y}, b[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[p][q] += a[p] * b[q];
  }
}

// trailing-update tile (ti >= tj) of a symmetric matrix from its transposed panel: Mat[i][i2] -= sum_j PT[j][i] PT[j][i2]
// over the NB panel rows, on the entries of the lower triangle with i < nr
template <int NB>
__device__ __forceinline__ void tc_update_tile(double* Mat, const double* PT, int ldt, int ld, int ti, int tj, int nr) {
  double old[4][4];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {  // issue the loads of the old values before the FMA chain
      const int i = 4 * ti + p, i2 = 4 * tj + q;
      old[p][q] = (i < nr && i2 <= i) ? Mat[(size_t)i * ld + i2] : 0.0;
    }
  double acc[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
  tc_tile_4x4(PT, PT, ldt, ldt, 4 * ti, 4 * tj, NB, acc);
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = 4 * ti + p, i2 = 4 * tj + q;
      if (i < nr && i2 <= i) Mat[(size_t)i * ld + i2] = old[p][q] - acc[p][q];
    }
}

// one W row (an RHS column of the substitution, kept in shared memory): solve its NB entries of the current block in
// registers, write them back (they are final) and, transposed, into XT for the tile update of the remaining entries
template <int NB>
__device__ __forceinline__ void tc_w_row(double* wrow, int nb, const double* D, const double* inv, double* XT, int c) {
  constexpr int LD = NB + 1;
  double x[NB];
#pragma unroll
  for (int j = 0; j < NB; ++j) x[j] = (j < nb) ? wrow[j] : 0.0;
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    x[j] *= inv[j];
#pragma unroll
    for (int jj = j + 1; jj < NB; ++jj) x[jj] -= x[j] * D[jj * LD + j];
  }
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    XT[j * NB + c] = x[j];
    if (j < nb) wrow[j] = x[j];
  }
}

// W = L^-1 [TP | r''] as a separate sweep over the finished factor (windows too large for the fused form): RHS columns
// sharded over the cluster, per chunk the L panel of each block is staged in shared memory
template <int NB>
__device__ __forceinline__ void tc_substitute(int n, int ld, int C, int crank, int tid, const double* __restrict__ Lout,
                                              const double* __restrict__ idiag, const int* __restrict__ keep,
                                              const double* __restrict__ TP, const double* __restrict__ r2, double* __restrict__ Wm,
                                              double* __restrict__ yv, double* DA, double* ida, double* Ws /*[n][per]*/,
                                              double* Lp /*[n][NB]*/, int* skeep /*[n]*/) {
  constexpr int LD = NB + 1;
  const int ncol = n + 1;
  const int per = max(1, min(NB, (ncol + C - 1) / C));  // columns per chunk: Ws [n][per] fits the A-panel buffer
  const int nchunk = (ncol + per - 1) / per;
  for (int k = tid; k < n; k += kTailThreads) skeep[k] = keep[k];
  for (int q = crank; q < nchunk; q += C) {
    const int col0 = q * per, cw = min(per, ncol - col0);
    __syncthreads();
    for (int e = tid; e < n * cw; e += kTailThreads) {
      const int row = e / cw, cc = e % cw, col = col0 + cc;
      double v = 0.0;
      if (skeep[row]) v = (col < n) ? TP[(size_t)row * ld + col] : r2[row];
      Ws[(size_t)row * per + cc] = v;
    }
    const int rgs = kTailThreads / cw;  // row groups for the update
    const int ucc = tid % cw, urg = tid / cw;
    for (int kb = 0; kb < n; kb += NB) {
      const int nb = min(NB, n - kb), r0 = kb + nb;
      __syncthreads();
      tc_load_diag<NB>(DA, Lout, ld, kb, nb, tid);
      if (tid < NB) ida[tid] = (tid < nb) ? idiag[kb + tid] : 0.0;
      for (int e = tid; e < (n - r0) * NB; e += kTailThreads) {  // coalesced panel load
        const int i = e / NB, j = e % NB;
        Lp[(size_t)i * NB + j] = (j < nb) ? Lout[(size_t)(r0 + i) * ld + kb + j] : 0.0;
      }
      __syncthreads();
      double x[NB];
      if (urg < rgs) {
        // every row group solves the diagonal block for its column redundantly (registers), then updates its rows
#pragma unroll
        for (int j = 0; j < NB; ++j) x[j] = (j < nb) ? Ws[(size_t)(kb + j) * per + ucc] : 0.0;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          x[j] *= ida[j];
#pragma unroll
          for (int jj = j + 1; jj < NB; ++jj) x[jj] -= x[j] * DA[jj * LD + j];
        }
      }
      __syncthreads();  // everybody has read the old block rows
      if (urg < rgs) {
        if (urg == 0) {
#pragma unroll
          for (int j = 0; j < NB; ++j)
            if (j < nb) Ws[(size_t)(kb + j) * per + ucc] = x[j];
        }
        for (int i = urg; i < n - r0; i += rgs) {
          const double* lrow = Lp + (size_t)i * NB;
          double s = 0.0;
#pragma unroll
          for (int j = 0; j < NB; j += 2) {
            const double2 l2 = *reinterpret_cast<const double2*>(lrow + j);
            s += l2.x * x[j] + l2.y * x[j + 1];
          }
          Ws[(size_t)(r0 + i) * per + ucc] -= s;
        }
      }
    }
    __syncthreads();
    for (int e = tid; e < n * cw; e += kTailThreads) {
      const int row = e / cw, cc = e % cw, col = col0 + cc;
      const double v = Ws[(size_t)row * per + cc];
      if (col < n) Wm[(size_t)row * ld + col] = v; else yv[row] = v;
    }
  }
}

template <class S, int NB>
__global__ void __launch_bounds__(kTailThreads) k_tail(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& ua = args[blockIdx.z];
  if (ua.n_tracks == 0 || ua.tail_kind != (NB == 32 ? 1 : 2)) return;  // (uniform over the cluster)
  const int n = ua.n, ld = ua.ld;
  const double* __restrict__ T2 = ua.T2;
  double* __restrict__ G = ua.G;
  double* __restrict__ A = ua.S2;
  double* __restrict__ Lout = ua.R2;     // receives L (R'' is consumed by k_gemm_s)
  int* __restrict__ keep = ua.keep;
  double* __restrict__ idiag = ua.idiag;
  const double thr = ua.rank_thr;
  int* __restrict__ rank_out = ua.rank_out;
  const int* __restrict__ m_in = ua.m_out;
  const double* __restrict__ TP = ua.TP;
  const double* __restrict__ r2 = ua.r2;
  double* __restrict__ Wm = ua.W;
  double* __restrict__ yv = ua.y;
  double* __restrict__ dx_out = ua.dx;
  unsigned long long* __restrict__ prof = ua.prof;  // optional phase timestamps
  static_assert(NB <= 32, "the diagonal block is factorised by one warp, one row per lane");
  cg::cluster_group cluster = cg::this_cluster();
  int prof_i = 0;
  auto stamp = [&]() {
    if (prof && blockIdx.x == 0 && threadIdx.x == 0 && prof_i < 64) prof[prof_i++] = globaltimer();
  };
  stamp();
  const int crank = (int)cluster.block_rank();
  const int C = (int)cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int LD = NB + 1;
  extern __shared__ __align__(16) double sm[];
  const int ldt = (n + 3) & ~3;              // row stride of the transposed panels (16-byte aligned rows)
  double* DG = sm;                           // [NB][LD]
  double* DA = DG + NB * LD;                 // [NB][LD]
  double* PT_A = DA + NB * LD + ((NB * LD) & 1);  // [NB][ldt]  panel of A, transposed (later: W slab, W k-blocks)
  double* PT_G = PT_A + (size_t)NB * ldt;    // [NB][ldt]  panel of G, transposed (later: L panel, dx)
  double* d0 = PT_G + (size_t)NB * ldt;      // [n] original diagonal of Gamma (CTA 0); later keep flags
  double* idg = d0 + ((n + 1) & ~1);         // [NB] 1 / diag of the current block of G's factor (0 = dropped)
  double* ida = idg + NB;                    // [NB] same for A
  __shared__ int s_rank;
  const int m = *m_in;
  const bool full = m <= n;  // all rows explicit and orthonormal: Gamma = I_m, nothing to decide, G untouched
  const int rank_cap = min(m, n);
  const int gtid = crank * kTailThreads + tid, gthreads = C * kTailThreads;

  if (m == 0) {  // nothing accepted: the reference returns before touching the state (msckf.h:401-403, :1328)
    for (int a = gtid; a < n; a += gthreads) dx_out[a] = 0.0;
    if (gtid == 0) *rank_out = 0;
    return;
  }
  // ---------------------------------------------------------------- Gamma = [[I_h, H_h], [H_h^T, Lambda]] from T''
  if (!full) {
    const size_t total = (size_t)n * n;
    for (size_t e = gtid; e < total; e += gthreads) {
      const int a = (int)(e / n), b = (int)(e % n);
      double v;
      if (a < kImuDim && b < kImuDim) v = (a == b) ? 1.0 : 0.0;
      else if (a < kImuDim) v = T2[(size_t)a * ld + b];
      else if (b < kImuDim) v = T2[(size_t)b * ld + a];
      else v = T2[(size_t)a * ld + b];
      G[(size_t)a * ld + b] = v;
    }
  }
  cluster.sync();
  stamp();  // Gamma built
  if (crank == 0) {
    for (int k = tid; k < n; k += kTailThreads) {
      d0[k] = full ? (k < m ? 1.0 : 0.0) : G[(size_t)k * ld + k];
      if (crank == 0) ua.pivr[n + k] = d0[k];  // (diagnostics: the denominators of msckf_b200_rank_pivots)
    }
    if (tid == 0) s_rank = 0;
  }
  __syncthreads();
  // ---------------------------------------------------------------- blocked rank-revealing Cholesky (G decides, A follows)
  for (int kb = 0; kb < n; kb += NB) {
    const int nb = min(NB, n - kb);
    const int r0 = kb + nb;
    // phase 1 (CTA 0): diagonal blocks, one warp, lane = row, both matrices interleaved, no divisions (rsqrt)
    if (crank == 0) {
      if (!full) tc_load_diag<NB>(DG, G, ld, kb, nb, tid);
      tc_load_diag<NB>(DA, A, ld, kb, nb, tid);
      __syncthreads();
      if (warp == 0) {
        int rank_now = s_rank;
        for (int k = 0; k < nb; ++k) {
          // left-looking: column k of both factors from the already final columns j < k (reads only, no RMW chain)
          double sa = 0.0, sg = 0.0;
          if (lane >= k && lane < nb) {
            sa = DA[lane * LD + k];
            if (!full) sg = DG[lane * LD + k];
            double a4[4] = {0.0, 0.0, 0.0, 0.0}, g4[4] = {0.0, 0.0, 0.0, 0.0};  // 4 partial sums: short FMA chains
            int j = 0;
            for (; j + 4 <= k; j += 4) {
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                a4[u] += DA[lane * LD + j + u] * DA[k * LD + j + u];
                if (!full) g4[u] += DG[lane * LD + j + u] * DG[k * LD + j + u];
              }
            }
            for (; j < k; ++j) { a4[0] += DA[lane * LD + j] * DA[k * LD + j]; if (!full) g4[0] += DG[lane * LD + j] * DG[k * LD + j]; }
            sa -= (a4[0] + a4[1]) + (a4[2] + a4[3]);
            sg -= (g4[0] + g4[1]) + (g4[2] + g4[3]);
          }
          const double pa = __shfl_sync(0xffffffffu, sa, k), pg = full ? 1.0 : __shfl_sync(0xffffffffu, sg, k);
          const double dk0 = d0[kb + k];
          const bool drop = !(dk0 > 0.0) || !(pg > thr * dk0) || rank_now >= rank_cap || !(pa > 0.0);
          if (!drop) rank_now++;
          if (lane == 0) ua.pivr[kb + k] = pg;
          const double ig = drop ? 0.0 : rsqrt(pg), ia = drop ? 0.0 : rsqrt(pa);
          __syncwarp();
          if (lane > k && lane < nb) { DA[lane * LD + k] = sa * ia; if (!full) DG[lane * LD + k] = sg * ig; }
          if (lane == k) {
            DA[k * LD + k] = drop ? 1.0 : pa * ia; DG[k * LD + k] = drop ? 1.0 : pg * ig;
            ida[k] = ia; idg[k] = ig;
          }
          if (drop && lane < k) { DA[k * LD + lane] = 0.0; DG[k * LD + lane] = 0.0; }
          __syncwarp();
        }
        if (lane == 0) s_rank = rank_now;
        for (int k = nb + lane; k < NB; k += 32) { ida[k] = 0.0; idg[k] = 0.0; }
      }
      __syncthreads();
      for (int e = tid; e < nb * nb; e += kTailThreads) {
        const int i = e / nb, j = e % nb;
        if (j <= i) {
          A[(size_t)(kb + i) * ld + kb + j] = DA[i * LD + j];     // read by the other CTAs in phase 2
          Lout[(size_t)(kb + i) * ld + kb + j] = DA[i * LD + j];  // the factor itself (A's panels stay
          if (!full) G[(size_t)(kb + i) * ld + kb + j] = DG[i * LD + j];  // untouched: the whole cluster is reading them)
        }
      }
      if (tid < nb) { keep[kb + tid] = ida[tid] != 0.0 ? 1 : 0; idiag[kb + tid] = ida[tid]; idiag[n + kb + tid] = idg[tid]; }
    }
    stamp();  // diagonal block done
    if (r0 >= n) break;  // last block: nothing below
    cluster.sync();
    // phase 2 (every CTA, redundantly): all panel rows below the block -> transposed shared panel (CTA 0 also -> global)
    if (crank != 0) {
      if (!full) tc_load_diag<NB>(DG, G, ld, kb, nb, tid);
      tc_load_diag<NB>(DA, A, ld, kb, nb, tid);
      if (tid < NB) { ida[tid] = (tid < nb) ? idiag[kb + tid] : 0.0; idg[tid] = (tid < nb) ? idiag[n + kb + tid] : 0.0; }
    }
    __syncthreads();
    const int nr = n - r0;
    for (int row = r0 + tid; row < n; row += kTailThreads) {
      tc_panel_row<NB>(A, ld, row, kb, nb, DA, ida, PT_A, ldt, row - r0, crank == 0 ? Lout : nullptr);
      if (!full) tc_panel_row<NB>(G, ld, row, kb, nb, DG, idg, PT_G, ldt, row - r0, nullptr);
    }
    {  // zero the tail of the padded rows so that partial tiles read zeros
      const int nrp = (nr + 3) & ~3;
      for (int e = tid; e < (nrp - nr) * NB; e += kTailThreads) {
        const int j = e / (nrp - nr), i = nr + e % (nrp - nr);
        PT_A[(size_t)j * ldt + i] = 0.0;
        if (!full) PT_G[(size_t)j * ldt + i] = 0.0;
      }
    }
    __syncthreads();
    stamp();  // panel done
    // phase 3 (cluster-wide): trailing update, 4x4 register tiles on the transposed panel.  Work items: the lower-triangle
    // tiles of A, then of G, dealt round-robin to the CTAs.
    {
      const int nt = (nr + 3) / 4, ntile = nt * (nt + 1) / 2;
      const int nitems = full ? ntile : 2 * ntile;
      const int mine = (nitems > crank) ? (nitems - crank + C - 1) / C : 0;
      const int nloc = mine;
      for (int q = tid; q < nloc; q += kTailThreads) {
        if (q < mine) {
          const int it = crank + C * q;
          const bool isG = it >= ntile;
          int ti, tj;
          tri_tile_index(isG ? it - ntile : it, ti, tj);
          tc_update_tile<NB>((isG ? G : A) + (size_t)r0 * ld + r0, isG ? PT_G : PT_A, ldt, ld, ti, tj, nr);
        }
      }
    }
    stamp();  // trailing computed (CTA 0)
    cluster.sync();
    stamp();  // trailing done
  }
  cluster.sync();
  if (gtid == 0) *rank_out = s_rank;
  {
    // dropped rows: clear what earlier panels wrote left of the diagonal
    for (size_t e = gtid; e < (size_t)n * n; e += gthreads) {
      const int k = (int)(e / n), cc = (int)(e % n);
      if (cc < k && !keep[k]) Lout[(size_t)k * ld + cc] = 0.0;
    }
    cluster.sync();
    stamp();  // factorisation complete
    tc_substitute<NB>(n, ld, C, crank, tid, Lout, idiag, keep, TP, r2, Wm, yv, DA, ida, PT_A, PT_G, reinterpret_cast<int*>(d0));
  }
  stamp();  // substitution complete (this CTA)
  stamp();  // end
  if (prof && blockIdx.x == 0 && threadIdx.x == 0 && prof_i < 64) prof[prof_i] = 0ull;
}


}  // namespace mb
