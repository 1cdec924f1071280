// msckf_mono_b200/csrc/gram_kernels.cuh
// Compression of the stacked measurement (msckf.h:1343-1366) in projector / Gram form.
//
// The reference keeps Q_1 = the first n columns of the Householder Q of the stacked H_o (rows 0..14 pass
// through because the 15 leading columns of H_o are zero) and forms T_H = Q_1^T H_o, r_n = Q_1^T r_o,
// R_n = Q_1^T R_o Q_1.  The EKF update only depends on span(Q_1) = span(E_15) + range(H_o) (+ directions
// of numerically zero pivots, which are rounding noise in the reference).  We use the basis
// Q'' = [E_15 | H_c] (H_c = H_o(:,15:)) of that subspace directly:
//     T'' = Q''^T H_o   = [[0, H_o(0:15,15:)], [0, Lambda]],    Lambda = H_c^T H_c
//     r'' = Q''^T r_o   = [r_o(0:15); beta],                    beta   = H_c^T r_o
//     R'' = Q''^T R_o Q''= [[R_o(0:15,0:15), (R_o H_c)(0:15,:)], [sym, Psi]],  Psi = H_c^T R_o H_c
// and since H_o,j = A_j^T X_j with A_j A_j^T = I - U_j U_j^T (U_j = first 3 columns of the per-feature Q),
//     Lambda = blkdiag(sum X_ji^T X_ji)     - Z^T Z            Z_j  = U_j^T X_j
//     Psi    = blkdiag(sum X_ji^T D X_ji)   - Z^T Yq - Yq^T Z   Yq_j = U_j^T D X_j - 1/2 (U_j^T D U_j) Z_j
//     beta   = blk(sum X_ji^T r_ji)         - Z^T (U^T r)
// so the stacked m x n matrix is never materialised: the Gram terms are one (c x 3N)(3N x c) GEMM pair.
// All accumulation is fp64 (for both filter precisions).
#pragma once
#include "common.cuh"

namespace mb {

constexpr int GT = 32;   // output tile
constexpr int GK = 16;   // k-step
constexpr int kMaxSplit = 16;  // split-K chunks of the Gram products, at most

// Partial Gram products over a K-split: G1p[s] = Z^T Z, G2p[s] = Z^T Yq + Yq^T Z, upper tiles only.
template <class S>
__global__ void __launch_bounds__(256) k_gram(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int K = A.K, c = A.n - kImuDim, kchunk = A.kchunk;
  const double* __restrict__ Z = A.Z;
  const double* __restrict__ Yq = A.Yq;
  double* __restrict__ G1p = A.G1p;
  double* __restrict__ G2p = A.G2p;
  __shared__ double sZa[GK][GT + 1], sZb[GK][GT + 1], sYa[GK][GT + 1], sYb[GK][GT + 1];
  __shared__ double sU[GK], sBz[8][GT + 1];
  const double* __restrict__ ur = A.ur;
  // decode the (ta <= tb) tile pair
  const int ntile = (c + GT - 1) / GT;
  if ((int)blockIdx.x >= ntile * (ntile + 1) / 2 || (int)blockIdx.y >= A.nsplit || A.n_tracks == 0 || A.gram_mma) return;
  int pidx = blockIdx.x, ta = 0;
  while (pidx >= ntile - ta) { pidx -= ntile - ta; ++ta; }
  const int tb = ta + pidx;
  const int split = blockIdx.y;
  const int k0 = split * kchunk, k1 = min(K, k0 + kchunk);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 2x2 outputs each
  double a1[2][2] = {{0, 0}, {0, 0}}, a2[2][2] = {{0, 0}, {0, 0}};
  // the diagonal tiles also accumulate this split's part of Z^T (U^T r) for their 32 columns (beta of the header): the
  // operand is in shared memory anyway; thread = (column, one of 8 k-groups)
  const bool diag = ta == tb;
  const int bc = threadIdx.x & 31, bg = threadIdx.x >> 5;
  double bz = 0.0;
  // operands of the next k-slab are fetched into registers while the current one is multiplied (the slabs are L2 hits of
  // microsecond latency; without the prefetch the kernel sat in long-scoreboard stalls: ncu)
  constexpr int NF = GK * GT / 256;
  double fza[NF], fya[NF], fzb[NF], fyb[NF], fu = 0.0;
  auto fetch = [&](int kb) {
#pragma unroll
    for (int u = 0; u < NF; ++u) {
      const int e = threadIdx.x + 256 * u, kk = e / GT, cc = e % GT;
      const int k = kb + kk;
      const int ca = ta * GT + cc, cb = tb * GT + cc;
      const bool kin = k < k1;
      fza[u] = (kin && ca < c) ? Z[(size_t)k * c + ca] : 0.0;
      fya[u] = (kin && ca < c) ? Yq[(size_t)k * c + ca] : 0.0;
      fzb[u] = diag ? fza[u] : ((kin && cb < c) ? Z[(size_t)k * c + cb] : 0.0);
      fyb[u] = diag ? fya[u] : ((kin && cb < c) ? Yq[(size_t)k * c + cb] : 0.0);
    }
    if (diag && threadIdx.x < GK) fu = (kb + (int)threadIdx.x < k1) ? ur[kb + threadIdx.x] : 0.0;
  };
  fetch(k0);
  for (int kb = k0; kb < k1; kb += GK) {
    if (diag && threadIdx.x < GK) sU[threadIdx.x] = fu;
#pragma unroll
    for (int u = 0; u < NF; ++u) {
      const int e = threadIdx.x + 256 * u, kk = e / GT, cc = e % GT;
      sZa[kk][cc] = fza[u]; sYa[kk][cc] = fya[u]; sZb[kk][cc] = fzb[u]; sYb[kk][cc] = fyb[u];
    }
    __syncthreads();
    if (kb + GK < k1) fetch(kb + GK);
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      const double za0 = sZa[kk][ty], za1 = sZa[kk][ty + 16], ya0 = sYa[kk][ty], ya1 = sYa[kk][ty + 16];
      const double zb0 = sZb[kk][tx], zb1 = sZb[kk][tx + 16], yb0 = sYb[kk][tx], yb1 = sYb[kk][tx + 16];
      a1[0][0] += za0 * zb0; a1[0][1] += za0 * zb1; a1[1][0] += za1 * zb0; a1[1][1] += za1 * zb1;
      a2[0][0] += za0 * yb0 + ya0 * zb0; a2[0][1] += za0 * yb1 + ya0 * zb1;
      a2[1][0] += za1 * yb0 + ya1 * zb0; a2[1][1] += za1 * yb1 + ya1 * zb1;
    }
    if (diag) bz += sZa[2 * bg][bc] * sU[2 * bg] + sZa[2 * bg + 1][bc] * sU[2 * bg + 1];
    __syncthreads();
  }
  if (diag) {
    sBz[bg][bc] = bz;
    __syncthreads();
    if (bg == 0 && ta * GT + bc < c) {
      double t = 0.0;
#pragma unroll
      for (int g = 0; g < 8; ++g) t += sBz[g][bc];
      A.bzp[(size_t)split * c + ta * GT + bc] = t;
    }
  }
  double* o1 = G1p + (size_t)split * c * c;
  double* o2 = G2p + (size_t)split * c * c;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int ra = ta * GT + ty + 16 * i, cb = tb * GT + tx + 16 * j;
      if (ra < c && cb < c) { o1[(size_t)ra * c + cb] = a1[i][j]; o2[(size_t)ra * c + cb] = a2[i][j]; }
    }
}

// The same partial Gram products on the FP64 tensor-core path: mma.sync.aligned.m8n8k4.row.col.f64 (SASS: DMMA), 4 warps per
// CTA, one 32 x 32 output tile per CTA, each warp a 16 x 16 quadrant = 2 x 2 MMA tiles for G1 and for G2, issued as two
// m16n8k4 per product (6 DMMA per 4-deep k-step against 8 fragment loads; the SIMT form above needs 32 LDS + 48 DFMA warp
// instructions for the same k-step).  m16n8k4 computes each output as two m8n8k4 would, bit for bit, in half the DMMA
// instructions: 53.7 -> 49.6 us at a batch of 8 config-B filters, 17.1 -> 15.1 us for one (H100 80GB HBM3, 700 W).
// 3 CTAs per SM, as without the bound (168 registers).
// Fragments (PTX ISA, m8n8k4 .f64): A (8x4, row): lane l holds A[l/4][l%4]; B (4x8, col): lane l holds B[l%4][l/4];
// C/D (8x8): lane l holds C[l/4][2(l%4)] and C[l/4][2(l%4)+1].  Here A = Z^T (or Yq^T) and B = Z (or Yq) of a k-slab
// staged in shared memory k-major with a row stride of 36 doubles (== 4 mod 16: the 16 lanes of a half warp hit 16 banks pairs).
// Accumulation order differs from k_gram (fixed, deterministic): results agree to fp64 rounding.
constexpr int GL = GT + 4;
__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
// Both 8 x 8 row tiles of a quadrant column in one m16n8k4: rows 0-7 (c0, a[0]) and rows 8-15 (c8, a[1]); lane l holds
// A[l/4][l%4] and A[8 + l/4][l%4], B[l%4][l/4], C[l/4][2(l%4) + {0,1}] and C[8 + l/4][2(l%4) + {0,1}].
__device__ __forceinline__ void dmma16(double (&c0)[2], double (&c8)[2], const double (&a)[2], double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c0[0]), "+d"(c0[1]), "+d"(c8[0]), "+d"(c8[1]) : "d"(a[0]), "d"(a[1]), "d"(b));
}
template <class S>
__global__ void __launch_bounds__(128, 3) k_gram_mma(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int K = A.K, c = A.n - kImuDim, kchunk = A.kchunk;
  const double* __restrict__ Z = A.Z;
  const double* __restrict__ Yq = A.Yq;
  __shared__ double sZa[GK][GL], sZb[GK][GL], sYa[GK][GL], sYb[GK][GL];
  __shared__ double sU[GK], sBz[4][GT + 1];
  const double* __restrict__ ur = A.ur;
  const int ntile = (c + GT - 1) / GT;
  if ((int)blockIdx.x >= ntile * (ntile + 1) / 2 || (int)blockIdx.y >= A.nsplit || A.n_tracks == 0 || !A.gram_mma) return;
  int pidx = blockIdx.x, ta = 0;
  while (pidx >= ntile - ta) { pidx -= ntile - ta; ++ta; }
  const int tb = ta + pidx;
  const int split = blockIdx.y;
  const int k0 = split * kchunk, k1 = min(K, k0 + kchunk);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp >> 1) * 16, wn = (warp & 1) * 16;  // this warp's quadrant
  const int fr = lane >> 2, fk = lane & 3;
  double c1[2][2][2], c2[2][2][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) { c1[i][j][0] = c1[i][j][1] = 0.0; c2[i][j][0] = c2[i][j][1] = 0.0; }
  const bool diag = ta == tb;  // (see k_gram: this split's part of Z^T (U^T r); thread = (column, one of 4 k-groups))
  double bzs = 0.0;
  constexpr int NF = GK * GT / 128;  // register prefetch of the next k-slab (see k_gram)
  double fza[NF], fya[NF], fzb[NF], fyb[NF], fu = 0.0;
  auto fetch = [&](int kb) {
#pragma unroll
    for (int u = 0; u < NF; ++u) {
      const int e = tid + 128 * u, kk = e / GT, cc = e % GT;
      const int k = kb + kk;
      const int ca = ta * GT + cc, cb = tb * GT + cc;
      const bool kin = k < k1;
      fza[u] = (kin && ca < c) ? Z[(size_t)k * c + ca] : 0.0;
      fya[u] = (kin && ca < c) ? Yq[(size_t)k * c + ca] : 0.0;
      fzb[u] = diag ? fza[u] : ((kin && cb < c) ? Z[(size_t)k * c + cb] : 0.0);
      fyb[u] = diag ? fya[u] : ((kin && cb < c) ? Yq[(size_t)k * c + cb] : 0.0);
    }
    if (diag && tid < GK) fu = (kb + tid < k1) ? ur[kb + tid] : 0.0;
  };
  fetch(k0);
  for (int kb = k0; kb < k1; kb += GK) {
    if (diag && tid < GK) sU[tid] = fu;
#pragma unroll
    for (int u = 0; u < NF; ++u) {
      const int e = tid + 128 * u, kk = e / GT, cc = e % GT;
      sZa[kk][cc] = fza[u]; sYa[kk][cc] = fya[u]; sZb[kk][cc] = fzb[u]; sYb[kk][cc] = fyb[u];
    }
    __syncthreads();
    if (kb + GK < k1) fetch(kb + GK);
#pragma unroll
    for (int ks = 0; ks < GK; ks += 4) {
      double az[2], ay[2], bz[2], by[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) { az[i] = sZa[ks + fk][wm + 8 * i + fr]; ay[i] = sYa[ks + fk][wm + 8 * i + fr]; }
#pragma unroll
      for (int j = 0; j < 2; ++j) { bz[j] = sZb[ks + fk][wn + 8 * j + fr]; by[j] = sYb[ks + fk][wn + 8 * j + fr]; }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        dmma16(c1[0][j], c1[1][j], az, bz[j]);
        dmma16(c2[0][j], c2[1][j], az, by[j]);
        dmma16(c2[0][j], c2[1][j], ay, bz[j]);
      }
    }
    if (diag) {
#pragma unroll
      for (int q = 0; q < 4; ++q) bzs += sZa[4 * warp + q][lane] * sU[4 * warp + q];
    }
    __syncthreads();
  }
  if (diag) {
    sBz[warp][lane] = bzs;
    __syncthreads();
    if (warp == 0 && ta * GT + lane < c) A.bzp[(size_t)split * c + ta * GT + lane] = (sBz[0][lane] + sBz[1][lane]) + (sBz[2][lane] + sBz[3][lane]);
  }
  double* o1 = A.G1p + (size_t)split * c * c;
  double* o2 = A.G2p + (size_t)split * c * c;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int ra = ta * GT + wm + 8 * i + fr, cb = tb * GT + wn + 8 * j + 2 * fk + q;
        if (ra < c && cb < c) { o1[(size_t)ra * c + cb] = c1[i][j][q]; o2[(size_t)ra * c + cb] = c2[i][j][q]; }
      }
}

// Block-diagonal terms, one CTA per clone: D1 = sum X^T X, D2 = sum X^T D X (6x6), b = sum X^T r (6),
// over the accepted tracks' observations of that clone.  Deterministic (fixed feature->thread map, tree reduce).
template <class S>
__global__ void __launch_bounds__(128) k_blockdiag(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int clone = blockIdx.x;
  if (clone >= A.M || A.n_tracks == 0) return;
  const int N = A.n_tracks;
  const int* __restrict__ obs_off = A.obs_off;
  const int* __restrict__ clone_idx = A.clone_idx;
  const int* __restrict__ accept = A.accept;
  const S* __restrict__ Xg = A.Xg;
  const S* __restrict__ rg = A.rg;
  const double du = (double)A.st->u_var, dv = (double)A.st->v_var;
  double* __restrict__ D1 = A.D1;
  double* __restrict__ D2 = A.D2;
  double* __restrict__ bb = A.bb;
  double acc[78];
#pragma unroll
  for (int k = 0; k < 78; ++k) acc[k] = 0.0;
  for (int j = threadIdx.x; j < N; j += 128) {
    if (!accept[j]) continue;
    const int o0 = obs_off[j], o1 = obs_off[j + 1];
    for (int o = o0; o < o1; ++o) {
      if (clone_idx[o] != clone) continue;
      double x0[6], x1[6];
#pragma unroll
      for (int b = 0; b < 6; ++b) { x0[b] = (double)Xg[12 * (size_t)o + b]; x1[b] = (double)Xg[12 * (size_t)o + 6 + b]; }
      const double r0 = (double)rg[2 * (size_t)o], r1 = (double)rg[2 * (size_t)o + 1];
#pragma unroll
      for (int p = 0; p < 6; ++p) {
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          acc[6 * p + q] += x0[p] * x0[q] + x1[p] * x1[q];
          acc[36 + 6 * p + q] += du * x0[p] * x0[q] + dv * x1[p] * x1[q];
        }
        acc[72 + p] += x0[p] * r0 + x1[p] * r1;
      }
    }
  }
  __shared__ double red[4][78];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 78; ++k) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 78) {
    const int k = threadIdx.x;
    const double v = (red[0][k] + red[1][k]) + (red[2][k] + red[3][k]);
    if (k < 36) D1[36 * (size_t)clone + k] = v;
    else if (k < 72) D2[36 * (size_t)clone + (k - 36)] = v;
    else bb[6 * (size_t)clone + (k - 72)] = v;
  }
}

// Assemble T'' (n x n), r'' (n), R'' (n x n) except the <=15 head rows (k_rows fills those beside this kernel).
// Grid: GT / kAsmRows CTAs per upper 32-tile pair (ta <= tb) of the c x c Gram block, each kAsmRows rows of the tile, then one
// border CTA (the T'' columns < 15 and r'').  A tile CTA issues the 2 nsplit coalesced row loads of its partials before summing
// them, in split order from 0.0, and writes its rows of the tile and, for ta < tb, the matching columns of the mirror tile
// through a shared-memory transpose, so that both stores are coalesced.  The mirror takes the same partial sums and its own
// block-diagonal term.  A diagonal 32-tile is read in both halves (the Gram kernels write both; G2's (i, j) and (j, i) add
// Z^T Yq and Yq^T Z in opposite order and need not agree bit for bit).
// When m <= n (plain uncompressed update) every CTA of the grid zeroes its share of the rows >= m.
constexpr int kAsmThreads = 256;
// rows of a tile per CTA: 15.3 us at a batch of 8 config-B filters, 8.5 us for one (8 rows: 16.8 / 7.6 us; 32 rows: 14.5 /
// 10.5 us; H100 80GB HBM3, 700 W)
constexpr int kAsmRows = 16;
__host__ __device__ inline int asm_ctas(int c) {
  const int ntile = (c + GT - 1) / GT;
  return ntile * (ntile + 1) / 2 * (GT / kAsmRows) + 1;
}
template <class S>
__global__ void __launch_bounds__(kAsmThreads) k_assemble(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  if (A.n_tracks == 0) return;
  const int n = A.n, ld = A.ld, nsplit = A.nsplit;
  const double* __restrict__ D1 = A.D1;
  const double* __restrict__ D2 = A.D2;
  double* __restrict__ T2 = A.T2;
  double* __restrict__ R2 = A.R2;
  double* __restrict__ r2 = A.r2;
  const int c = n - kImuDim;
  const int m = *A.m_out;
  const int tid = threadIdx.x;
  // The explicit head rows belong to k_rows, which runs BESIDE this kernel (side branch of the graph): rows < hcap of T'', R''
  // and r'', and -- when compressing -- columns < 15 of R'' (the coupling R_hH^T), are neither read nor written here.
  if (m <= n) {  // every stacked row explicit (k_rows), no Gram part: rows >= m are zero
    const size_t total = (size_t)(n - m) * n;
    for (size_t e = (size_t)blockIdx.x * kAsmThreads + tid; e < total; e += (size_t)gridDim.x * kAsmThreads) {
      const int a = m + (int)(e / n), b = (int)(e % n);
      T2[(size_t)a * ld + b] = 0.0;
      R2[(size_t)a * ld + b] = 0.0;
    }
    for (int a = m + blockIdx.x * kAsmThreads + tid; a < n; a += gridDim.x * kAsmThreads) r2[a] = 0.0;
    return;
  }
  constexpr int kParts = GT / kAsmRows;
  const int ntile = (c + GT - 1) / GT, nwork = ntile * (ntile + 1) / 2 * kParts;
  if ((int)blockIdx.x > nwork) return;
  if ((int)blockIdx.x == nwork) {  // border: T'' columns < 15 of rows >= 15, and beta = blk(sum X^T r) - Z^T (U^T r)
    for (int e = tid; e < c * kImuDim; e += kAsmThreads) T2[(size_t)(kImuDim + e / kImuDim) * ld + e % kImuDim] = 0.0;
    // Z^T (U^T r) arrives as split-K partials from the Gram kernels' diagonal tiles
    const double* __restrict__ bzp = A.bzp;
    for (int ac = tid; ac < c; ac += kAsmThreads) {
      double t = 0.0;
      for (int s = 0; s < nsplit; ++s) t += bzp[(size_t)s * c + ac];
      r2[kImuDim + ac] = A.bb[ac] - t;
    }
    return;
  }
  int pidx = blockIdx.x / kParts, ta = 0;
  while (pidx >= ntile - ta) { pidx -= ntile - ta; ++ta; }
  const int tb = ta + pidx, r0 = (blockIdx.x % kParts) * kAsmRows;
  __shared__ double sT[GT][kAsmRows + 1], sR[GT][kAsmRows + 1];  // this CTA's columns of the mirror tile
  const int tx = tid & 31, ty = tid >> 5;
  const int bc = tb * GT + tx;
  const size_t cc = (size_t)c * c;
#pragma unroll 1
  for (int r = ty; r < kAsmRows; r += kAsmThreads / GT) {
    const int ac = ta * GT + r0 + r;
    if (ac < c && bc < c) {
      const double* __restrict__ p1 = A.G1p + (size_t)ac * c + bc;
      const double* __restrict__ p2 = A.G2p + (size_t)ac * c + bc;
      double v1[kMaxSplit], v2[kMaxSplit];
#pragma unroll
      for (int s = 0; s < kMaxSplit; ++s)
        if (s < nsplit) { v1[s] = p1[s * cc]; v2[s] = p2[s * cc]; }
      double g1 = 0.0, g2 = 0.0;
#pragma unroll
      for (int s = 0; s < kMaxSplit; ++s)
        if (s < nsplit) { g1 += v1[s]; g2 += v2[s]; }
      const bool blk = ac / 6 == bc / 6;
      const size_t d = 36 * (size_t)(ac / 6), dab = d + 6 * (ac % 6) + (bc % 6), dba = d + 6 * (bc % 6) + (ac % 6);
      T2[(size_t)(kImuDim + ac) * ld + kImuDim + bc] = (blk ? D1[dab] : 0.0) - g1;
      R2[(size_t)(kImuDim + ac) * ld + kImuDim + bc] = (blk ? D2[dab] : 0.0) - g2;
      if (ta < tb) { sT[tx][r] = (blk ? D1[dba] : 0.0) - g1; sR[tx][r] = (blk ? D2[dba] : 0.0) - g2; }
    }
  }
  if (ta == tb) return;
  __syncthreads();
  for (int e = tid; e < GT * kAsmRows; e += kAsmThreads) {
    const int mr = tb * GT + e / kAsmRows, mc = ta * GT + r0 + e % kAsmRows;
    if (mr < c && mc < c) {
      T2[(size_t)(kImuDim + mr) * ld + kImuDim + mc] = sT[e / kAsmRows][e % kAsmRows];
      R2[(size_t)(kImuDim + mr) * ld + kImuDim + mc] = sR[e / kAsmRows][e % kAsmRows];
    }
  }
}

// Explicit stacked rows ("head rows"), one CTA per feature.
//  * m > n : the reference's QR leaves stacked rows 0..14 untouched (15 zero leading columns of H_o,
//            msckf.h:1343-1363); they enter the compressed system as themselves.  hcap = 15.
//  * m <= n: the reference's Q is square, i.e. the update is the plain uncompressed EKF update in the full
//            measurement space (orthogonal invariance) -- every stacked row is explicit, hcap = m, and the
//            Gram part is switched off (k_assemble).
// Row t of feature j is A_j(:,t)^T [X_j | r_j] with A_j(:,t) = Q e_{3+t},  Q = H0 H1 H2 = I - V T V^T (compact WY,
// exact reflectors tau_k = 2 / v_k^T v_k in fp64): every entry of Q costs O(1) from V (2L x 3) and T (3 x 3).
constexpr int kRowsFixed = 6 + 9 + 9 + 3 + 3 * kImuDim;  // s_g | s_T | s_Wd | s_s | s_adu
__host__ __device__ inline size_t rows_smem_doubles(int Lmax) { return (size_t)kRowsFixed + 12 * (size_t)Lmax; }
// is track j a head track of this update (explicit rows)?  uniform per CTA
template <class S>
__device__ __forceinline__ bool rows_is_head(const UpdArgs<S>& A, int j) {
  if (j >= A.n_tracks || !A.accept[j]) return false;
  const int m = *A.m_out;
  return A.row_off[j] < ((m <= A.n) ? m : kImuDim);
}
template <class S>
__device__ __forceinline__ void rows_work(const UpdArgs<S>& A, int j, double* __restrict__ smem) {
  const int nthr = blockDim.x;
  double* s_g = smem;
  double* s_T = s_g + 6;
  double* s_Wd = s_T + 9;
  double* s_s = s_Wd + 9;
  double (*s_adu)[3] = reinterpret_cast<double (*)[3]>(s_s + 3);
  double* sh = smem + kRowsFixed;  // V[2L][3] | W[2L][3]
  if (j >= A.n_tracks) return;
  const int n = A.n, ld = A.ld;
  const int* __restrict__ obs_off = A.obs_off;
  const int* __restrict__ clone_idx = A.clone_idx;
  const int* __restrict__ accept = A.accept;
  const int* __restrict__ row_off = A.row_off;
  const int* __restrict__ m_in = A.m_out;
  const S* __restrict__ Xg = A.Xg;
  const S* __restrict__ rg = A.rg;
  const S* __restrict__ Vg = A.Vg;
  const S* __restrict__ taug = A.taug;
  const double* __restrict__ Z = A.Z;
  const double du = (double)A.st->u_var, dv = (double)A.st->v_var;
  double* __restrict__ T2 = A.T2;
  double* __restrict__ R2 = A.R2;
  double* __restrict__ r2 = A.r2;
  if (!accept[j]) return;
  const int m = *m_in;
  const bool full = m <= n;
  const int hcap = full ? m : kImuDim;
  const int h0 = row_off[j];
  if (h0 >= hcap) return;
  const int c = n - kImuDim;
  const int o0 = obs_off[j], L = obs_off[j + 1] - o0, L2 = 2 * L;
  const int nh = min(L2 - 3, hcap - h0);
  const int tid = threadIdx.x;
  double* V = sh;
  double* W = sh + 3 * L2;
  for (int e = tid; e < 3 * L2; e += nthr) V[e] = (double)Vg[3 * 2 * (size_t)o0 + e];
  // this feature owns rows h0 .. h0+nh-1 of T'', R'' (and, when compressing, the same columns of R'' below row 15): clear them,
  // then fill in what is not zero -- k_assemble leaves them alone, so the two kernels run side by side
  for (int e = tid; e < nh * n; e += nthr) {
    const int t = e / n, b = e % n;
    T2[(size_t)(h0 + t) * ld + b] = 0.0;
    R2[(size_t)(h0 + t) * ld + b] = 0.0;
    if (!full && b >= kImuDim) R2[(size_t)b * ld + (h0 + t)] = 0.0;
  }
  __syncthreads();
  if (tid < 6) {  // v_k^T v_l : (0,0) (1,1) (2,2) (0,1) (0,2) (1,2)
    const int ka[6] = {0, 1, 2, 0, 0, 1}, kb[6] = {0, 1, 2, 1, 2, 2};
    double s = 0.0;
    for (int a = 0; a < L2; ++a) s += V[3 * a + ka[tid]] * V[3 * a + kb[tid]];
    s_g[tid] = s;
  }
  __syncthreads();
  if (tid == 0) {
    double tau[3];
    for (int k = 0; k < 3; ++k) tau[k] = ((double)taug[3 * j + k] != 0.0) ? 2.0 / s_g[k] : 0.0;
    double T[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    T[0][0] = tau[0]; T[1][1] = tau[1]; T[2][2] = tau[2];
    T[0][1] = -tau[1] * T[0][0] * s_g[3];
    T[0][2] = -tau[2] * (T[0][0] * s_g[4] + T[0][1] * s_g[5]);
    T[1][2] = -tau[2] * T[1][1] * s_g[5];
    for (int k = 0; k < 3; ++k) for (int l = 0; l < 3; ++l) s_T[3 * k + l] = T[k][l];
  }
  __syncthreads();
  for (int a = tid; a < L2; a += nthr)
    for (int l = 0; l < 3; ++l) W[3 * a + l] = V[3 * a] * s_T[l] + V[3 * a + 1] * s_T[3 + l] + V[3 * a + 2] * s_T[6 + l];
  __syncthreads();
  if (tid < 9) {  // Wd = sum_a d_a w_a^T w_a
    const int k = tid / 3, l = tid % 3;
    double s = 0.0;
    for (int a = 0; a < L2; ++a) s += ((a & 1) ? dv : du) * W[3 * a + k] * W[3 * a + l];
    s_Wd[tid] = s;
  } else if (tid < 12) {  // s = sum_a r_a w_a
    const int l = tid - 9;
    double s = 0.0;
    for (int a = 0; a < L2; ++a) s += (double)rg[2 * (size_t)o0 + a] * W[3 * a + l];
    s_s[l] = s;
  }
  __syncthreads();
  // Q^T D Q entry for columns b, b2 of Q
  auto qdq = [&](int b, int b2) {
    const double db = (b & 1) ? dv : du, db2 = (b2 & 1) ? dv : du;
    const double wb_vb2 = W[3 * b] * V[3 * b2] + W[3 * b + 1] * V[3 * b2 + 1] + W[3 * b + 2] * V[3 * b2 + 2];
    const double wb2_vb = W[3 * b2] * V[3 * b] + W[3 * b2 + 1] * V[3 * b + 1] + W[3 * b2 + 2] * V[3 * b + 2];
    double quad = 0.0;
    for (int k = 0; k < 3; ++k)
      for (int l = 0; l < 3; ++l) quad += V[3 * b + k] * s_Wd[3 * k + l] * V[3 * b2 + l];
    return ((b == b2) ? db : 0.0) - db * wb_vb2 - db2 * wb2_vb + quad;
  };
  auto qent = [&](int a, int b) {  // Q[a][b]
    return ((a == b) ? 1.0 : 0.0) - (W[3 * a] * V[3 * b] + W[3 * a + 1] * V[3 * b + 1] + W[3 * a + 2] * V[3 * b + 2]);
  };
  // r rows and the R_o block of this feature restricted to the explicit rows
  for (int e = tid; e < nh * (nh + 1); e += nthr) {
    const int t = e / (nh + 1), u = e % (nh + 1);
    const int b = 3 + t;
    if (u == nh) {
      r2[h0 + t] = (double)rg[2 * (size_t)o0 + b] - (s_s[0] * V[3 * b] + s_s[1] * V[3 * b + 1] + s_s[2] * V[3 * b + 2]);
    } else {
      R2[(size_t)(h0 + t) * ld + (h0 + u)] = qdq(b, 3 + u);
    }
  }
  if (!full && tid < nh * 3) s_adu[tid / 3][tid % 3] = qdq(3 + tid / 3, tid % 3);  // A_h^T D U
  __syncthreads();
  // H rows (and, when compressing, the coupling rows R_hH = A_h^T D Pi_j X_j)
  for (int e = tid; e < nh * L * 6; e += nthr) {
    const int t = e / (L * 6), rem = e % (L * 6), i = rem / 6, bb = rem % 6;
    const int b = 3 + t;
    const int col = 6 * clone_idx[o0 + i] + bb;
    const double x0 = (double)Xg[12 * (size_t)(o0 + i) + bb], x1 = (double)Xg[12 * (size_t)(o0 + i) + 6 + bb];
    const double q0 = qent(2 * i, b), q1 = qent(2 * i + 1, b);
    T2[(size_t)(h0 + t) * ld + kImuDim + col] = q0 * x0 + q1 * x1;
    if (!full) {
      double rv = du * q0 * x0 + dv * q1 * x1;
      for (int q = 0; q < 3; ++q) rv -= s_adu[t][q] * Z[(size_t)(3 * j + q) * c + col];
      R2[(size_t)(h0 + t) * ld + kImuDim + col] = rv;
      R2[(size_t)(kImuDim + col) * ld + (h0 + t)] = rv;
    }
  }
}
template <class S>
__global__ void __launch_bounds__(128) k_rows(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  extern __shared__ double rows_sm[];
  rows_work(args[blockIdx.z], blockIdx.x, rows_sm);
}

}  // namespace mb
