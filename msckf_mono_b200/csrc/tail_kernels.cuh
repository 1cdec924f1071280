// msckf_mono_b200/csrc/tail_kernels.cuh
// Dense n x n tail of the EKF update (msckf.h:1369-1418) in square-root form, fp64 throughout:
//   TP  = T'' P                      S'' = TP T''^T + R''          (k_gemm_tp, k_gemm_s: this file, all SMs)
//   S'' = L L^T over the independent rows, W = L^-1 [TP | r''], P+ = P - W^T W (== Joseph form for the optimal
//   gain of the projected system), dx = W^T (L^-1 r''), state injection       (k_tail: tail_cluster.cuh, one cluster)
#pragma once
#include "common.cuh"

namespace mb {

// One 32 x 32 output tile C[a][b] = sum_k A(k, a) B(k, b) per CTA of 256 threads: four groups of 64 threads (4 x 4 register
// tile per thread) split every 32-deep k-slab between them (8 k each, one fp64 FMA chain per output and group) and are
// summed once at the end through shared memory in a fixed order (deterministic; the same kernel serves one filter and a
// batch).  Operands stream through double-buffered shared memory (one barrier per slab) with the next slab prefetched into
// registers while the current one is multiplied; the ragged last slab is zero-padded.
// The summation order is part of the results: the rank decision keeps or drops an index of S'' on the sign of its pivot,
// and at config B some of those pivots are rounding noise.  An FP64 tensor-core form of this tile (mma.sync m8n8k4, one
// chain of DMMA per output) was 3-4x further from a long-double reference than these four FMA chains, changed the rank of
// 2 of 8 filters of the benchmark's batch and moved two fp64 parity cases past their bounds (DESIGN.md 4.5).
// Each operand is fetched along its memory layout, chosen by its template flag, so that a warp's global load reads 32
// consecutive elements:
//   KA / KB = false: stored along the output index (P[k][b], W[k][a]): consecutive threads take consecutive output indices;
//   KA / KB = true:  stored along k (T''[a][k], TP[a][k]): consecutive threads take consecutive k, and the slab is transposed
//                    on its way into shared memory.
// Slabs are staged k-major, s[k][i], with a row stride of 34 doubles: the transposing stores (32 lanes, 32 rows) hit 8 bank
// pairs per half warp instead of one, and the 16-byte fragment reads stay aligned.
// LA(k, a) / LB(k, b) fetch operand elements, EPI(a, b, acc) stores.
constexpr int kGemmThreads = 256;
constexpr int kGemmMinBlocks = 3;  // 3 CTAs per SM: a batch of 8 config-B filters (392 tiles of T''P) runs in one wave
constexpr int kGemmLd = 34;
constexpr int kGemmSlab = 32 * kGemmLd;  // doubles of one staged 32-deep operand slab
template <bool KA, bool KB, class LoadA, class LoadB, class Epi>
__device__ __forceinline__ void gemm_tile32(int n, int k_begin, int a0, int b0, LoadA LA, LoadB LB, Epi EPI) {
  constexpr int kParts = kGemmThreads / 64, kPer = 32 / kParts, kFetch = 1024 / kGemmThreads;
  static_assert((kParts - 1) * 1024 <= 4 * kGemmSlab, "the partial sums reuse the slab buffers");
  __shared__ __align__(16) double sm[4 * kGemmSlab];  // [2 stages][A | B] slabs; after the loop: the partial sums of 3 k-groups
  const int tid = threadIdx.x;
  const int part = tid >> 6, t = tid & 63;
  const int tx = t & 7, ty = t >> 3;
  // element e of a slab -> (k, i) of the operand
  auto ek = [](bool along_k, int e) { return along_k ? (e & 31) : (e >> 5); };
  auto ei = [](bool along_k, int e) { return along_k ? (e >> 5) : (e & 31); };
  double acc[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
  double pa[kFetch], pb[kFetch];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int u = 0; u < kFetch; ++u) {
      const int e = tid + kGemmThreads * u;
      const int ka = k0 + ek(KA, e), ia = a0 + ei(KA, e), kb = k0 + ek(KB, e), ib = b0 + ei(KB, e);
      pa[u] = (ka < n && ia < n) ? LA(ka, ia) : 0.0;
      pb[u] = (kb < n && ib < n) ? LB(kb, ib) : 0.0;
    }
  };
  const int nslab = (n - k_begin + 31) / 32;
  if (nslab > 0) fetch(k_begin);
  for (int s = 0; s < nslab; ++s) {
    // stage s & 1 was last read in slab s - 2, and every thread passed slab s - 1's barrier after that
    double* __restrict__ sA = sm + (s & 1) * 2 * kGemmSlab;
    double* __restrict__ sB = sA + kGemmSlab;
#pragma unroll
    for (int u = 0; u < kFetch; ++u) {
      const int e = tid + kGemmThreads * u;
      sA[ek(KA, e) * kGemmLd + ei(KA, e)] = pa[u];
      sB[ek(KB, e) * kGemmLd + ei(KB, e)] = pb[u];
    }
    __syncthreads();
    if (s + 1 < nslab) fetch(k_begin + 32 * (s + 1));
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int kk = kPer * part + q;
      const double2 a01 = *reinterpret_cast<const double2*>(&sA[kk * kGemmLd + 4 * ty]), a23 = *reinterpret_cast<const double2*>(&sA[kk * kGemmLd + 4 * ty + 2]);
      const double2 b01 = *reinterpret_cast<const double2*>(&sB[kk * kGemmLd + 4 * tx]), b23 = *reinterpret_cast<const double2*>(&sB[kk * kGemmLd + 4 * tx + 2]);
      const double a[4] = {a01.x, a01.y, a23.x, a23.y}, b[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) acc[p][qq] += a[p] * b[qq];
    }
  }
  double (*red)[16][64] = reinterpret_cast<double (*)[16][64]>(sm);
  __syncthreads();  // the last slab is read by everybody before its buffer takes the partial sums
  if (part > 0) {
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int q = 0; q < 4; ++q) red[part - 1][4 * p + q][t] = acc[p][q];
  }
  __syncthreads();
  if (part == 0) {
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int a = a0 + 4 * ty + p, b = b0 + 4 * tx + q;
        double v = acc[p][q];
#pragma unroll
        for (int r = 0; r < kParts - 1; ++r) v += red[r][4 * p + q][t];
        if (a < n && b < n) EPI(a, b, v);
      }
  }
}

// TP[a][b] = sum_k T2[a][k] * P[k][b]      (T2 columns < 15 are zero)
template <class S>
__global__ void __launch_bounds__(kGemmThreads, kGemmMinBlocks) k_gemm_tp(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int n = A.n, ld = A.ld, ldp = A.ldp;
  if ((int)blockIdx.x * 32 >= n || (int)blockIdx.y * 32 >= n || A.n_tracks == 0) return;
  const double* __restrict__ T2 = A.T2;
  const S* __restrict__ P = A.P;
  double* __restrict__ TP = A.TP;
  gemm_tile32<true, false>(n, kImuDim, blockIdx.y * 32, blockIdx.x * 32,
                           [&](int k, int a) { return T2[(size_t)a * ld + k]; },
                           [&](int k, int b) { return (double)P[(size_t)k * ldp + b]; },
                           [&](int a, int b, double v) { TP[(size_t)a * ld + b] = v; });
}

// S2[a][b] = sum_k TP[a][k] * T2[b][k] + R2[a][b] for b <= a: only the lower tile pairs (ta >= tb) run, and the diagonal
// tiles are written in full.  Both tail kernels read S'' from its lower triangle only (common.cuh, UpdArgs::S2).
template <class S>
__global__ void __launch_bounds__(kGemmThreads, kGemmMinBlocks) k_gemm_s(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int n = A.n, ld = A.ld;
  const int nt32 = (n + 31) / 32;
  if ((int)blockIdx.x >= nt32 * (nt32 + 1) / 2 || A.n_tracks == 0) return;
  int pidx = blockIdx.x, ta = 0;
  while (pidx >= ta + 1) { pidx -= ta + 1; ++ta; }  // (ta >= tb)
  const int tb = pidx;
  const double* __restrict__ TP = A.TP;
  const double* __restrict__ T2 = A.T2;
  const double* __restrict__ R2 = A.R2;
  double* __restrict__ S2 = A.S2;
  gemm_tile32<true, true>(n, kImuDim, ta * 32, tb * 32,  // T2 columns < 15 are zero
                          [&](int k, int a) { return TP[(size_t)a * ld + k]; },
                          [&](int k, int b) { return T2[(size_t)b * ld + k]; },
                          [&](int a, int b, double v) { S2[(size_t)a * ld + b] = v + R2[(size_t)a * ld + b]; });
}

// P <- P - W^T W (lower-triangular tile pairs; written in the filter precision, exactly symmetric by construction), and in
// the same launch  dx = W^T y  (the CTAs of the first tile column each take 32 components) followed by the state injection of
// msckf.h:1373-1391 by whichever CTA finishes last (ticket counter) -- round 1 ran both as a separate single-CTA kernel
// (k_inject: a whole launch for a 195 x 195 mat-vec).
template <class S>
__global__ void __launch_bounds__(kGemmThreads, kGemmMinBlocks) k_syrk(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& A = args[blockIdx.z];
  const int n = A.n, ld = A.ld, ldp = A.ldp;
  const int nt32 = (n + 31) / 32;
  if ((int)blockIdx.x >= nt32 * (nt32 + 1) / 2 || A.n_tracks == 0) return;
  const double* __restrict__ Wm = A.W;
  S* __restrict__ P = A.P;
  if (*A.m_out == 0) return;  // nothing accepted: the reference returns before touching the state (msckf.h:401-403, :1328)
  int pidx = blockIdx.x, ta = 0;
  while (pidx >= ta + 1) { pidx -= ta + 1; ++ta; }  // (ta >= tb)
  const int tb = pidx;
  gemm_tile32<false, false>(n, 0, ta * 32, tb * 32,
                            [&](int k, int a) { return Wm[(size_t)k * ld + a]; },
                            [&](int k, int b) { return Wm[(size_t)k * ld + b]; },
                            [&](int a, int b, double v) {
                              if (b <= a) {
                                const S r = (S)((double)P[(size_t)a * ldp + b] - v);
                                if (!isfinite((double)r)) A.m_out[2] = 1;  // MSCKF_B200_ERR_NUMERIC (benign race: every writer stores 1)
                                P[(size_t)a * ldp + b] = r;
                                P[(size_t)b * ldp + a] = r;
                              }
                            });
  const int tid = threadIdx.x;
  __shared__ double part[kGemmThreads / 32][33];
  __shared__ int s_last;
  if (tb == 0) {  // dx[a] = sum_k W[k][a] y[k] for the 32 components of this tile row
    const int al = tid & 31, kg = tid >> 5, a = ta * 32 + al;
    const double* __restrict__ yv = A.y;
    double s = 0.0;
    if (a < n)
      for (int k = kg; k < n; k += kGemmThreads / 32) s += Wm[(size_t)k * ld + a] * yv[k];
    part[kg][al] = s;
    __syncthreads();
    if (kg == 0 && a < n) {
      double t = 0.0;
#pragma unroll
      for (int g = 0; g < kGemmThreads / 32; ++g) t += part[g][al];
      A.dx[a] = t;
    }
  }
  // ---- the last CTA injects the correction (msckf.h:1373-1391)
  __syncthreads();
  if (tid == 0) { __threadfence(); s_last = (atomicAdd(A.done, 1u) == (unsigned)(nt32 * (nt32 + 1) / 2) - 1u) ? 1 : 0; }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  DevState<S>* st = A.st;
  S* __restrict__ poses = A.poses;
  const double* dx = A.dx;
  if (tid == 0) {
    *A.done = 0u;
    const S dth[3] = {(S)__ldcg(dx + 0), (S)__ldcg(dx + 1), (S)__ldcg(dx + 2)};
    S uq[4], qn[4];
    build_update_quat(dth, uq);
    quat_mul(uq, st->q_IG, qn);  // not renormalised (msckf.h:1376-1378)
    for (int i = 0; i < 4; ++i) st->q_IG[i] = qn[i];
    for (int i = 0; i < 3; ++i) {
      st->b_g[i] += (S)__ldcg(dx + 3 + i);
      st->v_I_G[i] += (S)__ldcg(dx + 6 + i);
      st->b_a[i] += (S)__ldcg(dx + 9 + i);
      st->p_I_G[i] += (S)__ldcg(dx + 12 + i);
    }
    st->n_updates += 1;
    st->last_m = A.m_out[0];
    st->last_rank = *A.rank_out;
  }
  double nn = 0.0;
  for (int a = tid; a < n; a += kGemmThreads) { const double v = __ldcg(dx + a); nn += v * v; }
  nn = warp_sum(nn);
  __syncthreads();
  if ((tid & 31) == 0) part[0][tid >> 5] = nn;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int w = 0; w < kGemmThreads / 32; ++w) t += part[0][w];
    st->last_dx_norm = sqrt(t);
    if (!isfinite(t)) A.m_out[2] = 1;  // non-finite delta-x
    st->last_status = A.m_out[2];
  }
  for (int ci = tid; ci < A.M; ci += kGemmThreads) {
    S* ps = poses + kPoseStride * ci;
    const S dth[3] = {(S)__ldcg(dx + 15 + 6 * ci), (S)__ldcg(dx + 16 + 6 * ci), (S)__ldcg(dx + 17 + 6 * ci)};
    S uq[4], qn[4];
    build_update_quat(dth, uq);
    quat_mul(uq, ps, qn);
    quat_normalize(qn);
    ps[0] = qn[0]; ps[1] = qn[1]; ps[2] = qn[2]; ps[3] = qn[3];
    ps[4] += (S)__ldcg(dx + 18 + 6 * ci); ps[5] += (S)__ldcg(dx + 19 + 6 * ci); ps[6] += (S)__ldcg(dx + 20 + 6 * ci);
  }
}

}  // namespace mb
