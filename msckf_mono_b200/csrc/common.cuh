// msckf_mono_b200/csrc/common.cuh -- device helpers shared by all kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cmath>

namespace mb {

constexpr int kImuDim = 15;
constexpr int kPoseStride = 8;  // q(x,y,z,w), p(x,y,z), pad  -> 32 B (fp32) / 64 B (fp64): TMA friendly

// Device-resident filter state that is not a matrix (mirrors types.h:70-77 imuState + camera/noise/params).
template <class S>
struct DevState {
  S q_IG[4], b_g[3], v_I_G[3], b_a[3], p_I_G[3], g[3];
  S q_IG_null[4], v_I_G_null[3], p_I_G_null[3];
  S q_CI[4], p_C_I[3];
  S u_var, v_var;
  S max_gn_cost_norm, translation_threshold;
  S Q_imu[144];
  S chi2[99];
  unsigned long long num_residualized;  // msckf.h:42 num_feature_tracks_residualized_
  unsigned long long pfg_shifted, pfg_oob, n_updates;
  int last_m, last_rank, last_status, pad_;
  double last_dx_norm;
};

// Everything one measurement update of one filter needs on the device: sizes, the packed input / report blocks, the
// filter's resident state and its workspaces.  One UpdArgs per filter lives at the head of the packed input block
// (engine.cu), so that a kernel launch only carries a pointer to an ARRAY of them and the filter index in blockIdx.z:
// the same launch (and the same captured CUDA graph) serves one filter or a whole batch of independent filters, and
// buffer swaps (prune) or re-allocations never invalidate a captured graph.
template <class S>
struct UpdArgs {
  int n_tracks, M, Lmax, ldp;
  int ld, n, mode, gram_mma; // gram_mma: this filter's Gram products run on the FP64 tensor-core kernel (else the SIMT tile kernel)
  int K, nsplit, kchunk, tail_kind;
  double rank_thr;
  // packed input block
  const int* obs_off;    // [N+1]
  const S* obs;          // [sumL*2] normalised image coordinates
  const int* clone_idx;  // [sumL] positional index of the observing clone
  const S* pfg_given;    // optional [N*3]: residualize tracks at given positions (pruneRedundantStates)
  // resident filter state
  S* poses;              // [M*8] current clone poses (q xyzw, p, pad)
  S* P;                  // [n x n], leading dim ldp
  DevState<S>* st;
  // packed report block
  int* m_out;            // total number of stacked rows m
  int* rank_out;
  int* cm_eff;           // [N] "not rejected by checkMotion" (msckf.h:354) as reported to the host
  int* cm_ok;            // [N] checkMotion result
  int* tri_ok;           // [N] initializePosition validity
  int* valid;            // [N]
  int* accept;           // [N]
  S* pfg;                // [N*3]
  S* gamma;              // [N]
  // workspaces
  unsigned long long* counter_snap;  // num_feature_tracks_residualized_ before this batch (read by k_jac)
  int* src;              // [N] index of the track whose p_f_G loop B uses (msckf.h:419)
  int* rows;             // [N] rho_j = 2L-3
  int* row_off;          // [N+1] ordered stacking (msckf.h:433-445)
  unsigned* done;        // CTA ticket counter of k_jac (zero between launches)
  S* Xg;                 // [sumL*12] H_x blocks (2x6 per observation)
  S* rg;                 // [sumL*2]  residuals
  S* Vg;                 // [sumL*2*3] Householder vectors of the null-space projection
  S* taug;               // [N*3]
  double* Z;             // [3N x c]  U_j^T X_j scattered to clone columns
  double* Yq;            // [3N x c]  U_j^T D X_j - 1/2 (U_j^T D U_j) Z_j
  double* ur;            // [3N]      U_j^T r_j
  double *G1p, *G2p;     // split-K partials of the Gram products
  double* bzp;           // split-K partials of Z^T (U^T r)  [nsplit][c], written by the diagonal tiles of the Gram kernel
  double *D1, *D2, *bb;  // per-clone 6x6 sums
  // S2 (S'' = TP T''^T + R''): only its lower triangle, diagonal included, is defined -- k_gemm_s writes the lower 32 x 32
  // tile pairs only, and both tail kernels (k_tail_fused, k_tail) read nothing above the diagonal
  double *T2, *R2, *r2, *TP, *S2, *W, *G, *y, *dx, *idiag;
  double* pivr;          // [n] diagnostics: Gamma's pivot / its original diagonal at the moment of the keep / drop decision
  int* keep;
  unsigned long long* prof;  // optional: %globaltimer stamps (profiling aid)
};

// Programmatic dependent launch (sm_90+): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// start while its predecessor in the stream is still running; pdl_wait() blocks until the predecessor grid has completed
// and its writes are visible.  EVERY kernel of the update calls it first, in every CTA, before any early return -- a grid
// that finished without waiting would release ITS dependent too early.  pdl_launch() lets the next kernel's CTAs be
// scheduled (they park in their own pdl_wait()).  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// %globaltimer (ns): the clock of the optional phase stamps (UpdArgs::prof, PropBatch::prof)
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t) : : "memory");
  return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) { return __reduce_add_sync(0xffffffffu, v); }  // (REDUX)
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// out-of-line versions for code that runs once per CTA in a single warp (k_jac's QR section has ~40 reductions: inlined,
// the shuffle sequences alone are 2400 instructions, and that section is bound by instruction fetch)
__device__ __noinline__ float warp_sum_call(float v) { return warp_sum(v); }
__device__ __noinline__ double warp_sum_call(double v) { return warp_sum(v); }
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <class S> __device__ __forceinline__ S tsqrt(S x);
template <> __device__ __forceinline__ float tsqrt<float>(float x) { return sqrtf(x); }
template <> __device__ __forceinline__ double tsqrt<double>(double x) { return sqrt(x); }
template <class S> __device__ __forceinline__ S trsqrt(S x);
template <> __device__ __forceinline__ float trsqrt<float>(float x) { return rsqrtf(x); }
template <> __device__ __forceinline__ double trsqrt<double>(double x) { return rsqrt(x); }
template <class S> __device__ __forceinline__ S tabs(S x) { return x < S(0) ? -x : x; }
// 1 / sqrt(p) on a dependent chain: float seed + two Newton steps in fp64 (a dozen instructions instead of the library's ~35)
__device__ __forceinline__ double fast_rsqrt(double p) {
  if (p > 1e-30 && p < 1e30) {
    double y = (double)rsqrtf((float)p);
    const double hp = 0.5 * p;
    y = y * (1.5 - hp * y * y);
    y = y * (1.5 - hp * y * y);
    return y;
  }
  return rsqrt(p);
}
__device__ __forceinline__ float fast_rsqrt(float p) { return rsqrtf(p); }
// tl -> (ti >= tj) of the lower triangle of a tile grid
__device__ __forceinline__ void tri_tile_index(int tl, int& ti, int& tj) {
  ti = (int)((sqrtf(8.0f * (float)tl + 1.0f) - 1.0f) * 0.5f);
  while (ti * (ti + 1) / 2 > tl) --ti;
  while ((ti + 1) * (ti + 2) / 2 <= tl) ++ti;
  tj = tl - ti * (ti + 1) / 2;
}

// Eigen QuaternionBase::toRotationMatrix restated; q = (x,y,z,w); R row-major 3x3.
template <class S>
__device__ __forceinline__ void quat_to_rot(const S* q, S* R) {
  const S x = q[0], y = q[1], z = q[2], w = q[3];
  const S tx = S(2) * x, ty = S(2) * y, tz = S(2) * z;
  const S twx = tx * w, twy = ty * w, twz = tz * w;
  const S txx = tx * x, txy = ty * x, txz = tz * x;
  const S tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = S(1) - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = S(1) - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = S(1) - (txx + tyy);
}
template <class S>
__device__ __forceinline__ void quat_mul(const S* a, const S* b, S* r) {  // Hamilton a*b, (x,y,z,w)
  const S ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  r[0] = aw * bx + ax * bw + ay * bz - az * by;
  r[1] = aw * by + ay * bw + az * bx - ax * bz;
  r[2] = aw * bz + az * bw + ax * by - ay * bx;
  r[3] = aw * bw - ax * bx - ay * by - az * bz;
}
template <class S>
__device__ __forceinline__ void quat_normalize(S* q) {
  const S n = tsqrt<S>(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
// Eigen _transformVector with the inverse quaternion q^-1 = conj(q)/|q|^2
template <class S>
__device__ __forceinline__ void quat_inv_rotate(const S* q, const S* v, S* out) {
  const S n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const S qi[4] = {-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2};
  S uv[3] = {qi[1] * v[2] - qi[2] * v[1], qi[2] * v[0] - qi[0] * v[2], qi[0] * v[1] - qi[1] * v[0]};
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  out[0] = v[0] + qi[3] * uv[0] + (qi[1] * uv[2] - qi[2] * uv[1]);
  out[1] = v[1] + qi[3] * uv[1] + (qi[2] * uv[0] - qi[0] * uv[2]);
  out[2] = v[2] + qi[3] * uv[2] + (qi[0] * uv[1] - qi[1] * uv[0]);
}
// msckf.h:851-872 buildUpdateQuat
template <class S>
__device__ __forceinline__ void build_update_quat(const S* dth, S* u) {
  const S d0 = S(0.5) * dth[0], d1 = S(0.5) * dth[1], d2 = S(0.5) * dth[2];
  const S cs = d0 * d0 + d1 * d1 + d2 * d2;
  u[3] = (cs > S(1)) ? S(1) : tsqrt<S>(S(1) - cs);
  u[0] = -d0; u[1] = -d1; u[2] = -d2;
  quat_normalize(u);
}

// The state injection of msckf.h:1373-1391 for delta-x component i = dx(i) (fp64): q_IG <- buildUpdateQuat(dtheta) * q_IG, not
// renormalised; b_g, v, b_a, p additive; clone k: q <- normalise(buildUpdateQuat(dtheta_k) * q), p additive.  The observability
// copies (*_null) are not touched.  Thread tid of nthr takes the IMU state (tid == 0) and every nthr-th clone.  (k_aid.  k_syrk
// keeps its own inlined copy of the same arithmetic: through this function its SASS is scheduled differently, DESIGN.md 4.8)
template <class S, class DX>
__device__ __forceinline__ void inject_state(DevState<S>* st, S* poses, int M, int tid, int nthr, const DX& dx) {
  if (tid == 0) {
    const S dth[3] = {(S)dx(0), (S)dx(1), (S)dx(2)};
    S uq[4], qn[4];
    build_update_quat(dth, uq);
    quat_mul(uq, st->q_IG, qn);  // not renormalised (msckf.h:1376-1378)
    for (int i = 0; i < 4; ++i) st->q_IG[i] = qn[i];
    for (int i = 0; i < 3; ++i) {
      st->b_g[i] += (S)dx(3 + i);
      st->v_I_G[i] += (S)dx(6 + i);
      st->b_a[i] += (S)dx(9 + i);
      st->p_I_G[i] += (S)dx(12 + i);
    }
  }
  for (int ci = tid; ci < M; ci += nthr) {
    S* ps = poses + kPoseStride * ci;
    const S dth[3] = {(S)dx(15 + 6 * ci), (S)dx(16 + 6 * ci), (S)dx(17 + 6 * ci)};
    S uq[4], qn[4];
    build_update_quat(dth, uq);
    quat_mul(uq, ps, qn);
    quat_normalize(qn);
    ps[0] = qn[0]; ps[1] = qn[1]; ps[2] = qn[2]; ps[3] = qn[3];
    ps[4] += (S)dx(18 + 6 * ci); ps[5] += (S)dx(19 + 6 * ci); ps[6] += (S)dx(20 + 6 * ci);
  }
}

// One warp (lane = row) factors the leading nb x nb block (nb <= 32) of the lower triangle of D in place, D = L L^T.  Returns
// the number of leading pivots that were positive (nb: positive definite); idg[i] = 1 / L[i][i] for those.  (cta_bordered_chol,
// k_aid)
template <int LD>
__device__ __forceinline__ int warp_chol(double (*D)[LD], int nb, double* idg, int lane) {
  int nv = nb;
  for (int j = 0; j < nb; ++j) {
    const double d = D[j][j];
    if (!(d > 0.0)) { nv = j; break; }  // (uniform across the warp: every lane read the same word)
    const double r = sqrt(d);
    __syncwarp();
    if (lane == j) D[j][j] = r;
    if (lane > j && lane < nb) D[lane][j] = D[lane][j] / r;
    __syncwarp();
    if (lane > j && lane < nb) {
      const double lij = D[lane][j];
      for (int c = j + 1; c <= lane; ++c) D[lane][c] -= lij * D[c][j];
    }
    __syncwarp();
  }
  if (lane < nv) idg[lane] = 1.0 / D[lane][lane];
  return nv;
}
// One row against that factor, x <- x L^-T over the first nv columns (lane = column): a forward substitution across the warp
template <int LD>
__device__ __forceinline__ double warp_row_solve(double x, const double (*D)[LD], const double* idg, int nv, int lane) {
  for (int c = 0; c < nv; ++c) {
    const double xc = __shfl_sync(0xffffffffu, x, c) * idg[c];
    if (lane == c) x = xc;
    else if (lane > c) x -= xc * D[lane][c];
  }
  return x;
}

// One 32 x 32 tile product over shared tiles, four outputs per thread of 256 (i = t >> 3):
// s[u] += D[i][p] B[(t & 7) + 8 u][p], p = 0 .. 31 in order.  (cta_bordered_chol's trailing update, k_lmk_downdate)
__device__ __forceinline__ void tile_dot32(const double (*D)[33], const double (*B)[33], int t, double (&s)[4]) {
  const int i = t >> 3;
#pragma unroll 8
  for (int p = 0; p < 32; ++p) {
    const double di = D[i][p];
#pragma unroll
    for (int u = 0; u < 4; ++u) s[u] += di * B[(t & 7) + 8 * u][p];
  }
}

// Blocked right-looking Cholesky (panels of 32, all 256 threads of the CTA) of the leading ncols x ncols block of the row-major
// A (leading dimension ld, lower triangle read), A = L L^T in place, with the rows ncols .. Rt - 1 beneath it solved alongside:
// each ends as x L^-T, x the row as given.  Returns -1, or the first pivot that is not positive (or NaN): at that panel only row
// Rt - 1 is solved, over the good columns before the pivot, and the factor stops.  Ends with the CTA synchronised.  (k_nees,
// k_lmk_gain)
__device__ __forceinline__ int cta_bordered_chol(double* __restrict__ A, int ld, int ncols, int Rt, int t) {
  __shared__ double D[32][33];  // diagonal block, then the row panel of a trailing tile
  __shared__ double B[32][33];  // column panel of a trailing tile
  __shared__ double idg[32];    // 1 / diagonal of the factored block
  __shared__ int s_nv;
  const int lane = t & 31;
  for (int k0 = 0; k0 < ncols; k0 += 32) {
    const int nb = min(32, ncols - k0);
    for (int idx = t; idx < 32 * 32; idx += 256) {
      const int i = idx / 32, j = idx - i * 32;
      if (j <= i) D[i][j] = (i < nb) ? A[(size_t)(k0 + i) * ld + k0 + j] : 0.0;
    }
    __syncthreads();
    if (t < 32) {  // unblocked factor of the diagonal block: lane = row
      const int nv = warp_chol(D, nb, idg, t);
      if (t == 0) s_nv = nv;
    }
    __syncthreads();
    const int nv = s_nv;
    // rows below the block: x = A[r, k0 : k0 + nb] L_kk^-T, one warp per row, lane = column
    if (nv < nb) {  // a bad pivot: only row Rt - 1, over the nv good columns
      if (t < 32) {
        double* row = A + (size_t)(Rt - 1) * ld + k0;
        const double x = warp_row_solve(lane < nv ? row[lane] : 0.0, D, idg, nv, lane);
        if (lane < nv) row[lane] = x;
      }
      __syncthreads();
      return k0 + nv;
    }
    for (int r = k0 + nb + (t >> 5); r < Rt; r += 8) {
      double* row = A + (size_t)r * ld + k0;
      const double x = warp_row_solve(lane < nb ? row[lane] : 0.0, D, idg, nb, lane);
      if (lane < nb) row[lane] = x;
    }
    __syncthreads();
    // trailing update A[r, c] -= L[r, k0:k1] . L[c, k0:k1] for k1 <= c <= r, c < ncols, r < Rt (nb = 32 here): 32 x 32 tiles of
    // the lower triangle, both panels staged through shared memory
    const int k1 = k0 + nb;
    if (k1 < ncols) {
      const int nti = (Rt - k1 + 31) / 32, ntj = (ncols - k1 + 31) / 32;
      for (int ti = 0; ti < nti; ++ti)
        for (int tj = 0; tj <= ti && tj < ntj; ++tj) {
          const int rb = k1 + 32 * ti, cb = k1 + 32 * tj;
          for (int idx = t; idx < 32 * 32; idx += 256) {
            const int i = idx / 32, p = idx - i * 32;
            D[i][p] = (rb + i < Rt) ? A[(size_t)(rb + i) * ld + k0 + p] : 0.0;
            B[i][p] = (cb + i < ncols) ? A[(size_t)(cb + i) * ld + k0 + p] : 0.0;
          }
          __syncthreads();
          double s[4] = {0.0, 0.0, 0.0, 0.0};
          tile_dot32(D, B, t, s);
          const int r = rb + (t >> 3);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int c = cb + (t & 7) + 8 * u;
            if (r < Rt && c < ncols && c <= r) A[(size_t)r * ld + c] -= s[u];
          }
          __syncthreads();
        }
    }
  }
  return -1;
}

// ---- TMA (bulk async copy) staging of a small contiguous table into shared memory -----------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned phase) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(phase)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned phase) {
  while (!mbar_try_wait(bar, phase)) {
  }
}
// bytes must be a multiple of 16, both addresses 16-byte aligned.  SASS: UBLKCP.
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// Called by all threads of the CTA: thread 0 issues the bulk copy, everybody waits for completion.
__device__ __forceinline__ void stage_table_tma(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar) {
  if (threadIdx.x == 0) mbar_init(bar, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, bytes);
    tma_bulk_g2s(smem_dst, gmem_src, bytes, bar);
  }
  mbar_wait(bar, 0);
}

}  // namespace mb
