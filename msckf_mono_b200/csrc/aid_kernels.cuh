// msckf_mono_b200/csrc/aid_kernels.cuh
// Aided measurements fused into the device-resident filter (msckf_b200_aid_update / _batch_aid_update):
//   k_aid : residual r (from the resident state, or the caller's), H P (rows of P for the selection models, a product for a
//           caller-linearised H), S = H P H^T + R = L L^T with r as an extra row (y = L^-1 r), W = L^-1 H P, NIS = y^T y,
//           the optional chi-square gate, dx = W^T y, P <- P - W^T W (lower triangle in fp64, both halves written, rounded to
//           the filter precision once) and the state injection of k_syrk (inject_state).  All arithmetic in fp64.
// One CTA per member, one launch for everything; one body for a single filter (NM = 1) and a device batch (NM =
// kBatchMembers), like k_nees.  W^T and dx live in dynamic shared memory where they fit, else in a per-member global workspace.
#pragma once
#include "common.cuh"
#include "nees_kernels.cuh"
#include "state_kernels.cuh"

namespace mb {

// the models of msckf_b200_aid_model (include/msckf_b200.h)
enum AidModel { kAidVelocity = 0, kAidPosition = 1, kAidPose = 2, kAidClonePose = 3, kAidLinear = 4 };
constexpr int kAidMaxRows = 32;      // m <= 32: S is factored by one warp
constexpr int kAidZ = kAidMaxRows;   // input block: [32] z (or r of LINEAR), then R [m][m], then H [m][n] (LINEAR)
constexpr int kAidThreads = 256;

// per-member result; the first five fields are msckf_b200_aid_result's
struct AidOut {
  double nis, dx_norm;
  int dof, applied, status;
  int numeric;  // a non-finite dx or P entry was written
};

template <class S>
struct AidArgs {
  DevState<S>* st;
  S* P;
  S* poses;
  const double* in;  // the member's input block (layout above)
  double* ws;        // W^T [n][m] then dx [n] in global memory, or nullptr: in dynamic shared memory
  AidOut* out;
  double chi2_max;   // > 0: gate on NIS
  int ldp, M, model, clone, m, pad_;
};
static_assert(sizeof(Members<AidArgs<double>, kBatchMembers>) <= 32764, "k_aid's batched arguments exceed the parameter limit");

// bytes of W^T and dx of one member (in shared or global memory)
__host__ __device__ constexpr size_t aid_ws_bytes(int n, int m) { return sizeof(double) * (size_t)n * (m + 1); }

// state index of row i of a selection model: VELOCITY 6..8, POSITION 12..14, POSE [0..2, 12..14], CLONE_POSE 15+6k .. 20+6k
__device__ __forceinline__ int aid_index(int model, int clone, int i) {
  return model == kAidVelocity ? 6 + i : model == kAidPosition ? 12 + i : model == kAidPose ? (i < 3 ? i : 9 + i) : 15 + 6 * clone + i;
}

template <class S, int NM>
__global__ void __launch_bounds__(kAidThreads) k_aid(const Members<AidArgs<S>, NM> a) {
  extern __shared__ double aid_dyn[];
  const int f = NM == 1 ? 0 : blockIdx.x;
  DevState<S>* const st = a.m[f].st;
  S* __restrict__ const P = a.m[f].P;
  S* const poses = a.m[f].poses;
  const double* __restrict__ const in = a.m[f].in;
  AidOut* const out = a.m[f].out;
  const int ldp = a.m[f].ldp, M = a.m[f].M, model = a.m[f].model, clone = a.m[f].clone, m = a.m[f].m, n = 15 + 6 * M;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* const Wt = a.m[f].ws ? a.m[f].ws : aid_dyn;  // [n][m]: column c of H P, then of W = L^-1 H P
  double* const dx = Wt + (size_t)n * m;
  const double* __restrict__ const R = in + kAidZ;
  const double* __restrict__ const H = R + m * m;      // LINEAR only
  __shared__ double L[kAidMaxRows + 1][kAidMaxRows + 1];  // S = L L^T (lower); row m: r, then y = L^-1 r
  __shared__ double idg[kAidMaxRows];
  __shared__ double part[kAidThreads / 32];
  __shared__ int s_idx[kAidMaxRows];
  __shared__ int s_nv, s_apply, s_bad;

  // ---- residual (fp64) and the selected state indices
  if (model == kAidLinear) {
    if (t < m) L[m][t] = in[t];
  } else {
    if (t < m) s_idx[t] = aid_index(model, clone, t);
    if (t == 0) {
      const double* z = in;
      if (model == kAidVelocity) {
        for (int i = 0; i < 3; ++i) L[3][i] = z[i] - (double)st->v_I_G[i];
      } else if (model == kAidPosition) {
        for (int i = 0; i < 3; ++i) L[3][i] = z[i] - (double)st->p_I_G[i];
      } else {  // [dtheta(q_z, q_est); z_p - p_est], dtheta in the convention of the NEES error state
        const S* q = model == kAidPose ? st->q_IG : poses + kPoseStride * clone;
        const S* p = model == kAidPose ? st->p_I_G : poses + kPoseStride * clone + 4;
        nees_quat_error(z + 3, q, &L[6][0]);
        for (int i = 0; i < 3; ++i) L[6][3 + i] = z[i] - (double)p[i];
      }
    }
  }
  __syncthreads();
  // ---- H P, stored transposed: Wt[c][i] = (H P)[i][c]
  if (model == kAidLinear) {
    for (int idx = t; idx < m * n; idx += kAidThreads) {
      const int i = idx / n, c = idx - i * n;
      const double* h = H + (size_t)i * n;
      double s = 0.0;
      for (int k = 0; k < n; ++k) s += h[k] * (double)P[(size_t)k * ldp + c];
      Wt[(size_t)c * m + i] = s;
    }
  } else {
    for (int idx = t; idx < m * n; idx += kAidThreads) {
      const int i = idx / n, c = idx - i * n;
      Wt[(size_t)c * m + i] = (double)P[(size_t)s_idx[i] * ldp + c];
    }
  }
  __syncthreads();
  // ---- S = H P H^T + R, lower triangle (only R's lower triangle is read)
  for (int idx = t; idx < m * m; idx += kAidThreads) {
    const int i = idx / m, j = idx - i * m;
    if (j > i) continue;
    double s;
    if (model == kAidLinear) {
      const double* h = H + (size_t)j * n;
      s = 0.0;
      for (int k = 0; k < n; ++k) s += Wt[(size_t)k * m + i] * h[k];
    } else {
      s = Wt[(size_t)s_idx[j] * m + i];
    }
    L[i][j] = s + R[i * m + j];
  }
  __syncthreads();
  // ---- S = L L^T (one warp), then y = L^-1 r and W = L^-1 H P: rows of [W^T ; y^T] against L^T, one warp per row
  if (warp == 0) {
    const int nv = warp_chol(L, m, idg, lane);
    if (lane == 0) s_nv = nv;
  }
  __syncthreads();
  if (s_nv < m) {  // S not positive definite: nothing is written
    if (t == 0) {
      out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
      out->dof = m; out->applied = 0; out->status = 1; out->numeric = 0;
    }
    return;
  }
  for (int r = warp; r <= n; r += kAidThreads / 32) {
    double* row = r < n ? Wt + (size_t)r * m : &L[m][0];
    const double x = warp_row_solve(lane < m ? row[lane] : 0.0, L, idg, m, lane);
    if (lane < m) row[lane] = x;
  }
  __syncthreads();
  if (t == 0) {
    double g = 0.0;
    for (int i = 0; i < m; ++i) g += L[m][i] * L[m][i];
    const double chi2_max = a.m[f].chi2_max;
    s_apply = !(chi2_max > 0.0 && g > chi2_max);
    s_bad = 0;
    out->nis = g; out->dof = m; out->status = 0; out->applied = s_apply;
  }
  __syncthreads();
  if (!s_apply) {
    if (t == 0) { out->dx_norm = 0.0; out->numeric = 0; }
    return;
  }
  // ---- dx = W^T y, and P <- P - W^T W (lower triangle in fp64, written to both halves: exactly symmetric)
  double nn = 0.0;
  for (int c = t; c < n; c += kAidThreads) {
    const double* w = Wt + (size_t)c * m;
    double s = 0.0;
    for (int i = 0; i < m; ++i) s += w[i] * L[m][i];
    dx[c] = s;
    nn += s * s;
  }
  int bad = 0;
  for (int idx = t; idx < n * n; idx += kAidThreads) {
    const int r = idx / n, c = idx - r * n;
    if (c > r) continue;
    const double* wr = Wt + (size_t)r * m;
    const double* wc = Wt + (size_t)c * m;
    double v = 0.0;
    for (int i = 0; i < m; ++i) v += wr[i] * wc[i];
    const S x = (S)((double)P[(size_t)r * ldp + c] - v);
    if (!isfinite((double)x)) bad = 1;
    P[(size_t)r * ldp + c] = x;
    P[(size_t)c * ldp + r] = x;
  }
  nn = warp_sum(nn);
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (lane == 0) part[warp] = nn;
  if (bad && lane == 0) s_bad = 1;  // (benign race: every writer stores 1)
  __syncthreads();
  // ---- the state injection of the vision update (k_syrk)
  inject_state(st, poses, M, t, kAidThreads, [&](int i) { return dx[i]; });
  if (t == 0) {
    double s = 0.0;
    for (int w = 0; w < kAidThreads / 32; ++w) s += part[w];
    out->dx_norm = sqrt(s);
    out->numeric = (s_bad || !isfinite(s)) ? 1 : 0;
  }
}

}  // namespace mb
