// msckf_mono_b200/csrc/nees_kernels.cuh
// Consistency of the device-resident estimate against a caller-given ground truth (msckf_b200_nees / _batch_nees):
//   k_nees : error state (fp64), NEES e^T P^-1 e of the orientation, IMU pose, full IMU state and whole state from ONE
//            forward solve y = L^-1 e (prefix sums of y^2 in the order [dtheta_I, dp_I, dv, db_g, db_a, clones...]), and
//            the position NEES from its own 3 x 3 solve.
// One CTA per member; one body for a single filter (NM = 1) and a device batch (NM = kBatchMembers), like k_propagate.
// Read-only on the filter: P, the state and the poses are only read.
#pragma once
#include "common.cuh"
#include "state_kernels.cuh"

namespace mb {

// layout of msckf_b200_nees_result (include/msckf_b200.h)
struct NeesOut {
  double orientation, position, pose, imu, full;
  int dim_full, first_bad_pivot;
};
constexpr int kNeesTruthImu = 19;  // p, v, b_g, b_a, g, q_IG (the layout of msckf_b200_initialize's imu_state)

template <class S>
struct NeesArgs {
  const DevState<S>* st;
  const S* P;
  const S* poses;
  const double* truth;  // [19] IMU truth, then [M][7] clone truth p_C_G(3) q_CG(4) when n > 15
  double* W;            // workspace: (n + 1) rows of n doubles (row n: the error vector, then y = L^-1 e)
  NeesOut* out;
  int ldp, M, n, full;  // full = 1: truth poses given, n = 15 + 6 M; else n = 15
};
static_assert(sizeof(Members<NeesArgs<double>, kBatchMembers>) <= 32764, "k_nees's batched arguments exceed the parameter limit");

// state index of the NEES order [dtheta_I, dp_I, dv, db_g, db_a, clones]: the engine's order is [dtheta, db_g, dv, db_a, dp, clones]
__device__ __forceinline__ int nees_perm(int a) {
  if (a >= 15) return a;
  const int blk = a / 3, r = a - 3 * blk;
  return (blk == 0 ? 0 : blk == 1 ? 12 : blk == 2 ? 6 : blk == 3 ? 3 : 9) + r;
}

// the inverse of the state injection q+ = buildUpdateQuat(dtheta) * q (msckf.h:851-872, :1376-1390):
// dq = q_true * q_est^-1 (true inverse: conj / |q|^2), sign fixed so that dq.w >= 0, dtheta = -2 vec(dq)
template <class S>
__device__ __forceinline__ void nees_quat_error(const double* qt, const S* qe_, double* dth) {
  const double qe[4] = {(double)qe_[0], (double)qe_[1], (double)qe_[2], (double)qe_[3]};
  const double n2 = qe[0] * qe[0] + qe[1] * qe[1] + qe[2] * qe[2] + qe[3] * qe[3];
  const double qi[4] = {-qe[0] / n2, -qe[1] / n2, -qe[2] / n2, qe[3] / n2};
  double d[4];
  quat_mul(qt, qi, d);
  const double s = d[3] < 0.0 ? 2.0 : -2.0;
  dth[0] = s * d[0]; dth[1] = s * d[1]; dth[2] = s * d[2];
}

template <class S, int NM>
__global__ void __launch_bounds__(256) k_nees(const Members<NeesArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.x;
  const DevState<S>* __restrict__ const st = a.m[f].st;
  const S* __restrict__ const P = a.m[f].P;
  const S* __restrict__ const poses = a.m[f].poses;
  const double* __restrict__ const truth = a.m[f].truth;
  double* __restrict__ const W = a.m[f].W;
  NeesOut* const out = a.m[f].out;
  const int ldp = a.m[f].ldp, n = a.m[f].n, t = threadIdx.x;
  const bool full = a.m[f].full != 0;
  double* __restrict__ const e = W + (size_t)n * n;  // row n

  // ---- error state (fp64), in the NEES order
  if (t == 0) {
    nees_quat_error(truth + 15, st->q_IG, e);
    for (int i = 0; i < 3; ++i) {
      e[3 + i] = truth[i] - (double)st->p_I_G[i];
      e[6 + i] = truth[3 + i] - (double)st->v_I_G[i];
      e[9 + i] = truth[6 + i] - (double)st->b_g[i];
      e[12 + i] = truth[9 + i] - (double)st->b_a[i];
    }
  }
  for (int k = t; k < (n - 15) / 6; k += 256) {  // clone k: pose table q(4) p(3) pad, truth p(3) q(4)
    const S* ps = poses + kPoseStride * k;
    const double* tr = truth + kNeesTruthImu + 7 * k;
    nees_quat_error(tr + 3, ps, e + 15 + 6 * k);
    for (int i = 0; i < 3; ++i) e[15 + 6 * k + 3 + i] = tr[i] - (double)ps[4 + i];
  }
  // ---- lower triangle of P_SS in the NEES order (fp64)
  for (int idx = t; idx < n * n; idx += 256) {
    const int r = idx / n, c = idx - r * n;
    if (c <= r) W[(size_t)r * n + c] = (double)P[(size_t)nees_perm(r) * ldp + nees_perm(c)];
  }
  __syncthreads();

  // ---- Cholesky of [P_SS ; e^T] ((n + 1) x n): row n ends as y = L^-1 e (over the good pivots).  The factor stays in W.
  const int bad = cta_bordered_chol(W, n, n, n + 1, t);

  // ---- prefix sums of y^2; the position block by its own 3 x 3 solve
  if (t == 0) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const int lim = bad < 0 ? n : bad;
    double acc = 0.0, v3 = nan, v6 = nan, v15 = nan, vall = nan;
    for (int i = 0; i < lim; ++i) {
      acc += e[i] * e[i];
      if (i == 2) v3 = acc;
      if (i == 5) v6 = acc;
      if (i == 14) v15 = acc;
      if (i == n - 1 && full) vall = acc;
    }
    double pp[9], y[3], vp = 0.0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) pp[3 * i + j] = (double)P[(size_t)(12 + i) * ldp + 12 + j];
    const double ep[3] = {truth[0] - (double)st->p_I_G[0], truth[1] - (double)st->p_I_G[1], truth[2] - (double)st->p_I_G[2]};
    for (int i = 0; i < 3 && vp == vp; ++i) {  // column-by-column Cholesky of pp with the forward solve alongside
      double d = pp[4 * i];
      for (int k = 0; k < i; ++k) d -= pp[3 * i + k] * pp[3 * i + k];
      if (!(d > 0.0)) { vp = nan; break; }
      const double l = sqrt(d);
      pp[4 * i] = l;
      for (int r = i + 1; r < 3; ++r) {
        double s = pp[3 * r + i];
        for (int k = 0; k < i; ++k) s -= pp[3 * r + k] * pp[3 * i + k];
        pp[3 * r + i] = s / l;
      }
      double s = ep[i];
      for (int k = 0; k < i; ++k) s -= pp[3 * i + k] * y[k];
      y[i] = s / l;
      vp += y[i] * y[i];
    }
    out->orientation = v3; out->position = vp; out->pose = v6; out->imu = v15; out->full = vall;
    out->dim_full = full ? n : 0;
    out->first_bad_pivot = bad;
  }
}

}  // namespace mb
