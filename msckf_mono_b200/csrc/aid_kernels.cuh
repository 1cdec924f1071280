// msckf_mono_b200/csrc/aid_kernels.cuh
// Aided measurements fused into the device-resident filter (msckf_b200_aid_update / _batch_aid_update, the stacked
// msckf_b200_aid_stack_update / _batch_aid_stack_update and their fault detection and exclusion, _fde).  k_aid<S, NM, FDE>,
// one body for both forms:
//   rows   residual r and H (a stack of up to 8 model items, each row at most 12 (state index, coefficient) pairs formed from
//          the resident state; or the caller's r and dense H).  A degenerate heading or range item ends a plain member
//          (status 2); the FDE form drops it from the kept set A.
//   H P    sparse gathers over rows of P, or a product for a dense H; kept in Wt until the update.
//   rounds S_AA = (H P H^T + R)_AA = L L^T with r_A as an extra row (y = L^-1 r_A), NIS = y^T y and the gate.  Plain: one
//          round over every row, gated on the optional chi2_max.  FDE: gated on chi2[d_A - 1]; while it fails, an exclusion
//          round removes the item with the largest t_j / chi2[d_j - 1] (t_j = y_j^T B_j^-1 y_j, y = S_AA^-1 r,
//          B_j = (S_AA^-1)_jj; one warp per item), and the next round rebuilds S_AA.
//   update W = L^-1 H P over A's rows, dx = W^T y, P <- P - W^T W (lower triangle in fp64, both halves written, rounded to the
//          filter precision once) and the state injection of k_syrk (inject_state).
// All arithmetic in fp64; the FDE form's update of the final A is the plain arithmetic on those rows, in their order.
// k_aid_iter<S, NM, FDE> (_iter, an iterated EKF) is the same body with IT: after linearisation 0 has decided everything but the
// step, each further linearisation forms the rows of A at the fp64 iterate x^ [+] delta_i (AidIterate), factors S_AA against the
// prior P with r~ = r + H delta_i and forms delta_{i+1} = W^T y over delta_i in dx, until the step is <= tol or max_iter
// linearisations are made; then the downdate and injection of the last one.  A degenerate item at an iterate ends the
// iteration with the previous linearisation's W and dx, which nothing has overwritten yet.
// One CTA per member, one launch for everything; one body for a single filter (NM = 1) and a device batch (NM =
// kBatchMembers), like k_nees.  W^T and dx live in dynamic shared memory where they fit, else in a per-member global workspace.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "nees_kernels.cuh"
#include "state_kernels.cuh"

namespace mb {

// the models of msckf_b200_aid_model (include/msckf_b200.h)
enum AidModel {
  kAidVelocity = 0, kAidPosition = 1, kAidPose = 2, kAidClonePose = 3, kAidLinear = 4, kAidBodyVelocity = 5, kAidRelativePose = 6,
  kAidAntennaPosition = 7, kAidCloneAntennaPosition = 8, kAidHeading = 9, kAidCloneHeading = 10,
  kAidRange = 11, kAidCloneRange = 12, kAidPlaneRange = 13, kAidClonePlaneRange = 14, kAidGyroAtRest = 15, kAidAccelAtRest = 16
};
constexpr double kAidHeadingMinHoriz = 1e-6;  // HEADING: d_x^2 + d_y^2 <= this |f|^2 (f within ~1e-3 rad of vertical) is degenerate
constexpr double kAidRangeMin = 1e-6;         // RANGE: a predicted range at or below this (m) leaves its direction undefined
constexpr double kAidPlaneMinBeamZ = 1e-6;    // PLANE_RANGE: b_z^2 <= this (the beam within ~1e-3 rad of the plane) is degenerate
constexpr int kAidMaxRows = 32;      // m <= 32: S is factored by one warp
constexpr int kAidMaxItems = 8;      // model items of one stack
constexpr int kAidItemZ = 8;         // doubles reserved for one item's z
constexpr int kAidNnz = 12;          // (state index, coefficient) pairs of one row of a model's H
constexpr int kAidZ = kAidMaxItems * kAidItemZ;  // input block: [8][8] z of the items (LINEAR: r [m]), R [m][m], H [m][n] (LINEAR)
constexpr int kAidThreads = 256;

// per-member result; the first five fields are msckf_b200_aid_result's
struct AidOut {
  double nis, dx_norm;
  int dof, applied, status;
  int numeric;  // a non-finite dx or P entry was written
};
// per-member result of the FDE form: the plain result, then msckf_b200_aid_fde_result's outcome, count and item block
struct AidItemOut {
  double nis, test;
  int state, round;
};
struct AidFdeOut {
  AidOut stack;
  int outcome, n_excluded;
  AidItemOut item[kAidMaxItems];
};
constexpr int kAidFdeIn = kAidMaxRows + 1;  // FDE: chi2[32] then max_exclude (as a double) follow R in the input block

// lane 0: v^T A^-1 v of a d x d symmetric A (row-major, lower triangle read, overwritten by its Cholesky factor; v by
// L^-1 v); NaN when A is not positive definite.  (k_aid<S, NM, true>: an item's NIS and its exclusion statistic)
__device__ __noinline__ double aid_small_quad(double* A, double* v, int d) {
  double q = 0.0;
  for (int j = 0; j < d; ++j) {
    double s = A[j * d + j];
    for (int k = 0; k < j; ++k) s -= A[j * d + k] * A[j * d + k];
    if (!(s > 0.0)) return __longlong_as_double(0x7ff8000000000000ll);
    const double l = sqrt(s);
    A[j * d + j] = l;
    for (int i = j + 1; i < d; ++i) {
      double t = A[i * d + j];
      for (int k = 0; k < j; ++k) t -= A[i * d + k] * A[j * d + k];
      A[i * d + j] = t / l;
    }
    double x = v[j];
    for (int k = 0; k < j; ++k) x -= A[j * d + k] * v[k];
    v[j] = x / l;
    q += v[j] * v[j];
  }
  return q;
}

// one item of a stack: its model, a (CLONE_POSE, RELATIVE_POSE, CLONE_ANTENNA_POSITION, CLONE_HEADING, CLONE_RANGE,
// CLONE_PLANE_RANGE: a clone's window position; BODY_VELOCITY, ANTENNA_POSITION: the row mask), b (RELATIVE_POSE: the second clone; CLONE_ANTENNA_POSITION: the row
// mask) and its first row in the stack
struct AidItem {
  short model, a, b, row;
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
  int ldp, M, m, n_items;  // LINEAR: one item of model kAidLinear
  AidItem item[kAidMaxItems];
};
static_assert(sizeof(Members<AidArgs<double>, kBatchMembers>) <= 32764, "k_aid's batched arguments exceed the parameter limit");

// bytes of W^T and dx of one member (in shared or global memory); the iterated form keeps delta_i in dx (below), so it needs
// no more
__host__ __device__ constexpr size_t aid_ws_bytes(int n, int m) { return sizeof(double) * (size_t)n * (m + 1); }

// The iterated form (IT): per member, the input block ends with max_iter and tol (as doubles), after R and the FDE block, and
// the result with AidIterOut, after AidOut or AidFdeOut (msckf_b200_aid_iter / _aid_iter_result)
constexpr int kAidMaxIter = 16;
struct AidIterOut {
  int iterations, converged;
  double step;
};

// Where aid_item_rows reads the state from its two pointers (st, poses): the IMU's q_IG, v_I_G, p_I_G and clone k's pose (q, p
// at offsets 0 and 4).  AidResident: the filter's own (DevState<S>, its poses), with b_g, b_a and g for the at-rest models.
template <class S>
struct AidResident {
  using St = DevState<S>;
  using Pose = S;
  static __device__ const S* q(const St* st, const S*) { return st->q_IG; }
  static __device__ const S* v(const St* st, const S*) { return st->v_I_G; }
  static __device__ const S* p(const St* st, const S*) { return st->p_I_G; }
  static __device__ const S* pose(const St*, const S* poses, const AidItem&, int k) { return poses + kPoseStride * k; }
  static __device__ const S* b_g(const St* st) { return st->b_g; }
  static __device__ const S* b_a(const St* st) { return st->b_a; }
  static __device__ const S* g(const St* st) { return st->g; }
};
// AidIterate: st is one item's fp64 iterate x^ [+] delta_i (kAidIterX doubles; poses is not read): [0, 7) q, p of the IMU or
// of clone a, [7, 14) q, p of clone b (RELATIVE_POSE), [14, 17) v_I_G.  Only the poses the item names are there.  It carries no
// biases, so the at-rest models are not formed at an iterate (the iterated calls refuse them).
constexpr int kAidIterX = 17;
struct AidIterate {
  using St = double;
  using Pose = double;
  static __device__ const double* q(const double* x, const double*) { return x; }
  static __device__ const double* v(const double* x, const double*) { return x + 14; }
  static __device__ const double* p(const double* x, const double*) { return x + 4; }
  static __device__ const double* pose(const double* x, const double*, const AidItem& it, int k) { return k == it.a ? x : x + 7; }
};

// q, p of x^ [+] delta in fp64 (inject_state's arithmetic on the widened values): the IMU's q <- buildUpdateQuat(dtheta) * q, not
// renormalised (clone = false), or a clone's q <- normalise(buildUpdateQuat(dtheta) * q); p <- p + dp.  d: the pose's
// [dtheta, dp] (IMU: dtheta at d[0..2], dp at d[12..14]).
template <class S>
__device__ __forceinline__ void aid_boxplus(const S* q, const S* p, const double* dth, const double* dp, bool clone, double* x) {
  const double qw[4] = {(double)q[0], (double)q[1], (double)q[2], (double)q[3]};
  double uq[4];
  build_update_quat(dth, uq);
  quat_mul(uq, qw, x);
  if (clone) quat_normalize(x);
  for (int i = 0; i < 3; ++i) x[4 + i] = (double)p[i] + dp[i];
}
// item `it`'s iterate table at x^ [+] delta (dx: delta over the full state)
template <class S>
__device__ __noinline__ void aid_iterate(const AidItem it, const DevState<S>* st, const S* poses, const double* dx, double* x) {
  const bool clone = it.model == kAidClonePose || it.model == kAidRelativePose || it.model == kAidCloneAntennaPosition ||
                     it.model == kAidCloneHeading || it.model == kAidCloneRange || it.model == kAidClonePlaneRange;
  if (clone) {
    const S* ps = poses + kPoseStride * it.a;
    aid_boxplus(ps, ps + 4, dx + 15 + 6 * it.a, dx + 18 + 6 * it.a, true, x);
  } else {
    aid_boxplus(st->q_IG, st->p_I_G, dx, dx + 12, false, x);
  }
  if (it.model == kAidRelativePose) {
    const S* ps = poses + kPoseStride * it.b;
    aid_boxplus(ps, ps + 4, dx + 15 + 6 * it.b, dx + 18 + 6 * it.b, true, x + 7);
  }
  for (int i = 0; i < 3; ++i) x[14 + i] = (double)st->v_I_G[i] + dx[6 + i];
}

// The rows of one model item: residual r[row + i] (fp64) and row row + i of H as nnz (state index, coefficient) pairs.
// Perturbations follow the state injection, C(q+) = (I - [dtheta]x) C(q) (q+ = buildUpdateQuat(dtheta) * q), and the
// rotation residual is dtheta(q_z, q^) of msckf_b200_nees, so that r ~ H dx to first order:
//   VELOCITY, POSITION, POSE, CLONE_POSE  one coefficient 1 per row (the state index the model selects)
//   BODY_VELOCITY  v^ = C(q_IG) v_I_G; row j of the mask: r = z_j - v^_j, H over dtheta [v^]x (row j), over dv C (row j)
//   RELATIVE_POSE  C^ = C_b C_a^T, q^ = q_b * q_a^-1, p^ = C_a (p_b - p_a) of clones a, b:
//                  rotation rows  H over dtheta_a -C^, over dtheta_b I, over dp_a and dp_b 0
//                  position rows  H over dtheta_a [p^]x, over dp_a -C_a, over dtheta_b 0, over dp_b C_a
//   ANTENNA_POSITION, CLONE_ANTENNA_POSITION  z = p_A_G (3), lever l (3) in the body frame of the IMU or of clone k; with
//                  C = C(q), d = C^T l: p^ = p + d; row j of the mask: r = z_j - p^_j, H over dtheta -C^T [l]x = -[d]x C^T (row j),
//                  over dp the unit row j
//   HEADING, CLONE_HEADING  z = psi (1), axis f (3) in the body frame; d = C^T f, psi^ = atan2(d_y, d_x), r = wrap(z - psi^)
//                  into (-pi, pi]; H over dtheta [-d_y, d_x, 0] / (d_x^2 + d_y^2) (-[d]x C^T).  d_x^2 + d_y^2 <=
//                  kAidHeadingMinHoriz |f|^2 (yaw undefined) forms no row and returns 1: k_aid writes nothing (status 2).
//   RANGE, CLONE_RANGE  z = rho, anchor a_G (3), lever l (3) in the body frame; e = p + d - a, rho^ = |e|, u = e / rho^,
//                  r = rho - rho^; H over dtheta u^T J, over dp u^T.  rho^ <= kAidRangeMin returns 1 (status 2).
//   PLANE_RANGE, CLONE_PLANE_RANGE  z = rho, plane height h, lever l (3), beam axis f (3) in the body frame; the plane is
//                  {x : x_z = h} in G.  b = C^T f / |f|, rho^ = (h - (p + d)_z) / b_z, r = rho - rho^; with d' = C^T (l + rho^ f/|f|)
//                  (the hit point from the body) and J' = -[d']x C^T: H over dtheta -J'_z / b_z (= e_z^T C^T [l + rho^ f/|f|]x / b_z),
//                  over dp_z -1 / b_z.  b_z^2 <= kAidPlaneMinBeamZ or rho^ <= 0 (the plane behind the sensor) returns 1 (status 2).
//   GYRO_AT_REST   z = the mean gyro reading of a standstill (3); r = z - b_g, H over db_g (3..5) the identity
//   ACCEL_AT_REST  z = the mean specific force of a standstill (3); h = b_a - C g (C = C(q_IG), g the resident gravity), r = z - h;
//                  H over dtheta -[C g]x (C+ g = C g + [C g]x dtheta), over db_a (9..11) the identity.  H_theta (C g) = 0: no yaw.
// The state X the rows are formed at: AidResident (the filter's) or AidIterate (an iterate of the iterated form).
// Returns 0 when the rows are formed.
// (Out of line, with the item by value: inlined into k_aid<double, 1>, this code made ptxas spill.)
template <class X>
__device__ __noinline__ int aid_item_rows(const AidItem it, const double* z, const typename X::St* st, const typename X::Pose* poses,
                                             double* r, int (*col)[kAidNnz], double (*coef)[kAidNnz], int* nnz) {
  const int r0 = it.row;
  if (it.model == kAidVelocity || it.model == kAidPosition) {
    const auto* v = it.model == kAidVelocity ? X::v(st, poses) : X::p(st, poses);
    for (int i = 0; i < 3; ++i) {
      r[r0 + i] = z[i] - (double)v[i];
      col[r0 + i][0] = (it.model == kAidVelocity ? 6 : 12) + i; coef[r0 + i][0] = 1.0; nnz[r0 + i] = 1;
    }
  } else if (it.model == kAidPose || it.model == kAidClonePose) {  // [dtheta(q_z, q_est); z_p - p_est]
    const bool imu = it.model == kAidPose;
    const auto* q = imu ? X::q(st, poses) : X::pose(st, poses, it, it.a);
    const auto* p = imu ? X::p(st, poses) : X::pose(st, poses, it, it.a) + 4;
    nees_quat_error(z + 3, q, r + r0);
    for (int i = 0; i < 3; ++i) r[r0 + 3 + i] = z[i] - (double)p[i];
    for (int i = 0; i < 6; ++i) {
      col[r0 + i][0] = imu ? (i < 3 ? i : 9 + i) : 15 + 6 * it.a + i; coef[r0 + i][0] = 1.0; nnz[r0 + i] = 1;
    }
  } else if (it.model == kAidBodyVelocity) {
    const auto* Q = X::q(st, poses);
    const auto* V = X::v(st, poses);
    const double q[4] = {(double)Q[0], (double)Q[1], (double)Q[2], (double)Q[3]};
    double C[9], v[3];
    quat_to_rot(q, C);
    for (int j = 0; j < 3; ++j) v[j] = C[3 * j] * (double)V[0] + C[3 * j + 1] * (double)V[1] + C[3 * j + 2] * (double)V[2];
    const double sk[9] = {0.0, -v[2], v[1], v[2], 0.0, -v[0], -v[1], v[0], 0.0};  // [v^]x
    int row = r0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if ((it.a >> j) & 1) {
        r[row] = z[j] - v[j];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          col[row][k] = k; coef[row][k] = sk[3 * j + k];
          col[row][3 + k] = 6 + k; coef[row][3 + k] = C[3 * j + k];
        }
        nnz[row++] = 6;
      }
    }
  } else if (it.model == kAidGyroAtRest || it.model == kAidAccelAtRest) {  // the IMU at rest (AidResident only)
    if constexpr (std::is_same<X, AidIterate>::value) {
      return 1;
    } else {
      const bool gyro = it.model == kAidGyroAtRest;
      const auto* b = gyro ? X::b_g(st) : X::b_a(st);
      double u[3] = {0.0, 0.0, 0.0};  // ACCEL_AT_REST: C g
      if (!gyro) {
        const auto* Q = X::q(st, poses);
        const auto* G = X::g(st);
        const double q[4] = {(double)Q[0], (double)Q[1], (double)Q[2], (double)Q[3]};
        double C[9];
        quat_to_rot(q, C);
        for (int j = 0; j < 3; ++j) u[j] = C[3 * j] * (double)G[0] + C[3 * j + 1] * (double)G[1] + C[3 * j + 2] * (double)G[2];
      }
      const double sk[9] = {0.0, u[2], -u[1], -u[2], 0.0, u[0], u[1], -u[0], 0.0};  // -[C g]x
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int row = r0 + j;
        r[row] = z[j] - ((double)b[j] - u[j]);
        if (gyro) {
          col[row][0] = 3 + j; coef[row][0] = 1.0; nnz[row] = 1;
        } else {
#pragma unroll
          for (int k = 0; k < 3; ++k) { col[row][k] = k; coef[row][k] = sk[3 * j + k]; }
          col[row][3] = 9 + j; coef[row][3] = 1.0; nnz[row] = 4;
        }
      }
    }
  } else if (it.model >= kAidAntennaPosition) {  // the antenna positions, headings and ranges, of the IMU or of clone a
    const bool clone = it.model == kAidCloneAntennaPosition || it.model == kAidCloneHeading || it.model == kAidCloneRange ||
                       it.model == kAidClonePlaneRange;
    const bool heading = it.model == kAidHeading || it.model == kAidCloneHeading;
    const bool range = it.model == kAidRange || it.model == kAidCloneRange;
    const bool plane = it.model == kAidPlaneRange || it.model == kAidClonePlaneRange;
    const auto* Q = clone ? X::pose(st, poses, it, it.a) : X::q(st, poses);
    const double q[4] = {(double)Q[0], (double)Q[1], (double)Q[2], (double)Q[3]};
    const double* l = heading ? z + 1 : range ? z + 4 : plane ? z + 2 : z + 3;  // the lever arm or the axis, in the body frame
    const int c0 = clone ? 15 + 6 * it.a : 0;   // the pose's dtheta
    const auto* p = clone ? X::pose(st, poses, it, it.a) + 4 : X::p(st, poses);
    const int cp = clone ? c0 + 3 : 12;         // the pose's dp
    double C[9], d[3], J[9];
    quat_to_rot(q, C);
    for (int i = 0; i < 3; ++i) d[i] = C[i] * l[0] + C[3 + i] * l[1] + C[6 + i] * l[2];
    double rho = 0.0, bz = 0.0;  // PLANE_RANGE: rho^ and b_z
    if (plane) {  // d becomes C^T (l + rho^ f/|f|), the hit point from the body, so that J below is J'
      const double* f = z + 5;
      const double nf = sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
      double b[3];
      for (int i = 0; i < 3; ++i) b[i] = (C[i] * f[0] + C[3 + i] * f[1] + C[6 + i] * f[2]) / nf;
      bz = b[2];
      rho = (z[1] - ((double)p[2] + d[2])) / bz;
      if (!(bz * bz > kAidPlaneMinBeamZ) || !(rho > 0.0)) return 1;
      for (int i = 0; i < 3; ++i) d[i] += rho * b[i];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {  // J = -[d]x C^T: column k is (row k of C) x d
      J[k] = C[3 * k + 1] * d[2] - C[3 * k + 2] * d[1];
      J[3 + k] = C[3 * k + 2] * d[0] - C[3 * k] * d[2];
      J[6 + k] = C[3 * k] * d[1] - C[3 * k + 1] * d[0];
    }
    if (range) {
      const double e[3] = {(double)p[0] + d[0] - z[1], (double)p[1] + d[1] - z[2], (double)p[2] + d[2] - z[3]};
      const double rh = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
      if (!(rh > kAidRangeMin)) return 1;
      r[r0] = z[0] - rh;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        col[r0][k] = c0 + k; coef[r0][k] = (e[0] * J[k] + e[1] * J[3 + k] + e[2] * J[6 + k]) / rh;
        col[r0][3 + k] = cp + k; coef[r0][3 + k] = e[k] / rh;
      }
      nnz[r0] = 6;
    } else if (plane) {
      r[r0] = z[0] - rho;
#pragma unroll
      for (int k = 0; k < 3; ++k) { col[r0][k] = c0 + k; coef[r0][k] = -J[6 + k] / bz; }
      col[r0][3] = cp + 2; coef[r0][3] = -1.0 / bz;
      nnz[r0] = 4;
    } else if (!heading) {
      const int mask = clone ? it.b : it.a;
      int row = r0;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        if ((mask >> j) & 1) {
          r[row] = z[j] - ((double)p[j] + d[j]);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            col[row][k] = c0 + k; coef[row][k] = J[3 * j + k];
            col[row][3 + k] = cp + k; coef[row][3 + k] = j == k ? 1.0 : 0.0;
          }
          nnz[row++] = 6;
        }
      }
    } else {
      const double h = d[0] * d[0] + d[1] * d[1];
      if (!(h > kAidHeadingMinHoriz * (l[0] * l[0] + l[1] * l[1] + l[2] * l[2]))) return 1;
      constexpr double kPi = 3.141592653589793, k2Pi = 6.283185307179586;
      double e = remainder(z[0] - atan2(d[1], d[0]), k2Pi);
      if (e <= -kPi) e += k2Pi;
      r[r0] = e;
      const double gx = -d[1] / h, gy = d[0] / h;
#pragma unroll
      for (int k = 0; k < 3; ++k) { col[r0][k] = c0 + k; coef[r0][k] = gx * J[k] + gy * J[3 + k]; }
      nnz[r0] = 3;
    }
  } else {  // kAidRelativePose
    const auto* A = X::pose(st, poses, it, it.a);
    const auto* B = X::pose(st, poses, it, it.b);
    const double qa[4] = {(double)A[0], (double)A[1], (double)A[2], (double)A[3]};
    const double qb[4] = {(double)B[0], (double)B[1], (double)B[2], (double)B[3]};
    const double na = qa[0] * qa[0] + qa[1] * qa[1] + qa[2] * qa[2] + qa[3] * qa[3];
    const double qai[4] = {-qa[0] / na, -qa[1] / na, -qa[2] / na, qa[3] / na};
    double Ca[9], Cb[9], Ch[9], qh[4], ph[3];
    quat_to_rot(qa, Ca);
    quat_to_rot(qb, Cb);
    quat_mul(qb, qai, qh);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Ch[3 * i + j] = Cb[3 * i] * Ca[3 * j] + Cb[3 * i + 1] * Ca[3 * j + 1] + Cb[3 * i + 2] * Ca[3 * j + 2];
    const double d[3] = {(double)B[4] - (double)A[4], (double)B[5] - (double)A[5], (double)B[6] - (double)A[6]};
    for (int i = 0; i < 3; ++i) ph[i] = Ca[3 * i] * d[0] + Ca[3 * i + 1] * d[1] + Ca[3 * i + 2] * d[2];
    nees_quat_error(z + 3, qh, r + r0);
    for (int i = 0; i < 3; ++i) r[r0 + 3 + i] = z[i] - ph[i];
    const double sk[9] = {0.0, -ph[2], ph[1], ph[2], 0.0, -ph[0], -ph[1], ph[0], 0.0};  // [p^]x
    const int ca = 15 + 6 * it.a, cb = 15 + 6 * it.b;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        col[r0 + i][k] = ca + k; col[r0 + i][3 + k] = ca + 3 + k; col[r0 + i][6 + k] = cb + k; col[r0 + i][9 + k] = cb + 3 + k;
        if (i < 3) {
          coef[r0 + i][k] = -Ch[3 * i + k]; coef[r0 + i][3 + k] = 0.0; coef[r0 + i][6 + k] = i == k ? 1.0 : 0.0; coef[r0 + i][9 + k] = 0.0;
        } else {
          coef[r0 + i][k] = sk[3 * (i - 3) + k]; coef[r0 + i][3 + k] = -Ca[3 * (i - 3) + k];
          coef[r0 + i][6 + k] = 0.0; coef[r0 + i][9 + k] = Ca[3 * (i - 3) + k];
        }
      }
      nnz[r0 + i] = kAidNnz;
    }
  }
  return 0;
}

// The member's result when nothing is written: NIS NaN, no step, not applied
__device__ __forceinline__ void aid_nothing(AidOut* out, int dof, int status) {
  out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
  out->dof = dof; out->applied = 0; out->status = status; out->numeric = 0;
}

// The body of k_aid and k_aid_iter (IT: the iterated form).  Two kernel names keep each form's resource lines apart.
template <class S, int NM, bool FDE, bool IT>
__device__ __forceinline__ void aid_body(const Members<AidArgs<S>, NM>& a) {
  extern __shared__ double aid_dyn[];
  const int f = NM == 1 ? 0 : blockIdx.x;
  DevState<S>* const st = a.m[f].st;
  S* __restrict__ const P = a.m[f].P;
  S* const poses = a.m[f].poses;
  const double* __restrict__ const in = a.m[f].in;
  AidOut* const out = a.m[f].out;
  const int ldp = a.m[f].ldp, M = a.m[f].M, m = a.m[f].m, n = 15 + 6 * M;
  const int& n_items = a.m[f].n_items;  // (read where used: a copy held in a register cost the batched forms 8 registers)
  const bool lin = !FDE && !IT && a.m[f].item[0].model == kAidLinear;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* const Wt = a.m[f].ws ? a.m[f].ws : aid_dyn;  // [n][m]: column c of H P, then of W = L^-1 H P
  double* const dx = Wt + (size_t)n * m;               // (IT: delta_i until the pass that forms delta_{i+1} over it)
  const double* __restrict__ const R = in + kAidZ;
  const double* __restrict__ const H = R + m * m;      // LINEAR only
  __shared__ double L[kAidMaxRows + 1][kAidMaxRows + 1];  // S_AA = L L^T (lower); row m_A: r_A, then y = L^-1 r_A
  __shared__ double idg[kAidMaxRows];
  __shared__ double part[kAidThreads / 32];
  __shared__ int s_col[kAidMaxRows][kAidNnz];             // the model rows of H: (state index, coefficient) pairs
  __shared__ double s_coef[kAidMaxRows][kAidNnz];
  __shared__ int s_nnz[kAidMaxRows];
  __shared__ int s_nv, s_apply, s_bad;
  // FDE or IT only (r kept apart from the factor): the plain form never touches it, so it allocates none of it
  __shared__ double s_r[kAidMaxRows];                    // r, for every round and every linearisation
  // FDE only
  __shared__ int s_ri[kAidMaxRows], s_c0[kAidMaxItems];  // row k of S_AA is stack row s_ri[k]; item w's first row in S_AA
  __shared__ double s_t[kAidMaxItems], s_blk[kAidMaxItems][42];  // t_j of the round; a warp's d x d block and vector
  __shared__ unsigned s_A;  // the items of A (bits)
  __shared__ int s_mA, s_done;  // s_done: the outcome once it is decided, else -1
  // IT only
  __shared__ double s_x[kAidMaxItems][kAidIterX];  // each item's iterate
  __shared__ int s_go;
  AidFdeOut* const fo = reinterpret_cast<AidFdeOut*>(out);
  const double* __restrict__ const chi2 = R + m * m;     // FDE: chi2[32], then max_exclude
  const double* __restrict__ const itin = chi2 + (FDE ? kAidFdeIn : 0);  // IT: max_iter, tol
  AidIterOut* const io = reinterpret_cast<AidIterOut*>(reinterpret_cast<char*>(out) + (FDE ? sizeof(AidFdeOut) : sizeof(AidOut)));
  const auto rows_of = [&](int k) { return (k + 1 < n_items ? a.m[f].item[k + 1].row : m) - a.m[f].item[k].row; };
  double* const rv = FDE || IT ? s_r : &L[m][0];

  // Linearisation li (IT: 0 .. max_iter - 1; otherwise 0 only) at the iterate x^ [+] delta_li (delta_0 = 0).  Linearisation 0
  // decides everything the result reports but the step: the NIS, dof, the gate and FDE's kept set A; the later ones rebuild
  // the rows of A at the iterate and factor S_AA against the prior P with r~ = r + H delta_li.
  int ma = m, n_exc = 0;
  double nn = 0.0;
  for (int li = 0;; ++li) {
    // ---- residual (fp64) and the rows of H, one thread per item.  A degenerate item (a heading whose yaw or a range whose
    // prediction is undefined) ends a plain member at linearisation 0; the FDE form drops it from A and never reads its rows.
    // At an iterate, a degenerate item of A ends the iteration: the previous linearisation is applied.
    int degenerate = 0;
    if (lin) {
      if (t < m) L[m][t] = in[t];
    } else if (t < n_items) {
      if (!IT || li == 0) {
        degenerate = aid_item_rows<AidResident<S>>(a.m[f].item[t], in + kAidItemZ * t, st, poses, rv, s_col, s_coef, s_nnz);
        if constexpr (FDE)
          fo->item[t] = {__longlong_as_double(0x7ff8000000000000ll), __longlong_as_double(0x7ff8000000000000ll), degenerate ? 2 : 3, -1};
      } else if constexpr (IT) {
        if (!FDE || ((s_A >> t) & 1u)) {
          aid_iterate(a.m[f].item[t], st, poses, dx, s_x[t]);
          degenerate = aid_item_rows<AidIterate>(a.m[f].item[t], in + kAidItemZ * t, s_x[t], nullptr, rv, s_col, s_coef, s_nnz);
        }
      }
    }
    bool stop;
    if (IT && li > 0) {
      stop = __syncthreads_or(degenerate);
      if (stop) break;
    } else if constexpr (FDE) {
      const unsigned keep = __ballot_sync(0xffffffffu, t < n_items && !degenerate);
      if (t == 0) s_A = keep;
      __syncthreads();
      stop = s_A == 0u;  // every item degenerate
    } else {
      stop = __syncthreads_or(degenerate);
    }
    if (stop) {  // nothing is written
      if (t == 0) {
        aid_nothing(out, FDE ? 0 : m, 2);
        if constexpr (FDE) { fo->outcome = -1; fo->n_excluded = 0; }
        if constexpr (IT) *io = {0, 0, 0.0};
      }
      return;
    }
    // ---- H P, stored transposed: Wt[c][i] = (H P)[i][c] (FDE: of the kept rows); every round forms S_AA from it
    if (lin) {
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
        if constexpr (FDE) {
          int k = 0;
          while (k + 1 < n_items && a.m[f].item[k + 1].row <= i) ++k;
          if (!((s_A >> k) & 1u)) continue;
        }
        double s = s_coef[i][0] * (double)P[(size_t)s_col[i][0] * ldp + c];  // (exact for the one-coefficient rows)
        for (int k = 1; k < s_nnz[i]; ++k) s += s_coef[i][k] * (double)P[(size_t)s_col[i][k] * ldp + c];
        Wt[(size_t)c * m + i] = s;
      }
    }
    __syncthreads();
    if constexpr (FDE) {  // each kept item alone against the prior: r_j^T S_jj^-1 r_j (warp j, lane 0)
      if (li == 0 && warp < n_items && lane == 0 && ((s_A >> warp) & 1u)) {
        const int r0 = a.m[f].item[warp].row, d = rows_of(warp);
        double* B = s_blk[warp];
        for (int i = 0; i < d; ++i) {
          for (int j = 0; j <= i; ++j) {
            const int ri = r0 + i, rj = r0 + j;
            double s = s_coef[rj][0] * Wt[(size_t)s_col[rj][0] * m + ri];
            for (int q = 1; q < s_nnz[rj]; ++q) s += s_coef[rj][q] * Wt[(size_t)s_col[rj][q] * m + ri];
            B[i * d + j] = s + R[ri * m + rj];
          }
          B[36 + i] = s_r[r0 + i];
        }
        fo->item[warp].nis = aid_small_quad(B, B + 36, d);
      }
    }
    // ---- rounds over the kept set A (plain: one round, A every row): S_AA, its factor, y = L^-1 r_A, NIS and the gate.
    // FDE outcome 0: applied; 1: applied after exclusions; 2: rejected (at max_exclude); 3: no identifiable fault.  A later
    // linearisation is one round over the A linearisation 0 kept, with no gate.
    for (int round = 0;; ++round) {
      if constexpr (FDE) {
        if (t == 0) {
          int k = 0;
          for (int w = 0; w < n_items; ++w) {
            if (!((s_A >> w) & 1u)) continue;
            s_c0[w] = k;
            for (int i = 0, r0 = a.m[f].item[w].row, d = rows_of(w); i < d; ++i) s_ri[k++] = r0 + i;
          }
          s_mA = k;
        }
        __syncthreads();
        ma = s_mA;
      }
      // S_AA = (H P H^T + R)_AA, lower triangle (only R's lower triangle is read); R is block-diagonal across items, so S_AA is
      // a principal submatrix of S
      for (int idx = t; idx < ma * ma; idx += kAidThreads) {
        const int i = idx / ma, j = idx - i * ma;
        if (j > i) continue;
        const int ri = FDE ? s_ri[i] : i, rj = FDE ? s_ri[j] : j;
        double s;
        if (lin) {
          const double* h = H + (size_t)j * n;
          s = 0.0;
          for (int k = 0; k < n; ++k) s += Wt[(size_t)k * m + i] * h[k];
        } else {
          s = s_coef[rj][0] * Wt[(size_t)s_col[rj][0] * m + ri];
          for (int k = 1; k < s_nnz[rj]; ++k) s += s_coef[rj][k] * Wt[(size_t)s_col[rj][k] * m + ri];
        }
        L[i][j] = s + R[ri * m + rj];
      }
      if constexpr (FDE || IT) {
        if (t < ma) {
          const int ri = FDE ? s_ri[t] : t;
          double v = s_r[ri];
          if (IT && li > 0)  // r~ = r + H delta_li
            for (int k = 0; k < s_nnz[ri]; ++k) v += s_coef[ri][k] * dx[s_col[ri][k]];
          L[ma][t] = v;
        }
      }
      __syncthreads();
      if (warp == 0) {
        const int nv = warp_chol(L, ma, idg, lane);
        if (lane == 0) s_nv = nv;
        if (nv == ma) {
          const double x = warp_row_solve(lane < ma ? L[ma][lane] : 0.0, L, idg, ma, lane);
          if (lane < ma) L[ma][lane] = x;
        }
      }
      __syncthreads();
      if (s_nv < ma) {  // S_AA not positive definite (at any linearisation): nothing is written
        if (t == 0) {
          aid_nothing(out, ma, 1);
          if constexpr (FDE) { fo->outcome = -1; fo->n_excluded = n_exc; }
          if constexpr (IT) *io = {0, 0, 0.0};
        }
        return;
      }
      if (IT && li > 0) break;
      if (t == 0) {
        double g = 0.0;
        for (int i = 0; i < ma; ++i) g += L[ma][i] * L[ma][i];
        out->nis = g; out->dof = ma; out->status = 0;
        if constexpr (FDE) {
          const int max_exclude = (int)chi2[kAidMaxRows];
          s_done = !(g > chi2[ma - 1]) ? (n_exc ? 1 : 0) : n_exc >= max_exclude ? 2 : __popc(s_A) == 1 ? 3 : -1;
        } else {
          const double chi2_max = a.m[f].chi2_max;
          s_apply = !(chi2_max > 0.0 && g > chi2_max);
        }
      }
      __syncthreads();
      if constexpr (!FDE) {
        break;
      } else {
        if (s_done >= 0) break;
        // ---- exclusion round: warp w of A forms g_a = L^-1 e_a over its rows, y_w = G^T (L^-1 r_A), B_w = G^T G, t_w
        if (warp < n_items && ((s_A >> warp) & 1u)) {
          const int d = rows_of(warp), c0 = s_c0[warp];
          const double u = lane < ma ? L[ma][lane] : 0.0;
          double g[6];
#pragma unroll
          for (int p = 0; p < 6; ++p) {  // (lanes >= m_A hold whatever rows past the factor give: kept out of the sums)
            if (p < d) g[p] = warp_row_solve(lane == c0 + p ? 1.0 : 0.0, L, idg, ma, lane);
            if (lane >= ma) g[p] = 0.0;
          }
          double* B = s_blk[warp];
#pragma unroll
          for (int p = 0; p < 6; ++p) {
            if (p >= d) break;
            const double yp = warp_sum(g[p] * u);
            if (lane == 0) B[36 + p] = yp;
#pragma unroll
            for (int q = 0; q <= p; ++q) {
              const double bpq = warp_sum(g[p] * g[q]);
              if (lane == 0) B[p * d + q] = bpq;
            }
          }
          if (lane == 0) {
            s_t[warp] = aid_small_quad(B, B + 36, d);
            fo->item[warp].test = s_t[warp];
          }
        }
        __syncthreads();
        if (t == 0) {  // j* = argmax t_j / chi2[d_j - 1], the lowest item on a tie; not above 1: no single item explains it
          int best = -1;
          double rb = 1.0;
          for (int w = 0; w < n_items; ++w) {
            if (!((s_A >> w) & 1u)) continue;
            const double rw = s_t[w] / chi2[rows_of(w) - 1];
            if (rw > rb) { rb = rw; best = w; }
          }
          if (best < 0) {
            s_done = 3;
          } else {
            s_A &= ~(1u << best);
            fo->item[best].state = 1; fo->item[best].round = round;
          }
        }
        __syncthreads();
        if (s_done >= 0) break;
        ++n_exc;
      }
    }
    if (!IT || li == 0) {
      if (t == 0) {
        if constexpr (FDE) {
          fo->outcome = s_done; fo->n_excluded = n_exc;
          for (int w = 0; w < n_items; ++w)
            if ((s_A >> w) & 1u) fo->item[w].state = s_done <= 1 ? 0 : 3;
          s_apply = s_done <= 1;
        }
        out->applied = s_apply;
        s_bad = 0;
        if (!s_apply) { out->dx_norm = 0.0; out->numeric = 0; }
        if constexpr (IT) *io = {0, 0, 0.0};
      }
      __syncthreads();
      if (!s_apply) return;
    }
    // ---- W = L^-1 H P over the rows of A (FDE: gathered in order into the first m_A entries of each Wt row), one warp per row
    for (int r = warp; r < n; r += kAidThreads / 32) {
      double* row = Wt + (size_t)r * m;
      const double x0 = lane < ma ? row[FDE ? s_ri[lane] : lane] : 0.0;
      __syncwarp();
      const double x = warp_row_solve(x0, L, idg, ma, lane);
      if (lane < ma) row[lane] = x;
    }
    __syncthreads();
    // ---- dx = W^T y (IT: delta_{li+1}; each thread reads its own entries of delta_li before it overwrites them)
    nn = 0.0;
    double step = 0.0;
    for (int c = t; c < n; c += kAidThreads) {
      const double* w = Wt + (size_t)c * m;
      double s = 0.0;
      for (int i = 0; i < ma; ++i) s += w[i] * L[ma][i];
      if constexpr (IT) {  // |delta_{li+1} - delta_li|, NaN counted as infinite
        const double dc = fabs(s - (li == 0 ? 0.0 : dx[c]));
        step = fmax(step, isnan(dc) ? __longlong_as_double(0x7ff0000000000000ll) : dc);
      }
      dx[c] = s;
      if constexpr (!IT) nn += s * s;
    }
    if constexpr (!IT) {
      break;
    } else {  // stop after max_iter linearisations, or when the step is <= tol (converged); else relinearise at delta_{li+1}
      if (t == 0) io->iterations = li + 1;
      if (li + 1 >= (int)itin[0]) break;
      step = warp_max(step);
      if (lane == 0) part[warp] = step;
      __syncthreads();
      if (t == 0) {
        double s = part[0];
        for (int w = 1; w < kAidThreads / 32; ++w) s = fmax(s, part[w]);
        const int conv = s <= itin[1];
        io->step = s; io->converged = conv;
        s_go = !conv;
      }
      __syncthreads();
      if (!s_go) break;
    }
  }
  if constexpr (IT)  // |dx|^2 of the last linearisation (the sums of its pass, in the same order)
    for (int c = t; c < n; c += kAidThreads) nn += dx[c] * dx[c];
  // ---- P <- P - W^T W (lower triangle in fp64, written to both halves: exactly symmetric)
  int bad = 0;
  for (int idx = t; idx < n * n; idx += kAidThreads) {
    const int r = idx / n, c = idx - r * n;
    if (c > r) continue;
    const double* wr = Wt + (size_t)r * m;
    const double* wc = Wt + (size_t)c * m;
    double v = 0.0;
    for (int i = 0; i < ma; ++i) v += wr[i] * wc[i];
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

template <class S, int NM, bool FDE = false>
__global__ void __launch_bounds__(kAidThreads) k_aid(const Members<AidArgs<S>, NM> a) {
  aid_body<S, NM, FDE, false>(a);
}
// (one CTA per SM is what one member per CTA uses anyway; asked for, ptxas keeps the FDE form free of spills)
template <class S, int NM, bool FDE = false>
__global__ void __launch_bounds__(kAidThreads, 1) k_aid_iter(const Members<AidArgs<S>, NM> a) {
  aid_body<S, NM, FDE, true>(a);
}

}  // namespace mb
