// msckf_mono_b200/csrc/aid_kernels.cuh
// Aided measurements fused into the device-resident filter (msckf_b200_aid_update / _batch_aid_update and the stacked
// msckf_b200_aid_stack_update / _batch_aid_stack_update):
//   k_aid : residual r and H (a stack of up to 8 model items, each row at most 12 (state index, coefficient) pairs formed from
//           the resident state; or the caller's r and dense H; a degenerate heading or range item ends the member: status 2), H P (sparse gathers over rows of P, or a product for a dense H),
//           S = H P H^T + R = L L^T with r as an extra row (y = L^-1 r), W = L^-1 H P, NIS = y^T y, the optional chi-square
//           gate, dx = W^T y, P <- P - W^T W (lower triangle in fp64, both halves written, rounded to the filter precision
//           once) and the state injection of k_syrk (inject_state).  All arithmetic in fp64.
//   k_aid<S, NM, true> (msckf_b200_aid_stack_update_fde): the same kernel with fault detection and exclusion over the stack's
//           items.  A degenerate item is dropped instead of ending the member; rounds over the kept set A rebuild S_AA from
//           H P (kept in Wt until the update) and R, factor it, gate NIS_A on chi2[d_A - 1] and, while it fails, exclude the
//           item with the largest t_j / chi2[d_j - 1] (t_j = y_j^T B_j^-1 y_j, y = S_AA^-1 r, B_j = (S_AA^-1)_jj; one warp per
//           item).  The update of the final A runs the arithmetic of the plain kernel on those rows, in their order.
// One CTA per member, one launch for everything; one body for a single filter (NM = 1) and a device batch (NM =
// kBatchMembers), like k_nees.  W^T and dx live in dynamic shared memory where they fit, else in a per-member global workspace.
#pragma once
#include "common.cuh"
#include "nees_kernels.cuh"
#include "state_kernels.cuh"

namespace mb {

// the models of msckf_b200_aid_model (include/msckf_b200.h)
enum AidModel {
  kAidVelocity = 0, kAidPosition = 1, kAidPose = 2, kAidClonePose = 3, kAidLinear = 4, kAidBodyVelocity = 5, kAidRelativePose = 6,
  kAidAntennaPosition = 7, kAidCloneAntennaPosition = 8, kAidHeading = 9, kAidCloneHeading = 10,
  kAidRange = 11, kAidCloneRange = 12, kAidPlaneRange = 13, kAidClonePlaneRange = 14
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

// bytes of W^T and dx of one member (in shared or global memory)
__host__ __device__ constexpr size_t aid_ws_bytes(int n, int m) { return sizeof(double) * (size_t)n * (m + 1); }

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
// Returns 0 when the rows are formed.
// (Out of line, with the item by value: inlined into k_aid<double, 1>, this code made ptxas spill.)
template <class S>
__device__ __noinline__ int aid_item_rows(const AidItem it, const double* z, const DevState<S>* st, const S* poses,
                                             double* r, int (*col)[kAidNnz], double (*coef)[kAidNnz], int* nnz) {
  const int r0 = it.row;
  if (it.model == kAidVelocity || it.model == kAidPosition) {
    const S* x = it.model == kAidVelocity ? st->v_I_G : st->p_I_G;
    for (int i = 0; i < 3; ++i) {
      r[r0 + i] = z[i] - (double)x[i];
      col[r0 + i][0] = (it.model == kAidVelocity ? 6 : 12) + i; coef[r0 + i][0] = 1.0; nnz[r0 + i] = 1;
    }
  } else if (it.model == kAidPose || it.model == kAidClonePose) {  // [dtheta(q_z, q_est); z_p - p_est]
    const bool imu = it.model == kAidPose;
    const S* q = imu ? st->q_IG : poses + kPoseStride * it.a;
    const S* p = imu ? st->p_I_G : poses + kPoseStride * it.a + 4;
    nees_quat_error(z + 3, q, r + r0);
    for (int i = 0; i < 3; ++i) r[r0 + 3 + i] = z[i] - (double)p[i];
    for (int i = 0; i < 6; ++i) {
      col[r0 + i][0] = imu ? (i < 3 ? i : 9 + i) : 15 + 6 * it.a + i; coef[r0 + i][0] = 1.0; nnz[r0 + i] = 1;
    }
  } else if (it.model == kAidBodyVelocity) {
    const double q[4] = {(double)st->q_IG[0], (double)st->q_IG[1], (double)st->q_IG[2], (double)st->q_IG[3]};
    double C[9], v[3];
    quat_to_rot(q, C);
    for (int j = 0; j < 3; ++j) v[j] = C[3 * j] * (double)st->v_I_G[0] + C[3 * j + 1] * (double)st->v_I_G[1] + C[3 * j + 2] * (double)st->v_I_G[2];
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
  } else if (it.model >= kAidAntennaPosition) {  // the antenna positions, headings and ranges, of the IMU or of clone a
    const bool clone = it.model == kAidCloneAntennaPosition || it.model == kAidCloneHeading || it.model == kAidCloneRange ||
                       it.model == kAidClonePlaneRange;
    const bool heading = it.model == kAidHeading || it.model == kAidCloneHeading;
    const bool range = it.model == kAidRange || it.model == kAidCloneRange;
    const bool plane = it.model == kAidPlaneRange || it.model == kAidClonePlaneRange;
    const S* Q = clone ? poses + kPoseStride * it.a : st->q_IG;
    const double q[4] = {(double)Q[0], (double)Q[1], (double)Q[2], (double)Q[3]};
    const double* l = heading ? z + 1 : range ? z + 4 : plane ? z + 2 : z + 3;  // the lever arm or the axis, in the body frame
    const int c0 = clone ? 15 + 6 * it.a : 0;   // the pose's dtheta
    const S* p = clone ? poses + kPoseStride * it.a + 4 : st->p_I_G;
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
    const S* A = poses + kPoseStride * it.a;
    const S* B = poses + kPoseStride * it.b;
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

template <class S, int NM, bool FDE = false>
__global__ void __launch_bounds__(kAidThreads) k_aid(const Members<AidArgs<S>, NM> a) {
  extern __shared__ double aid_dyn[];
  const int f = NM == 1 ? 0 : blockIdx.x;
  DevState<S>* const st = a.m[f].st;
  S* __restrict__ const P = a.m[f].P;
  S* const poses = a.m[f].poses;
  const double* __restrict__ const in = a.m[f].in;
  AidOut* const out = a.m[f].out;
  const int ldp = a.m[f].ldp, M = a.m[f].M, m = a.m[f].m, n = 15 + 6 * M;
  const bool lin = a.m[f].item[0].model == kAidLinear;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* const Wt = a.m[f].ws ? a.m[f].ws : aid_dyn;  // [n][m]: column c of H P, then of W = L^-1 H P
  double* const dx = Wt + (size_t)n * m;
  const double* __restrict__ const R = in + kAidZ;
  const double* __restrict__ const H = R + m * m;      // LINEAR only
  __shared__ double L[kAidMaxRows + 1][kAidMaxRows + 1];  // S = L L^T (lower); row m: r, then y = L^-1 r
  __shared__ double idg[kAidMaxRows];
  __shared__ double part[kAidThreads / 32];
  __shared__ int s_col[kAidMaxRows][kAidNnz];             // the model rows of H: (state index, coefficient) pairs
  __shared__ double s_coef[kAidMaxRows][kAidNnz];
  __shared__ int s_nnz[kAidMaxRows];
  __shared__ int s_nv, s_apply, s_bad;

  // ---- residual (fp64) and the rows of H, one thread per item
  int degenerate = 0;
  int mA = m;  // the rows of the update (FDE: of the kept items, the first mA entries of each Wt row; y in row mA of L)
  if constexpr (FDE) {  // r stays in s_r for every round; a degenerate item is dropped from A (its rows are never read)
    __shared__ double s_r[kAidMaxRows];
    __shared__ int s_ri[kAidMaxRows], s_c0[kAidMaxItems];  // row k of S_AA is stack row s_ri[k]; item w's first row in S_AA
    __shared__ double s_t[kAidMaxItems], s_blk[kAidMaxItems][42];  // t_j of the round; a warp's d x d block and vector
    __shared__ unsigned s_A;  // the items of A (bits)
    __shared__ int s_mA, s_done;
    AidFdeOut* const fo = reinterpret_cast<AidFdeOut*>(out);
    const double* __restrict__ const chi2 = R + m * m;
    const int n_items = a.m[f].n_items;
    const auto rows_of = [&](int k) { return (k + 1 < n_items ? a.m[f].item[k + 1].row : m) - a.m[f].item[k].row; };
    if (t < n_items) {
      degenerate = aid_item_rows(a.m[f].item[t], in + kAidItemZ * t, st, poses, s_r, s_col, s_coef, s_nnz);
      fo->item[t] = {__longlong_as_double(0x7ff8000000000000ll), __longlong_as_double(0x7ff8000000000000ll), degenerate ? 2 : 3, -1};
    }
    const unsigned keep = __ballot_sync(0xffffffffu, t < n_items && !degenerate);
    if (t == 0) { s_A = keep; s_mA = 0; }
    __syncthreads();
    if (s_A == 0u) {  // every item degenerate: nothing is written
      if (t == 0) {
        out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
        out->dof = 0; out->applied = 0; out->status = 2; out->numeric = 0;
        fo->outcome = -1; fo->n_excluded = 0;
      }
      return;
    }
    // H P of the kept rows, stored transposed (stride m): kept until the update, S_AA of every round is formed from it
    for (int idx = t; idx < m * n; idx += kAidThreads) {
      const int i = idx / n, c = idx - i * n;
      int k = 0;
      while (k + 1 < n_items && a.m[f].item[k + 1].row <= i) ++k;
      if (!((s_A >> k) & 1u)) continue;
      double s = s_coef[i][0] * (double)P[(size_t)s_col[i][0] * ldp + c];
      for (int q = 1; q < s_nnz[i]; ++q) s += s_coef[i][q] * (double)P[(size_t)s_col[i][q] * ldp + c];
      Wt[(size_t)c * m + i] = s;
    }
    __syncthreads();
    // each kept item alone against the prior: r_j^T S_jj^-1 r_j (warp j, lane 0)
    if (warp < n_items && lane == 0 && ((s_A >> warp) & 1u)) {
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
    const int max_exclude = (int)R[m * m + kAidMaxRows];
    int outcome = -1, n_exc = 0;
    for (int round = 0;; ++round) {
      // ---- S_AA (lower) from H P and R with the expression of the plain kernel, r_A as row m_A
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
      const int ma = s_mA;
      for (int idx = t; idx < ma * ma; idx += kAidThreads) {
        const int i = idx / ma, j = idx - i * ma;
        if (j > i) continue;
        const int ri = s_ri[i], rj = s_ri[j];
        double s = s_coef[rj][0] * Wt[(size_t)s_col[rj][0] * m + ri];
        for (int q = 1; q < s_nnz[rj]; ++q) s += s_coef[rj][q] * Wt[(size_t)s_col[rj][q] * m + ri];
        L[i][j] = s + R[ri * m + rj];
      }
      if (t < ma) L[ma][t] = s_r[s_ri[t]];
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
      if (s_nv < ma) {  // S_AA not positive definite: nothing is written
        if (t == 0) {
          out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
          out->dof = ma; out->applied = 0; out->status = 1; out->numeric = 0;
          fo->outcome = -1; fo->n_excluded = n_exc;
        }
        return;
      }
      if (t == 0) {
        double g = 0.0;
        for (int i = 0; i < ma; ++i) g += L[ma][i] * L[ma][i];
        out->nis = g; out->dof = ma; out->status = 0;
        s_done = !(g > chi2[ma - 1]) ? (n_exc ? 1 : 0) : n_exc >= max_exclude ? 2 : __popc(s_A) == 1 ? 3 : -1;
      }
      __syncthreads();
      if (s_done >= 0) { outcome = s_done; break; }
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
      if (s_done >= 0) { outcome = s_done; break; }
      ++n_exc;
    }
    if (t == 0) {
      fo->outcome = outcome; fo->n_excluded = n_exc;
      for (int w = 0; w < n_items; ++w)
        if ((s_A >> w) & 1u) fo->item[w].state = outcome <= 1 ? 0 : 3;
      out->applied = outcome <= 1;
      s_apply = outcome <= 1;
      s_bad = 0;
      if (!s_apply) { out->dx_norm = 0.0; out->numeric = 0; }
    }
    __syncthreads();
    if (!s_apply) return;
    // ---- W = L^-1 H P over the rows of A, gathered in order into the first m_A entries of each Wt row
    mA = s_mA;
    for (int r = warp; r < n; r += kAidThreads / 32) {
      double* row = Wt + (size_t)r * m;
      const double x0 = lane < mA ? row[s_ri[lane]] : 0.0;
      __syncwarp();
      const double x = warp_row_solve(x0, L, idg, mA, lane);
      if (lane < mA) row[lane] = x;
    }
    __syncthreads();
  } else {  // the plain single-model, LINEAR and stacked update (left at its original indentation)
  if (lin) {
    if (t < m) L[m][t] = in[t];
  } else if (t < a.m[f].n_items) {
    degenerate = aid_item_rows(a.m[f].item[t], in + kAidItemZ * t, st, poses, &L[m][0], s_col, s_coef, s_nnz);
  }
  if (__syncthreads_or(degenerate)) {  // a heading whose yaw or a range whose prediction is undefined: nothing is written
    if (t == 0) {
      out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
      out->dof = m; out->applied = 0; out->status = 2; out->numeric = 0;
    }
    return;
  }
  // ---- H P, stored transposed: Wt[c][i] = (H P)[i][c]
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
      double s = s_coef[i][0] * (double)P[(size_t)s_col[i][0] * ldp + c];  // (exact for the one-coefficient rows)
      for (int k = 1; k < s_nnz[i]; ++k) s += s_coef[i][k] * (double)P[(size_t)s_col[i][k] * ldp + c];
      Wt[(size_t)c * m + i] = s;
    }
  }
  __syncthreads();
  // ---- S = H P H^T + R, lower triangle (only R's lower triangle is read)
  for (int idx = t; idx < m * m; idx += kAidThreads) {
    const int i = idx / m, j = idx - i * m;
    if (j > i) continue;
    double s;
    if (lin) {
      const double* h = H + (size_t)j * n;
      s = 0.0;
      for (int k = 0; k < n; ++k) s += Wt[(size_t)k * m + i] * h[k];
    } else {
      s = s_coef[j][0] * Wt[(size_t)s_col[j][0] * m + i];
      for (int k = 1; k < s_nnz[j]; ++k) s += s_coef[j][k] * Wt[(size_t)s_col[j][k] * m + i];
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
  }  // (FDE)
  // ---- dx = W^T y, and P <- P - W^T W (lower triangle in fp64, written to both halves: exactly symmetric)
  double nn = 0.0;
  for (int c = t; c < n; c += kAidThreads) {
    const double* w = Wt + (size_t)c * m;
    double s = 0.0;
    for (int i = 0; i < mA; ++i) s += w[i] * L[mA][i];
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
    for (int i = 0; i < mA; ++i) v += wr[i] * wc[i];
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
