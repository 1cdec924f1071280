// msckf_mono_b200/csrc/landmark_kernels.cuh
// Image observations of landmarks whose position is known (a prior map, surveyed markers, relocalisation matches), fused into
// the device-resident filter (msckf_b200_landmark_update / _batch_landmark_update).  Observation i = (clone k_i, z_i, p_L,i):
// p_C = C(q_CG,k) (p_L - p_C_G,k), z^ = p_C[0:2] / p_C[2], r_i = z_i - z^ (calcResidual, msckf.h:960-978), and the 2 x 6 block
// X_i = [J_i [p_C]x, -J_i C] over the clone's [dtheta, dp] (msckf.h:929-936) WITHOUT the observability projection of
// msckf.h:938-944: that projection removes global position and yaw, which a known landmark observes.  All arithmetic in fp64.
//   k_lmk_clone    : one CTA per (touched clone, member).  Residual, per-observation gate gamma_i = r^T (X P_kk X^T + R)^-1 r
//                    and flag, rows whitened by R = L_R L_R^T, then a Householder QR (one warp) of the clone's used rows
//                    [X~ | r~] (2a x 7): q = min(2a, 6) rows [T_k | rho_k] and the leftover e_k^2 go to the member's workspace.
//   k_lmk_gain     : one CTA per member.  T P (rows of T in window order), S = T P T^T + I, and one blocked Cholesky
//                    (cta_bordered_chol) of [S ; (T P)^T ; rho^T]: the extra rows end as W^T = (L^-1 T P)^T and y = L^-1 rho.
//                    NIS = |y|^2 + sum_k e_k^2 (the NIS of the dense stacked system).
//   k_lmk_downdate : 32 x 32 tiles of the lower triangle of P - W^T W (fp64, rounded once, both halves written, in place) and
//                    dx = W^T y on the diagonal tiles; the last tile of a member (ticket counter) runs the state injection.
// Iterated form (max_iter >= 2, an IEKF): after k_lmk_gain, k_lmk_step forms delta_{i+1} = W^T y and the iterate clone poses
// x^ [+] delta_{i+1} (fp64); k_lmk_clone<..., true> relinearises there with linearisation 0's flags, adding X~ e_k (e_k: delta_i of
// clone k) to the whitened residual, and k_lmk_gain<..., true> refactors against the same prior P without touching the NIS.
// k_lmk_downdate then applies the last W, y.  P and the resident state are not written before the downdate.
// Map uncertainty (MAP: Sigma_L given, DESIGN.md 4.12): each landmark's position error dp_l ~ N(0, Sigma_l) is marginalised
// over its observations in the call.  k_lmk_clone<..., MAP> gates with X P_kk X^T + F Sigma F^T + R (F = J C) and whitens a
// one-clone landmark by R + F Sigma F^T before the clone's QR; k_lmk_set eliminates the landmarks seen from 2 .. 8 clones and
// compresses each group of one clone set; k_lmk_gain<..., MAP> gathers a row over its group's clone blocks.  A chunk with a
// Sigma_L member launches clone, set, gain (and step, clone, set, gain per extra linearisation), then the same downdate.
// One body for a single filter (NM = 1) and a device batch (NM = kBatchMembers), like k_aid.  Each member's arithmetic depends
// only on its own inputs: a batch equals single calls bit for bit.
#pragma once
#include "common.cuh"
#include "state_kernels.cuh"

#include <type_traits>

namespace mb {

constexpr int kLmkMaxPerClone = 256;  // observations of one clone in one call (2 x 256 rows of 7 doubles in shared memory)
constexpr int kLmkMaxObs = 4096;      // observations of one member in one call
constexpr int kLmkMaxIter = 16;       // linearisations of the iterated form
constexpr int kLmkThreads = 256;
constexpr int kLmkSlot = 48;          // doubles per touched clone: T [6][6], rho [6], e^2, used, q
constexpr int kLmkNB = 32;            // tile size of the downdate (tile_dot32's)

// per-member result; every field but numeric is msckf_b200_landmark_result's, at its offset
struct LmkOut {
  double nis, dx_norm;
  int dof, rows, used, applied, status;
  int iterations, converged;  // written by the iterated form only (the host fills them for max_iter <= 1)
  int numeric;                // a non-finite dx or P entry was written
  double step;
};
// per-member control words in the workspace (k_lmk_gain -> k_lmk_downdate)
struct LmkCtl {
  int m, apply, bad;
  unsigned ticket;  // tiles of k_lmk_downdate done (reset by k_lmk_gain and by the last tile)
};

template <class S>
struct LmkArgs {
  DevState<S>* st;
  S* P;
  S* poses;
  const double* obs;  // [n_obs][5]: z (2), p_L (3), grouped by clone in window order
  const int* grp;     // [G][3]: clone, first observation, count
  double* slot;       // [G][kLmkSlot]
  double* A;          // [ld + n + 1][ld]: S (lower), then (T P)^T -> W^T, then rho -> y
  double* dx;         // [n]
  LmkCtl* ctl;
  LmkOut* out;
  double* gamma;      // [n_obs] (packed order)
  int* flag;          // [n_obs]
  double R[3];        // uu, uv, vv (use_R), else the filter's diag(u_var, v_var)
  double chi2;        // > 0: per-observation gate
  int ldp, M, G, ld, ntiles, use_R;
};
static_assert(sizeof(Members<LmkArgs<double>, kBatchMembers>) <= 32764, "the landmark kernels' batched arguments exceed the parameter limit");

// the iterated form's per-member control words (k_lmk_step writes them at its first launch of a call)
struct alignas(8) LmkIt {
  int done;  // converged, stopped or out of iterations: every later iteration kernel returns at once
  int stop;  // a used observation is behind the camera or not finite at the iterate (k_lmk_clone<..., true>)
};
// done or stop, in one load (two loads of the words cost k_lmk_gain<..., 32, true> an 8-byte spill)
__device__ __forceinline__ bool lmk_it_ended(const LmkIt* ic) {
  const int2 w = __ldcg(reinterpret_cast<const int2*>(ic));
  return (w.x | w.y) != 0;
}
template <class S>
struct LmkItArgs : LmkArgs<S> {
  double* xi;    // [M][7] iterate clone poses x^ [+] delta_i: q (x, y, z, w), p_C_G
  double* d;     // [n] delta_i
  LmkIt* it;
  double tol;    // stop when max |delta_{i+1} - delta_i| <= tol
  int max_iter;  // linearisations; <= 1: the member does not iterate and every iteration kernel returns at once
};
static_assert(sizeof(Members<LmkItArgs<double>, kBatchMembers>) <= 32764, "the iterated landmark kernels' arguments exceed the parameter limit");
// Map uncertainty (MAP, Sigma_L given): a landmark seen from one clone (so by one observation) is whitened with
// R + F Sigma F^T inside k_lmk_clone; the observations of a landmark seen from c >= 2 clones leave k_lmk_clone as row pairs,
// whitened by L_R, and k_lmk_set marginalises each landmark and compresses each group of landmarks with one clone set.
constexpr int kLmkMapClones = 8;                       // clones that see one landmark
constexpr int kLmkMaxPerSet = 256;                     // observations of one clone-set group
constexpr int kLmkMaxSets = 256;                       // clone-set groups of one member
constexpr int kLmkMaxRows = 6 * kMaxKeep;              // rows of the compressed system (k_lmk_gain's row table)
constexpr int kLmkSetLd = 6 * kLmkMapClones;           // T_g row stride
constexpr int kLmkSetSlot = kLmkSetLd * (kLmkSetLd + 1) + 8;  // doubles per group: T [48][48], rho [48], e^2, used, q
constexpr int kLmkPair = 16;                           // doubles per row pair: [X~ | r~] (2 x 7), flag
constexpr int kLmkSetDesc = 16;                        // ints per group: c, landmarks, first pair, first landmark,
                                                       // E offset, B offset, 2 spare, clones [8] (window order)
template <class S>
struct LmkMapArgs : LmkItArgs<S> {
  const double* sig;   // [n_obs][6] Sigma of each observation's landmark (packed order), or NULL: an exact-map member
  const int* wrow;     // [n_obs] the observation's pair (a landmark seen from >= 2 clones), or -1
  const int* sdesc;    // [H][kLmkSetDesc]
  const double* lsig;  // [landmarks of the groups][6] Sigma, group by group
  double* pair;        // [pairs][kLmkPair] (k_lmk_clone -> k_lmk_set)
  double* E;           // per landmark [3 + 2c][6c + 4]: prior rows, then its used rows [X~ | r~ | F~]
  double* B;           // per group [2 obs][6c + 1]: the marginalised rows [X~' | r~']
  double* sslot;       // [H][kLmkSetSlot]
  int H;
};
static_assert(sizeof(Members<LmkMapArgs<double>, kBatchMembers>) <= 32764, "the map landmark kernels' arguments exceed the parameter limit");
template <class S, bool IT, bool MAP = false>
using LmkArgsT = std::conditional_t<MAP, LmkMapArgs<S>, std::conditional_t<IT, LmkItArgs<S>, LmkArgs<S>>>;

// Consensus on the map matches (DESIGN.md 4.17, consensus_kernels.cuh): k_lmk_hyp scores sampled 4-dof corrections of the
// window, k_lmk_cons picks and refits the best and pre-sets flag 3 on the outliers, which k_lmk_clone<..., CONS> keeps.
constexpr int kLmkMaxHyp = 1024;  // hypotheses of one member in one call
struct LmkHyp {
  double th[4];  // psi, t
  int count;     // inliers (0 when not valid)
  int valid;
};
// per-member consensus result; msckf_b200_landmark_consensus_result's fields at their offsets
struct LmkConsOut {
  int status, inliers, best, valid, refit;
  double yaw, t[3], pivot[3];
};
template <class S>
struct LmkConsArgs : LmkMapArgs<S> {
  const int* pairs;  // [nh][2] the sampled observations (packed order)
  const int* ogrp;   // [n_obs] each observation's group (touched clone) in grp
  LmkHyp* hyp;       // [nh]
  LmkConsOut* cres;
  int* score;        // [nh] out: each hypothesis's inliers, or -1 when it is not valid
  double thresh;     // inlier when depth > 0 and (z - z^)^T R^-1 (z - z^) <= thresh
  int n_obs, nh, min_inl;
  int cons;          // 0: the member runs no consensus (its consensus kernels return at once, its flags are not pre-set)
};
static_assert(sizeof(Members<LmkConsArgs<double>, kBatchMembers>) <= 32764, "the consensus kernels' arguments exceed the parameter limit");
template <class S, bool IT, bool MAP, bool CONS>
using LmkArgsC = std::conditional_t<CONS, LmkConsArgs<S>, LmkArgsT<S, IT, MAP>>;

__host__ __device__ constexpr int lmk_tiles(int n) { return ((n + kLmkNB - 1) / kLmkNB) * ((n + kLmkNB - 1) / kLmkNB + 1) / 2; }

// one observation against clone pose (C, p_C_G): rows [X | r] (2 x 7), flag (0 used, 1 gated out, 2 behind the camera or not
// finite) and gamma = r^T (X P_kk X^T + R)^-1 r (NaN for flag 2)
__device__ __forceinline__ double lmk_obs(const double* o, const double* Cr, const double* pc, const double (*Pk)[6], const double* Rm,
                                          double chi2, double (&row)[2][7], int& fg) {
  const double d[3] = {o[2] - pc[0], o[3] - pc[1], o[4] - pc[2]};
  double p[3];
  for (int i = 0; i < 3; ++i) p[i] = Cr[3 * i] * d[0] + Cr[3 * i + 1] * d[1] + Cr[3 * i + 2] * d[2];
  const double zh0 = p[0] / p[2], zh1 = p[1] / p[2];
  fg = 2;
  if (!(p[2] > 0.0 && isfinite(zh0) && isfinite(zh1))) return __longlong_as_double(0x7ff8000000000000ll);
  const double iz = 1.0 / p[2];
  const double J[2][3] = {{iz, 0.0, -zh0 * iz}, {0.0, iz, -zh1 * iz}};
  const double sk[3][3] = {{0.0, -p[2], p[1]}, {p[2], 0.0, -p[0]}, {-p[1], p[0], 0.0}};
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) {
      row[r][c] = J[r][0] * sk[0][c] + J[r][1] * sk[1][c] + J[r][2] * sk[2][c];
      row[r][3 + c] = -(J[r][0] * Cr[c] + J[r][1] * Cr[3 + c] + J[r][2] * Cr[6 + c]);
    }
  row[0][6] = o[0] - zh0;
  row[1][6] = o[1] - zh1;
  double s00 = Rm[0], s10 = Rm[1], s11 = Rm[2];
  for (int c = 0; c < 6; ++c) {
    double x0 = 0.0, x1 = 0.0;
    for (int j = 0; j < 6; ++j) { x0 += row[0][j] * Pk[j][c]; x1 += row[1][j] * Pk[j][c]; }
    s00 += x0 * row[0][c];
    s10 += x1 * row[0][c];
    s11 += x1 * row[1][c];
  }
  const double r0 = row[0][6], r1 = row[1][6];
  const double gam = (s11 * r0 * r0 - 2.0 * s10 * r0 * r1 + s00 * r1 * r1) / (s00 * s11 - s10 * s10);
  fg = (chi2 > 0.0 && gam > chi2) ? 1 : 0;
  return gam;
}

// Ri += F Sigma F^T with F = J C, the observation's block over the landmark position (= -X[:, 3:6]); Ri unchanged behind the
// camera (lmk_obs flags that).  sg: Sigma's lower triangle xx, yx, yy, zx, zy, zz.
__device__ __forceinline__ void lmk_map_R(const double* o, const double* Cr, const double* pc, const double* sg, double (&Ri)[3]) {
  const double d[3] = {o[2] - pc[0], o[3] - pc[1], o[4] - pc[2]};
  double p[3];
  for (int i = 0; i < 3; ++i) p[i] = Cr[3 * i] * d[0] + Cr[3 * i + 1] * d[1] + Cr[3 * i + 2] * d[2];
  if (!(p[2] > 0.0)) return;
  const double iz = 1.0 / p[2];
  const double J[2][3] = {{iz, 0.0, -p[0] / p[2] * iz}, {0.0, iz, -p[1] / p[2] * iz}};
  const double Sm[3][3] = {{sg[0], sg[1], sg[3]}, {sg[1], sg[2], sg[4]}, {sg[3], sg[4], sg[5]}};
  double F[2][3], FS[2][3];
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) F[r][c] = J[r][0] * Cr[c] + J[r][1] * Cr[3 + c] + J[r][2] * Cr[6 + c];
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) FS[r][c] = F[r][0] * Sm[0][c] + F[r][1] * Sm[1][c] + F[r][2] * Sm[2][c];
  Ri[0] += FS[0][0] * F[0][0] + FS[0][1] * F[0][1] + FS[0][2] * F[0][2];
  Ri[1] += FS[1][0] * F[0][0] + FS[1][1] * F[0][1] + FS[1][2] * F[0][2];
  Ri[2] += FS[1][0] * F[1][0] + FS[1][1] * F[1][1] + FS[1][2] * F[1][2];
}

// IT: the iterate form.  The clone pose comes from the iterate table, the flags are linearisation 0's (gamma and flag are not
// written), X~ e_k is added to the whitened residual, and a used observation that fails at the iterate raises the stop word.
// MAP: gamma includes F Sigma F^T; a one-clone landmark's rows are whitened by the Cholesky factor of R + F Sigma F^T (exact
// marginalisation of its position), and the rows of a landmark seen from several clones go to its pair (whitened by L_R, with
// the flag) instead of the clone's QR.  A member without Sigma runs the exact-map arithmetic.
// CONS (linearisation 0 only): a consensus member's observation pre-set to flag 3 by k_lmk_cons keeps it unless it is flag 2;
// gamma is written as without consensus.
template <class S, int NM, bool IT = false, bool MAP = false, bool CONS = false>
__global__ void __launch_bounds__(kLmkThreads) k_lmk_clone(const Members<LmkArgsC<S, IT, MAP, CONS>, NM> a) {
  static_assert(!(CONS && IT), "consensus pre-sets linearisation 0's flags only");
  const int f = NM == 1 ? 0 : blockIdx.y, g = blockIdx.x;
  if constexpr (IT) {
    if (a.m[f].max_iter <= 1 || lmk_it_ended(a.m[f].it)) return;
  }
  if (g >= a.m[f].G) return;
  const S* __restrict__ const P = a.m[f].P;
  const int ldp = a.m[f].ldp, t = threadIdx.x, lane = t & 31;
  const int k = a.m[f].grp[3 * g], i0 = a.m[f].grp[3 * g + 1], cnt = a.m[f].grp[3 * g + 2];
  const double* __restrict__ const obs = a.m[f].obs + 5 * (size_t)(i0 + t);
  const double chi2 = a.m[f].chi2;
  __shared__ double Q[2 * kLmkMaxPerClone][7];  // used rows [X~ | r~], input order, then R and the Householder vectors
  __shared__ double Pk[6][6], Cr[9], pc[3], LR[3], Rm[3];
  __shared__ int fl[kLmkMaxPerClone], pos[kLmkMaxPerClone], s_used;
  __shared__ double ek[IT ? 6 : 1];

  if (t < 36) Pk[t / 6][t % 6] = (double)P[(size_t)(15 + 6 * k + t / 6) * ldp + 15 + 6 * k + t % 6];
  if constexpr (IT) {
    if (t >= 64 && t < 70) ek[t - 64] = a.m[f].d[15 + 6 * k + t - 64];
  }
  if (t == 0) {
    if constexpr (IT) {
      const double* x = a.m[f].xi + 7 * k;
      quat_to_rot(x, Cr);
      pc[0] = x[4]; pc[1] = x[5]; pc[2] = x[6];
    } else {
      const S* ps = a.m[f].poses + kPoseStride * k;
      const double q[4] = {(double)ps[0], (double)ps[1], (double)ps[2], (double)ps[3]};
      quat_to_rot(q, Cr);
      pc[0] = (double)ps[4]; pc[1] = (double)ps[5]; pc[2] = (double)ps[6];
    }
    if (a.m[f].use_R) {
      Rm[0] = a.m[f].R[0]; Rm[1] = a.m[f].R[1]; Rm[2] = a.m[f].R[2];
    } else {
      Rm[0] = (double)a.m[f].st->u_var; Rm[1] = 0.0; Rm[2] = (double)a.m[f].st->v_var;
    }
    LR[0] = sqrt(Rm[0]);
    LR[1] = Rm[1] / LR[0];
    LR[2] = sqrt(Rm[2] - LR[1] * LR[1]);
  }
  __syncthreads();
  // ---- per observation: residual, Jacobian block, gate; then the used rows, compacted in input order (recomputed rather than
  // kept in registers across the compaction)
  double row[2][7];
  int fg = 2;
  // MAP: R + F Sigma F^T of a member with Sigma (sg), and the observation's pair (wr >= 0: a landmark seen from >= 2 clones)
  [[maybe_unused]] double Ri[3];
  [[maybe_unused]] const double* sg = nullptr;
  int wr = -1;
  if constexpr (MAP) {
    Ri[0] = Rm[0]; Ri[1] = Rm[1]; Ri[2] = Rm[2];
    sg = a.m[f].sig;
    wr = sg && t < cnt ? a.m[f].wrow[i0 + t] : -1;
  }
  const double* const Ro = MAP ? Ri : Rm;  // the gate's observation noise
  if (t < cnt) {
    [[maybe_unused]] int pre = 0;  // CONS: k_lmk_cons's flag
    if constexpr (CONS) {
      if (a.m[f].cons) pre = a.m[f].flag[i0 + t];
    }
    if constexpr (MAP) {
      if (sg) lmk_map_R(obs, Cr, pc, sg + 6 * (size_t)(i0 + t), Ri);
    }
    const double gam = lmk_obs(obs, Cr, pc, Pk, Ro, chi2, row, fg);
    if constexpr (IT) {
      const int f0 = a.m[f].flag[i0 + t];  // linearisation 0's
      if (f0 == 0 && fg == 2) a.m[f].it->stop = 1;
      fg = f0;
    } else {
      if constexpr (CONS) {
        if (pre == 3 && fg != 2) fg = 3;
      }
      a.m[f].gamma[i0 + t] = gam;
      a.m[f].flag[i0 + t] = fg;
    }
    if constexpr (MAP) {
      if (wr >= 0) a.m[f].pair[(size_t)kLmkPair * wr + 14] = (double)fg;
    }
    fl[t] = wr >= 0 && fg == 0 ? 3 : fg;  // 3: used, in a pair
  }
  __syncthreads();
  if (t == 0) {
    int u = 0;
    for (int i = 0; i < cnt; ++i) { pos[i] = u; u += fl[i] == 0; }
    s_used = u;
  }
  __syncthreads();
  if (t < cnt && fg == 0) {
    lmk_obs(obs, Cr, pc, Pk, Ro, chi2, row, fg);
    [[maybe_unused]] double Li[3];  // MAP: L_R, or the Cholesky factor of Ri for a one-clone landmark
    if constexpr (MAP) {
      Li[0] = LR[0]; Li[1] = LR[1]; Li[2] = LR[2];
      if (sg && wr < 0) { Li[0] = sqrt(Ri[0]); Li[1] = Ri[1] / Li[0]; Li[2] = sqrt(Ri[2] - Li[1] * Li[1]); }
    }
    const double* const L = MAP ? Li : LR;
    // whiten in place: L^-1 [X | r].  The exact map's single linearisation changes the rows no further and stores each
    // column as it is whitened (storing after the loop costs its schedule a few instructions); the other forms store below.
    for (int c = 0; c < 7; ++c) {
      row[0][c] /= L[0];
      if constexpr (!IT && !MAP) Q[2 * pos[t]][c] = row[0][c];
      row[1][c] = (row[1][c] - row[0][c] * L[1]) / L[2];
      if constexpr (!IT && !MAP) Q[2 * pos[t] + 1][c] = row[1][c];
    }
    if constexpr (IT) {  // r~ + X~ e_k
      for (int c = 0; c < 6; ++c) { row[0][6] += row[0][c] * ek[c]; row[1][6] += row[1][c] * ek[c]; }
    }
    if (wr >= 0) {
      if constexpr (MAP) {
        double* pr = a.m[f].pair + (size_t)kLmkPair * wr;
        for (int c = 0; c < 7; ++c) { pr[c] = row[0][c]; pr[7 + c] = row[1][c]; }
      }
    } else if constexpr (IT || MAP) {
      for (int c = 0; c < 7; ++c) { Q[2 * pos[t]][c] = row[0][c]; Q[2 * pos[t] + 1][c] = row[1][c]; }
    }
  }
  __syncthreads();
  // ---- Householder QR of the used rows (one warp): R's first q rows are [T_k | rho_k], rows q.. of column 6 give e_k^2
  const int nr = 2 * s_used, q = min(nr, 6);
  if (t < 32) {
    for (int j = 0; j < q; ++j) {
      double s = 0.0;
      for (int r = j + lane; r < nr; r += 32) s += Q[r][j] * Q[r][j];
      s = warp_sum(s);
      const double x0 = Q[j][j];
      __syncwarp();
      if (s > 0.0) {
        const double al = x0 >= 0.0 ? -sqrt(s) : sqrt(s);
        const double tau = 1.0 / (s - al * x0);
        if (lane == 0) Q[j][j] = x0 - al;
        __syncwarp();
        for (int c = j + 1; c < 7; ++c) {
          double d = 0.0;
          for (int r = j + lane; r < nr; r += 32) d += Q[r][j] * Q[r][c];
          d = tau * warp_sum(d);
          for (int r = j + lane; r < nr; r += 32) Q[r][c] -= d * Q[r][j];
        }
        __syncwarp();
        if (lane == 0) Q[j][j] = al;
      }
      __syncwarp();
    }
    double e2 = 0.0;
    for (int r = q + lane; r < nr; r += 32) e2 += Q[r][6] * Q[r][6];
    e2 = warp_sum(e2);
    double* sl = a.m[f].slot + (size_t)kLmkSlot * g;
    for (int i = lane; i < 42; i += 32) {
      const int r = i / 7, c = i - 7 * r;
      const double v = (r < q && c >= r) ? Q[r][c] : 0.0;
      if (c < 6) sl[6 * r + c] = v;
      else sl[36 + r] = v;
    }
    if (lane == 0) { sl[42] = e2; sl[43] = (double)s_used; sl[44] = (double)q; }
  }
}

// One CTA per (clone-set group h, member): for each landmark of the group (one warp each), the 3 prior rows [0 | L_S^-1 | 0]
// (Sigma = L_S L_S^T) over its used rows [X~ | r~ | F~] (F~ = -X~[:, 3:6]) and three Householder reflectors on the F columns;
// its rows below the prior rows are then [X~' | r~'] with noise I, the exact marginalisation of its position.  Then one
// Householder QR of the group's rows over its 6c clone columns: q = min(2 used, 6c) rows [T_g | rho_g] and e_g^2 to the slot.
template <class S, int NM, bool IT = false>
__global__ void __launch_bounds__(kLmkThreads, 1) k_lmk_set(const Members<LmkMapArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.y, h = blockIdx.x;
  if constexpr (IT) {
    if (a.m[f].max_iter <= 1 || lmk_it_ended(a.m[f].it)) return;
  }
  if (h >= a.m[f].H) return;
  const int* const D = a.m[f].sdesc + kLmkSetDesc * h;
  const int c = D[0], nl = D[1], p0 = D[2], l0 = D[3], w = 6 * c, ne = w + 4, nb = w + 1, er = 3 + 2 * c;
  const double* __restrict__ const pair = a.m[f].pair;
  double* const E = a.m[f].E + D[4];
  double* const B = a.m[f].B + D[5];
  const int t = threadIdx.x, lane = t & 31, wp = t >> 5;
  __shared__ int uo[kLmkMaxPerSet / 2 + 1];  // used observations before each landmark
  __shared__ double s_al, s_tau;
  __shared__ int s_ok;
  if (t == 0) {
    int u = 0;
    for (int j = 0; j < nl; ++j) {
      uo[j] = u;
      for (int b = 0; b < c; ++b) u += pair[(size_t)kLmkPair * (p0 + j * c + b) + 14] == 0.0;
    }
    uo[nl] = u;
  }
  __syncthreads();
  // ---- per landmark: each lane owns one row of E_j
  for (int j = wp; j < nl; j += kLmkThreads / 32) {
    const int nr = 3 + 2 * (uo[j + 1] - uo[j]);
    if (nr == 3) continue;
    double* const Ej = E + (size_t)j * er * ne;
    double* const er_ = Ej + (size_t)lane * ne;
    if (lane < 3) {  // row lane of L_S^-1
      const double* sg = a.m[f].lsig + 6 * (size_t)(l0 + j);
      const double L00 = sqrt(sg[0]), L10 = sg[1] / L00, L20 = sg[3] / L00;
      const double L11 = sqrt(sg[2] - L10 * L10), L21 = (sg[4] - L20 * L10) / L11;
      const double L22 = sqrt(sg[5] - L20 * L20 - L21 * L21);
      const double I00 = 1.0 / L00, I11 = 1.0 / L11, I22 = 1.0 / L22, I10 = -L10 * I00 / L11, I21 = -L21 * I11 / L22;
      const double I20 = -(L20 * I00 + L21 * I10) / L22;
      for (int col = 0; col <= w; ++col) er_[col] = 0.0;
      er_[w + 1] = lane == 0 ? I00 : lane == 1 ? I10 : I20;
      er_[w + 2] = lane == 0 ? 0.0 : lane == 1 ? I11 : I21;
      er_[w + 3] = lane == 2 ? I22 : 0.0;
    } else if (lane < nr) {  // half (lane - 3) & 1 of the ((lane - 3) >> 1)-th used observation
      int k = (lane - 3) >> 1, b = 0;
      for (;; ++b)
        if (pair[(size_t)kLmkPair * (p0 + j * c + b) + 14] == 0.0 && k-- == 0) break;
      const double* src = pair + (size_t)kLmkPair * (p0 + j * c + b) + 7 * ((lane - 3) & 1);
      for (int col = 0; col < w; ++col) er_[col] = (col / 6 == b) ? src[col - 6 * b] : 0.0;
      er_[w] = src[6];
      er_[w + 1] = -src[3]; er_[w + 2] = -src[4]; er_[w + 3] = -src[5];
    }
    __syncwarp();
    for (int jj = 0; jj < 3; ++jj) {
      const int cj = w + 1 + jj;
      double v = (lane >= jj && lane < nr) ? er_[cj] : 0.0;
      const double s = warp_sum(v * v), x0 = __shfl_sync(0xffffffffu, v, jj);
      if (!(s > 0.0)) continue;
      const double al = x0 >= 0.0 ? -sqrt(s) : sqrt(s), tau = 1.0 / (s - al * x0);
      if (lane == jj) v = x0 - al;
      for (int col = 0; col < ne; ++col) {
        if (col > w && col <= cj) continue;
        const double dd = tau * warp_sum((lane >= jj && lane < nr) ? v * er_[col] : 0.0);
        if (lane >= jj && lane < nr) er_[col] -= dd * v;
      }
    }
    if (lane >= 3 && lane < nr)
      for (int col = 0; col <= w; ++col) B[(size_t)(2 * uo[j] + lane - 3) * nb + col] = er_[col];
  }
  __syncthreads();
  // ---- Householder QR of the group's 2 used rows over 6c + 1 columns (warp 0 forms each reflector, all warps apply it)
  const int nr = 2 * uo[nl], q = min(nr, w);
  for (int j = 0; j < q; ++j) {
    if (wp == 0) {
      double s = 0.0;
      for (int r = j + lane; r < nr; r += 32) s += B[(size_t)r * nb + j] * B[(size_t)r * nb + j];
      s = warp_sum(s);
      if (lane == 0) {
        const double x0 = B[(size_t)j * nb + j];
        s_ok = s > 0.0;
        if (s > 0.0) {
          s_al = x0 >= 0.0 ? -sqrt(s) : sqrt(s);
          s_tau = 1.0 / (s - s_al * x0);
          B[(size_t)j * nb + j] = x0 - s_al;
        }
      }
    }
    __syncthreads();
    if (s_ok) {
      for (int col = j + 1 + wp; col < nb; col += kLmkThreads / 32) {
        double dd = 0.0;
        for (int r = j + lane; r < nr; r += 32) dd += B[(size_t)r * nb + j] * B[(size_t)r * nb + col];
        dd = s_tau * warp_sum(dd);
        for (int r = j + lane; r < nr; r += 32) B[(size_t)r * nb + col] -= dd * B[(size_t)r * nb + j];
      }
    }
    __syncthreads();
    if (t == 0 && s_ok) B[(size_t)j * nb + j] = s_al;
    __syncthreads();
  }
  double* const sl = a.m[f].sslot + (size_t)kLmkSetSlot * h;
  for (int i = t; i < q * w; i += kLmkThreads) {
    const int r = i / w, col = i - r * w;
    sl[kLmkSetLd * r + col] = col >= r ? B[(size_t)r * nb + col] : 0.0;
  }
  for (int r = t; r < q; r += kLmkThreads) sl[kLmkSetLd * kLmkSetLd + r] = B[(size_t)r * nb + w];
  if (wp == 0) {
    double e2 = 0.0;
    for (int r = q + lane; r < nr; r += 32) e2 += B[(size_t)r * nb + w] * B[(size_t)r * nb + w];
    e2 = warp_sum(e2);
    if (lane == 0) {
      double* tl = sl + kLmkSetLd * (kLmkSetLd + 1);
      tl[0] = e2; tl[1] = (double)uo[nl]; tl[2] = (double)q;
    }
  }
}

// the T row lr of group g of a MAP member (g < G: clone slot g, else clone-set slot g - G): its first entry, width and clones
template <class A>
__device__ __forceinline__ const double* lmk_map_row(const A& m0, const double* slot, const int* grp, int G, int g, int lr, int& w,
                                                    const int*& cl) {
  if (g < G) { w = 6; cl = grp + 3 * g; return slot + (size_t)kLmkSlot * g + 6 * lr; }
  const int* D = m0.sdesc + kLmkSetDesc * (g - G);
  w = 6 * D[0]; cl = D + 8;
  return m0.sslot + (size_t)kLmkSetSlot * (g - G) + kLmkSetLd * lr;
}

// IT: the iterate form.  A raised stop word ends the iteration with nothing written (the previous W, y stay); otherwise the
// factorisation is today's, and only apply, iterations and (S not positive definite) the status are written.
// MAP: the rows of the clone-set groups follow the clones' rows, and a T row spans its group's 6c clone columns.
template <class S, int NM, bool IT = false, bool MAP = false>
__global__ void __launch_bounds__(kLmkThreads) k_lmk_gain(const Members<LmkArgsT<S, IT, MAP>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.x;
  if constexpr (IT) {
    if (a.m[f].max_iter <= 1 || lmk_it_ended(a.m[f].it)) return;
  }
  const S* __restrict__ const P = a.m[f].P;
  double* __restrict__ const A = a.m[f].A;
  const double* __restrict__ const slot = a.m[f].slot;
  LmkCtl* const ctl = a.m[f].ctl;
  LmkOut* const out = a.m[f].out;
  const int ldp = a.m[f].ldp, G = a.m[f].G, ld = a.m[f].ld, n = 15 + 6 * a.m[f].M, t = threadIdx.x;
  __shared__ int off[(MAP ? kMaxKeep + kLmkMaxSets : kMaxKeep) + 1], ck[MAP ? 1 : kMaxKeep], rg[kLmkMaxRows];
  __shared__ double s_e2;
  __shared__ int s_used;
  int Gt = G;  // groups: the clones, then (MAP) the clone sets
  if constexpr (MAP) Gt = G + a.m[f].H;

  if (t == 0) {
    int o = 0, u = 0;
    double e2 = 0.0;
    for (int g = 0; g < Gt; ++g) {  // e^2, used, q of each slot
      const double* tl = slot + (size_t)kLmkSlot * g + 42;
      if constexpr (MAP) {
        if (g >= G) tl = a.m[f].sslot + (size_t)kLmkSetSlot * (g - G) + kLmkSetLd * (kLmkSetLd + 1);
      }
      off[g] = o;
      o += (int)tl[2];
      u += (int)tl[1];
      e2 += tl[0];
    }
    off[Gt] = o; s_used = u; s_e2 = e2;
    ctl->ticket = 0u; ctl->bad = 0; ctl->m = o;
  }
  if constexpr (!MAP) {
    for (int g = t; g < G; g += kLmkThreads) ck[g] = a.m[f].grp[3 * g];
  }
  __syncthreads();
  const int m = off[Gt];
  if (s_used == 0) {  // no observation used: nothing is written (the iterate form never gets here: k_lmk_step stops it)
    if (!IT && t == 0) {
      ctl->apply = 0;
      out->nis = 0.0; out->dx_norm = 0.0; out->dof = 0; out->rows = 0; out->used = 0; out->applied = 0; out->status = 0;
      out->numeric = 0;
    }
    return;
  }
  for (int g = t; g < Gt; g += kLmkThreads)
    for (int r = off[g]; r < off[g + 1]; ++r) rg[r] = g;
  __syncthreads();
  // ---- (T P)^T into rows m .. m + n - 1, rho into row m + n.  A row's T entries and clone columns: its clone's 6 (the
  // clone table ck), or (MAP) its group's 6c (lmk_map_row)
  [[maybe_unused]] const int* const grp = a.m[f].grp;
  for (int idx = t; idx < m * n; idx += kLmkThreads) {
    const int r = idx / n, c = idx - r * n, g = rg[r], lr = r - off[g];
    const double* T;
    const S* pc;
    int w = 6;
    [[maybe_unused]] const int* cl;
    if constexpr (MAP) {
      T = lmk_map_row(a.m[f], slot, grp, G, g, lr, w, cl);
      pc = P + c;
    } else {
      T = slot + (size_t)kLmkSlot * g + 6 * lr;
      pc = P + (size_t)(15 + 6 * ck[g]) * ldp + c;
    }
    double s = 0.0;
    for (int j = lr; j < w; ++j) s += T[j] * (double)pc[(size_t)(MAP ? 15 + 6 * cl[j / 6] + j % 6 : j) * ldp];
    A[(size_t)(m + c) * ld + r] = s;
  }
  for (int r = t; r < m; r += kLmkThreads) {
    if constexpr (MAP) {
      int w;
      const int* cl;
      const double* T = lmk_map_row(a.m[f], slot, grp, G, rg[r], 0, w, cl);
      A[(size_t)(m + n) * ld + r] = T[(rg[r] < G ? 36 : kLmkSetLd * kLmkSetLd) + r - off[rg[r]]];
    } else {
      A[(size_t)(m + n) * ld + r] = slot[(size_t)kLmkSlot * rg[r] + 36 + r - off[rg[r]]];
    }
  }
  __syncthreads();
  // ---- S = T P T^T + I, lower triangle
  for (int idx = t; idx < m * m; idx += kLmkThreads) {
    const int r = idx / m, s_ = idx - r * m;
    if (s_ > r) continue;
    const int h = rg[s_], ls = s_ - off[h];
    const double* T;
    const double* tp;
    int w = 6;
    [[maybe_unused]] const int* cl;
    if constexpr (MAP) {
      T = lmk_map_row(a.m[f], slot, grp, G, h, ls, w, cl);
      tp = A + (size_t)(m + 15) * ld + r;
    } else {
      T = slot + (size_t)kLmkSlot * h + 6 * ls;
      tp = A + (size_t)(m + 15 + 6 * ck[h]) * ld + r;
    }
    double v = r == s_ ? 1.0 : 0.0;
    for (int j = ls; j < w; ++j) v += tp[(size_t)(MAP ? 6 * cl[j / 6] + j % 6 : j) * ld] * T[j];
    A[(size_t)r * ld + s_] = v;
  }
  __syncthreads();
  // ---- Cholesky of [S ; (T P)^T ; rho^T] (m + n + 1 rows): the extra rows end as W^T and y
  const int bad = cta_bordered_chol(A, ld, m, m + n + 1, t);
  if (t == 0) {
    if (bad >= 0) {  // S not positive definite: nothing is written
      ctl->apply = 0;
      out->nis = __longlong_as_double(0x7ff8000000000000ll); out->dx_norm = 0.0;
      out->status = 1; out->applied = 0;
      if constexpr (IT) out->iterations = 0;  // (k_lmk_step sees apply = 0 and ends the iteration)
    } else if constexpr (IT) {  // linearisation 0's NIS, dof and counts stay
      ctl->apply = 1;
      out->iterations += 1;
    } else {
      const double* y = A + (size_t)(m + n) * ld;
      double g = s_e2;
      for (int i = 0; i < m; ++i) g += y[i] * y[i];
      ctl->apply = 1;
      out->nis = g; out->status = 0; out->applied = 1;
    }
    if constexpr (!IT) { out->dof = 2 * s_used; out->rows = m; out->used = s_used; out->numeric = 0; }
  }
}

// One CTA per member, after linearisation `it` (0-based): delta_{i+1} = W^T y (the rows of dx in k_lmk_downdate, same order),
// step = max |delta_{i+1} - delta_i| (NaN counts as infinite), then either the member is done (step <= tol: converged; or
// max_iter linearisations made) or the iterate table x^ [+] delta_{i+1} is written for the next linearisation: q <-
// normalise(buildUpdateQuat(dtheta_k) * q^), p <- p^ + dp_k in fp64 (inject_state's clone arithmetic on the widened poses).
template <class S, int NM>
__global__ void __launch_bounds__(kLmkThreads) k_lmk_step(const Members<LmkItArgs<S>, NM> a, int it) {
  const int f = NM == 1 ? 0 : blockIdx.x;
  if (a.m[f].max_iter <= 1) return;
  LmkIt* const ic = a.m[f].it;
  if (it > 0 && ic->done) return;
  if (it + 1 >= a.m[f].max_iter) {  // the member's max_iter linearisations are made (a chunk with a larger max_iter goes on)
    if (threadIdx.x == 0) ic->done = 1;
    return;
  }
  const LmkCtl* const ctl = a.m[f].ctl;
  LmkOut* const out = a.m[f].out;
  const int t = threadIdx.x, lane = t & 31, ld = a.m[f].ld, M = a.m[f].M, n = 15 + 6 * M;
  __shared__ double red[kLmkThreads / 32];
  __shared__ int s_go;
  if (it > 0 && (ic->stop || !ctl->apply)) {  // stopped at the last iterate, or S was not positive definite there
    if (t == 0) ic->done = 1;
    return;
  }
  if (it == 0) {  // the call's first step: reset the control words
    const int ap = ctl->apply;
    if (t == 0) {
      ic->stop = 0; ic->done = !ap;
      out->iterations = ap; out->converged = 0; out->step = 0.0;
    }
    if (!ap) return;
  }
  const int m = ctl->m;
  const double* __restrict__ const Wt = a.m[f].A + (size_t)m * ld;
  const double* __restrict__ const y = a.m[f].A + (size_t)(m + n) * ld;
  double* const d = a.m[f].d;
  double c = 0.0;
  for (int r = t; r < n; r += kLmkThreads) {
    const double* w = Wt + (size_t)r * ld;
    double v = 0.0;
    for (int p = 0; p < m; ++p) v += w[p] * y[p];
    const double dc = fabs(v - (it == 0 ? 0.0 : d[r]));
    c = fmax(c, isnan(dc) ? __longlong_as_double(0x7ff0000000000000ll) : dc);
    d[r] = v;
  }
  for (int o = 16; o > 0; o >>= 1) c = fmax(c, __shfl_xor_sync(0xffffffffu, c, o));
  if (lane == 0) red[t >> 5] = c;
  __syncthreads();
  if (t == 0) {
    double s = red[0];
    for (int w = 1; w < kLmkThreads / 32; ++w) s = fmax(s, red[w]);
    const int conv = s <= a.m[f].tol, go = !conv && it + 2 <= a.m[f].max_iter;
    out->step = s; out->converged = conv;
    if (!go) ic->done = 1;
    s_go = go;
  }
  __syncthreads();
  if (!s_go) return;
  for (int k = t; k < M; k += kLmkThreads) {
    const S* ps = a.m[f].poses + kPoseStride * k;
    const double q[4] = {(double)ps[0], (double)ps[1], (double)ps[2], (double)ps[3]};
    const double dth[3] = {d[15 + 6 * k], d[16 + 6 * k], d[17 + 6 * k]};
    double uq[4], qn[4];
    build_update_quat(dth, uq);
    quat_mul(uq, q, qn);
    quat_normalize(qn);
    double* x = a.m[f].xi + 7 * k;
    x[0] = qn[0]; x[1] = qn[1]; x[2] = qn[2]; x[3] = qn[3];
    x[4] = (double)ps[4] + d[18 + 6 * k]; x[5] = (double)ps[5] + d[19 + 6 * k]; x[6] = (double)ps[6] + d[20 + 6 * k];
  }
}

template <class S, int NM>
__global__ void __launch_bounds__(kLmkThreads) k_lmk_downdate(const Members<LmkArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.y, tl = blockIdx.x;
  if (tl >= a.m[f].ntiles) return;
  LmkCtl* const ctl = a.m[f].ctl;
  if (!ctl->apply) return;
  S* __restrict__ const P = a.m[f].P;
  const int ldp = a.m[f].ldp, ld = a.m[f].ld, M = a.m[f].M, n = 15 + 6 * M, m = ctl->m, t = threadIdx.x;
  const double* __restrict__ const Wt = a.m[f].A + (size_t)m * ld;  // row c: W[:, c]
  const double* __restrict__ const y = a.m[f].A + (size_t)(m + n) * ld;
  double* const dx = a.m[f].dx;
  __shared__ double D[kLmkNB][kLmkNB + 1], B[kLmkNB][kLmkNB + 1];
  __shared__ int s_last;
  int ti, tj;
  tri_tile_index(tl, ti, tj);
  const int rb = kLmkNB * ti, cb = kLmkNB * tj, i = t >> 3, r = rb + i;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int p0 = 0; p0 < m; p0 += kLmkNB) {
    for (int idx = t; idx < kLmkNB * kLmkNB; idx += kLmkThreads) {
      const int ii = idx / kLmkNB, p = idx - ii * kLmkNB;
      D[ii][p] = (rb + ii < n && p0 + p < m) ? Wt[(size_t)(rb + ii) * ld + p0 + p] : 0.0;
      B[ii][p] = (cb + ii < n && p0 + p < m) ? Wt[(size_t)(cb + ii) * ld + p0 + p] : 0.0;
    }
    __syncthreads();
    tile_dot32(D, B, t, s);
    __syncthreads();
  }
  int bad = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int c = cb + (t & 7) + 8 * u;
    if (r < n && c < n && c <= r) {
      const S x = (S)((double)P[(size_t)r * ldp + c] - s[u]);
      if (!isfinite((double)x)) bad = 1;
      P[(size_t)r * ldp + c] = x;
      P[(size_t)c * ldp + r] = x;
    }
  }
  if (ti == tj && t < kLmkNB && rb + t < n) {  // dx = W^T y for this tile's rows
    const double* w = Wt + (size_t)(rb + t) * ld;
    double v = 0.0;
    for (int p = 0; p < m; ++p) v += w[p] * y[p];
    dx[rb + t] = v;
  }
  __threadfence();
  bad = __syncthreads_or(bad);
  if (t == 0) {
    if (bad) atomicOr(&ctl->bad, 1);
    __threadfence();
    s_last = atomicAdd(&ctl->ticket, 1u) == (unsigned)a.m[f].ntiles - 1;
  }
  __syncthreads();
  if (!s_last) return;
  // ---- the last tile of the member: the state injection of the vision update (k_syrk, k_aid)
  __threadfence();
  inject_state(a.m[f].st, a.m[f].poses, M, t, kLmkThreads, [&](int k) { return __ldcg(dx + k); });
  if (t == 0) {
    double nn = 0.0;
    for (int k = 0; k < n; ++k) { const double v = __ldcg(dx + k); nn += v * v; }
    LmkOut* const out = a.m[f].out;
    out->dx_norm = sqrt(nn);
    out->numeric = (atomicOr(&ctl->bad, 0) || !isfinite(nn)) ? 1 : 0;
    ctl->ticket = 0u;
  }
}

}  // namespace mb
