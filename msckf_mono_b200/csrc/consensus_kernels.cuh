// msckf_mono_b200/csrc/consensus_kernels.cuh
// Consensus on the matches of a mapped-landmark call (msckf_b200_landmark_update_consensus, DESIGN.md 4.17).  A hypothesis is
// a 4-dof rigid correction of the whole window applied to the map: p_L' = Rz(psi)^T (p_L - c - t) + c (c: the mean p_C_G of
// the touched clones), projected with the filter's clone pose as lmk_obs does.  Observation i is an inlier of (psi, t) when
// its depth is > 0 and e_i = (z_i - z^_i)^T R^-1 (z_i - z^_i) <= thresh.  All arithmetic in fp64.
//   k_lmk_hyp  : grid (ceil(H / 8), members), one warp per hypothesis.  The lanes solve the pair's 4 x 4 Gauss-Newton
//                redundantly in registers, then score the member's observations lane-strided (__ballot_sync / __popc).
//   k_lmk_cons : one CTA per member.  Arg-max of the counts (ties: the lowest index), Gauss-Newton over the best hypothesis's
//                inliers (J^T J, J^T r by a fixed-order CTA reduction), one rescoring, flag 3 / 0 pre-set for k_lmk_clone.
#pragma once
#include "landmark_kernels.cuh"

namespace mb {

constexpr int kConsWarps = 8;       // hypotheses per CTA of k_lmk_hyp
constexpr int kConsSteps = 8;       // Gauss-Newton steps of the minimal fit and of the refit
constexpr int kConsPerThread = kLmkMaxObs / kLmkThreads;  // observations of one k_lmk_cons thread (its inlier masks' bits)
static_assert(kConsPerThread <= 32, "k_lmk_cons keeps a thread's inlier bits in one word");

// a touched clone's pose: C = C(q_CG), p_C_G
struct ConsPose { double C[9], p[3]; };

// the member's touched clones' poses (by group) and the pivot c = their mean p_C_G (fixed order), into shared memory
template <class S, class A>
__device__ __forceinline__ void cons_poses(const A& m, ConsPose* ps, double* piv) {
  for (int g = threadIdx.x; g < m.G; g += blockDim.x) {
    const S* x = m.poses + kPoseStride * m.grp[3 * g];
    const double q[4] = {(double)x[0], (double)x[1], (double)x[2], (double)x[3]};
    quat_to_rot(q, ps[g].C);
    ps[g].p[0] = (double)x[4]; ps[g].p[1] = (double)x[5]; ps[g].p[2] = (double)x[6];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s[3] = {0.0, 0.0, 0.0};
    for (int g = 0; g < m.G; ++g) { s[0] += ps[g].p[0]; s[1] += ps[g].p[1]; s[2] += ps[g].p[2]; }
    piv[0] = s[0] / m.G; piv[1] = s[1] / m.G; piv[2] = s[2] / m.G;
  }
  __syncthreads();
}

// R^-1 = W (ww, wu, wv: W00, W01, W11) of the call's R or the filter's diag(u_var, v_var)
template <class A>
__device__ __forceinline__ void cons_W(const A& m, double (&W)[3]) {
  double uu = m.R[0], uv = m.R[1], vv = m.R[2];
  if (!m.use_R) { uu = (double)m.st->u_var; uv = 0.0; vv = (double)m.st->v_var; }
  const double det = uu * vv - uv * uv;
  W[0] = vv / det; W[1] = -uv / det; W[2] = uu / det;
}

// observation o (z 2, p_L 3) under th = (psi, t) about pivot c from pose ps: r = z - z^ and e = r^T W r; false when the depth
// is not > 0 or z^ is not finite.  jac: also the 2 x 4 Jacobian of z^ over th.
template <bool JAC>
__device__ __forceinline__ bool cons_obs(const double* o, const ConsPose& ps, const double* c, const double (&th)[4], const double (&W)[3],
                                         double (&r)[2], double& e, double (&Jz)[2][4]) {
  double sn, cs;
  sincos(th[0], &sn, &cs);
  const double d[3] = {o[2] - c[0] - th[1], o[3] - c[1] - th[2], o[4] - c[2] - th[3]};
  const double u[3] = {cs * d[0] + sn * d[1] + c[0] - ps.p[0], -sn * d[0] + cs * d[1] + c[1] - ps.p[1], d[2] + c[2] - ps.p[2]};
  double p[3];
  for (int i = 0; i < 3; ++i) p[i] = ps.C[3 * i] * u[0] + ps.C[3 * i + 1] * u[1] + ps.C[3 * i + 2] * u[2];
  const double zh0 = p[0] / p[2], zh1 = p[1] / p[2];
  if (!(p[2] > 0.0 && isfinite(zh0) && isfinite(zh1))) return false;
  r[0] = o[0] - zh0; r[1] = o[1] - zh1;
  e = W[0] * r[0] * r[0] + 2.0 * W[1] * r[0] * r[1] + W[2] * r[1] * r[1];
  if constexpr (JAC) {
    // dp_L'/dth: columns psi, t0, t1, t2
    const double D[3][4] = {{-sn * d[0] + cs * d[1], -cs, -sn, 0.0}, {-cs * d[0] - sn * d[1], sn, -cs, 0.0}, {0.0, 0.0, 0.0, -1.0}};
    const double iz = 1.0 / p[2];
    const double J[2][3] = {{iz, 0.0, -zh0 * iz}, {0.0, iz, -zh1 * iz}};
    double JC[2][3];
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 3; ++b) JC[a][b] = J[a][0] * ps.C[b] + J[a][1] * ps.C[3 + b] + J[a][2] * ps.C[6 + b];
    for (int a = 0; a < 2; ++a)
      for (int k = 0; k < 4; ++k) Jz[a][k] = JC[a][0] * D[0][k] + JC[a][1] * D[1][k] + JC[a][2] * D[2][k];
  }
  return true;
}

__device__ __forceinline__ bool cons_inlier(const double* o, const ConsPose& ps, const double* c, const double (&th)[4], const double (&W)[3],
                                            double thresh) {
  double r[2], e, J[2][4];
  return cons_obs<false>(o, ps, c, th, W, r, e, J) && e <= thresh;
}

// h[0..9] += the upper triangle of Jz^T W Jz (00 01 02 03 11 12 13 22 23 33), h[10..13] += Jz^T W r; false behind the camera
__device__ __forceinline__ bool cons_acc(const double* o, const ConsPose& ps, const double* c, const double (&th)[4], const double (&W)[3],
                                         double (&h)[14]) {
  double r[2], e, J[2][4];
  if (!cons_obs<true>(o, ps, c, th, W, r, e, J)) return false;
  double WJ[2][4];
  for (int k = 0; k < 4; ++k) { WJ[0][k] = W[0] * J[0][k] + W[1] * J[1][k]; WJ[1][k] = W[1] * J[0][k] + W[2] * J[1][k]; }
  int q = 0;
  for (int a = 0; a < 4; ++a)
    for (int b = a; b < 4; ++b) h[q++] += J[0][a] * WJ[0][b] + J[1][a] * WJ[1][b];
  for (int a = 0; a < 4; ++a) h[10 + a] += WJ[0][a] * r[0] + WJ[1][a] * r[1];
  return true;
}

// th += (J^T W J)^-1 J^T W r by a 4 x 4 Cholesky; false when a pivot is not > 1e-12 x its diagonal entry.  mx: max |step|.
__device__ __forceinline__ bool cons_step(const double (&h)[14], double (&th)[4], double& mx) {
  double L[4][4];
  int q = 0;
  for (int a = 0; a < 4; ++a)
    for (int b = a; b < 4; ++b) L[b][a] = h[q++];
  for (int j = 0; j < 4; ++j) {
    double d = L[j][j];
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    if (!(d > 1e-12 * L[j][j])) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 4; ++i) {
      double s = L[i][j];
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      L[i][j] = s / L[j][j];
    }
  }
  double y[4], x[4];
  for (int i = 0; i < 4; ++i) {
    double s = h[10 + i];
    for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
    y[i] = s / L[i][i];
  }
  for (int i = 3; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < 4; ++k) s -= L[k][i] * x[k];
    x[i] = s / L[i][i];
  }
  mx = 0.0;
  for (int i = 0; i < 4; ++i) {
    th[i] += x[i];
    mx = fmax(mx, isnan(x[i]) ? __longlong_as_double(0x7ff0000000000000ll) : fabs(x[i]));
  }
  return true;
}

template <class S, int NM>
__global__ void __launch_bounds__(kConsWarps * 32) k_lmk_hyp(const Members<LmkConsArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.y;
  const LmkConsArgs<S>& m = a.m[f];
  if (!m.cons || (int)blockIdx.x * kConsWarps >= m.nh) return;
  __shared__ ConsPose ps[kMaxKeep];
  __shared__ double piv[3];
  cons_poses<S>(m, ps, piv);
  const int h = blockIdx.x * kConsWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (h >= m.nh) return;
  double W[3];
  cons_W(m, W);
  const int i = m.pairs[2 * h], j = m.pairs[2 * h + 1];
  const double* oi = m.obs + 5 * (size_t)i;
  const double* oj = m.obs + 5 * (size_t)j;
  const ConsPose& pi = ps[m.ogrp[i]];
  const ConsPose& pj = ps[m.ogrp[j]];
  // ---- the minimal fit (every lane the same arithmetic)
  double th[4] = {0.0, 0.0, 0.0, 0.0};
  bool ok = true;
  for (int s = 0; s < kConsSteps && ok; ++s) {
    double hh[14] = {};
    double mx;
    ok = cons_acc(oi, pi, piv, th, W, hh) && cons_acc(oj, pj, piv, th, W, hh) && cons_step(hh, th, mx);
    if (ok && mx <= 1e-12) break;
  }
  ok = ok && cons_inlier(oi, pi, piv, th, W, m.thresh) && cons_inlier(oj, pj, piv, th, W, m.thresh);
  // lane 0's outcome for the whole warp
  ok = __shfl_sync(0xffffffffu, ok, 0);
  for (int k = 0; k < 4; ++k) th[k] = __shfl_sync(0xffffffffu, th[k], 0);
  int cnt = 0;
  if (ok) {
    for (int b = 0; b < m.n_obs; b += 32) {
      const int o = b + lane;
      const bool in = o < m.n_obs && cons_inlier(m.obs + 5 * (size_t)o, ps[m.ogrp[o]], piv, th, W, m.thresh);
      cnt += __popc(__ballot_sync(0xffffffffu, in));
    }
  }
  if (lane == 0) {
    LmkHyp& y = m.hyp[h];
    for (int k = 0; k < 4; ++k) y.th[k] = th[k];
    y.count = cnt; y.valid = ok;
    m.score[h] = ok ? cnt : -1;
  }
}

template <class S, int NM>
__global__ void __launch_bounds__(kLmkThreads) k_lmk_cons(const Members<LmkConsArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.x;
  const LmkConsArgs<S>& m = a.m[f];
  if (!m.cons) return;
  const int t = threadIdx.x, lane = t & 31, wp = t >> 5, n = m.n_obs;
  __shared__ ConsPose ps[kMaxKeep];
  __shared__ double piv[3], th[4], red[kLmkThreads / 32][14];
  __shared__ int s_key[kLmkThreads / 32], s_val[kLmkThreads / 32], s_best, s_nv, s_ok, s_go;
  cons_poses<S>(m, ps, piv);
  double W[3];
  cons_W(m, W);
  // ---- arg-max of (count, -index) over the valid hypotheses, and the number of valid ones (integers: no order enters)
  int bc = -1, bh = 0x7fffffff, nv = 0;
  for (int h = t; h < m.nh; h += kLmkThreads) {
    const LmkHyp& y = m.hyp[h];
    if (!y.valid) continue;
    ++nv;
    if (y.count > bc) { bc = y.count; bh = h; }  // h ascending: a tie keeps the lower index
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int c2 = __shfl_xor_sync(0xffffffffu, bc, o), h2 = __shfl_xor_sync(0xffffffffu, bh, o);
    if (c2 > bc || (c2 == bc && h2 < bh)) { bc = c2; bh = h2; }
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
  }
  if (lane == 0) { s_key[wp] = bc; s_val[wp] = bh; red[wp][0] = (double)nv; }
  __syncthreads();
  if (t == 0) {
    int c = -1, b = 0x7fffffff, v = 0;
    for (int w = 0; w < kLmkThreads / 32; ++w) {
      if (s_key[w] > c || (s_key[w] == c && s_val[w] < b)) { c = s_key[w]; b = s_val[w]; }
      v += (int)red[w][0];
    }
    s_best = c >= 0 ? b : -1; s_nv = v;
    if (c >= 0)
      for (int k = 0; k < 4; ++k) th[k] = m.hyp[b].th[k];
    s_ok = c >= 0;
  }
  __syncthreads();
  const int best = s_best;
  unsigned m0 = 0u, m1 = 0u;  // bit r: observation t + 256 r is an inlier of the hypothesis / of the refit
  int c0 = 0, c1 = 0, refit = 0;
  double fin[4] = {0.0, 0.0, 0.0, 0.0};
  if (best >= 0) {
    const double t0[4] = {th[0], th[1], th[2], th[3]};
    for (int r = 0; r < kConsPerThread; ++r) {
      const int o = t + kLmkThreads * r;
      if (o < n && cons_inlier(m.obs + 5 * (size_t)o, ps[m.ogrp[o]], piv, t0, W, m.thresh)) m0 |= 1u << r;
    }
    // ---- the refit: Gauss-Newton over the hypothesis's inliers
    for (int s = 0; s < kConsSteps; ++s) {
      double hh[14] = {};
      bool front = true;
      const double tc[4] = {th[0], th[1], th[2], th[3]};
      for (int r = 0; r < kConsPerThread; ++r)
        if ((m0 >> r) & 1u) front = cons_acc(m.obs + 5 * (size_t)(t + kLmkThreads * r), ps[m.ogrp[t + kLmkThreads * r]], piv, tc, W, hh) && front;
      for (int k = 0; k < 14; ++k) hh[k] = warp_sum(hh[k]);
      const int all_front = __syncthreads_and(front);
      if (lane == 0)
        for (int k = 0; k < 14; ++k) red[wp][k] = hh[k];
      __syncthreads();
      if (t == 0) {
        double g[14];
        for (int k = 0; k < 14; ++k) {
          g[k] = red[0][k];
          for (int w = 1; w < kLmkThreads / 32; ++w) g[k] += red[w][k];
        }
        double x[4] = {th[0], th[1], th[2], th[3]}, mx = 0.0;
        const bool ok = all_front && cons_step(g, x, mx);
        if (ok)
          for (int k = 0; k < 4; ++k) th[k] = x[k];
        s_ok = ok;
        s_go = ok && !(mx <= 1e-12);
      }
      __syncthreads();
      if (!s_go) break;
    }
    const double tr[4] = {th[0], th[1], th[2], th[3]};
    bool fin_ok = s_ok;
    for (int k = 0; k < 4; ++k) fin_ok = fin_ok && isfinite(tr[k]);
    if (fin_ok)
      for (int r = 0; r < kConsPerThread; ++r) {
        const int o = t + kLmkThreads * r;
        if (o < n && cons_inlier(m.obs + 5 * (size_t)o, ps[m.ogrp[o]], piv, tr, W, m.thresh)) m1 |= 1u << r;
      }
    // ---- the two inlier counts (integer sums)
    int k0 = __popc(m0), k1 = __popc(m1);
    for (int o = 16; o > 0; o >>= 1) { k0 += __shfl_xor_sync(0xffffffffu, k0, o); k1 += __shfl_xor_sync(0xffffffffu, k1, o); }
    if (lane == 0) { s_key[wp] = k0; s_val[wp] = k1; }
    __syncthreads();
    for (int w = 0; w < kLmkThreads / 32; ++w) { c0 += s_key[w]; c1 += s_val[w]; }
    refit = fin_ok && c1 >= c0;
    for (int k = 0; k < 4; ++k) fin[k] = refit ? tr[k] : t0[k];
  }
  const unsigned fm = refit ? m1 : m0;
  const int inl = refit ? c1 : c0, ok = best >= 0 && inl >= m.min_inl;
  for (int r = 0; r < kConsPerThread; ++r) {
    const int o = t + kLmkThreads * r;
    if (o < n) m.flag[o] = ok && ((fm >> r) & 1u) ? 0 : 3;
  }
  if (t == 0) {
    LmkConsOut& z = *m.cres;
    z.status = ok ? 0 : 1; z.inliers = best >= 0 ? inl : 0; z.best = best; z.valid = s_nv; z.refit = refit;
    z.yaw = fin[0]; z.t[0] = fin[1]; z.t[1] = fin[2]; z.t[2] = fin[3];
    z.pivot[0] = piv[0]; z.pivot[1] = piv[1]; z.pivot[2] = piv[2];
  }
}

}  // namespace mb
