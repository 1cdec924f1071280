// msckf_mono_b200/csrc/feature_kernels.cuh
// Per-feature stage of the MSCKF measurement update, one warp per feature track:
//   k_tri     : checkMotion (msckf.h:980-1025) + inverse-depth LM triangulation (msckf.h:1147-1285)
//   k_jac     : one CTA per track: loop-A bookkeeping of marginalize() (msckf.h:352-399, incl. the p_f_G_vec index
//               quirk of :419), calcResidual (:960-978), calcMeasJacobian (:905-958, left null space by 3 Householder
//               reflectors of the column-pivoted QR of H_f), gatingTest (:1103-1124)
//   (ordered stacking offsets, msckf.h:433-445: prefix sum by the last CTA of k_jac)
// Clone poses are staged into shared memory with one TMA bulk copy per CTA.
#pragma once
#include "common.cuh"

namespace mb {

// Eigen::LDLT (diagonal pivoting) solve of a symmetric 3x3 system, msckf.h:1222, register-only.
// Eigen's unblocked LDLT is left-looking: at step k it picks the largest |diagonal| among the not yet eliminated
// (and not yet updated) entries, i.e. the elimination order is the descending order of the ORIGINAL |a_ii|
// (first index wins ties).  The symmetric permutation is applied with uniform branches, then the recurrences of
// ldlt_inplace<Lower>::unblocked follow literally.
template <class S>
__device__ __forceinline__ void ldlt3_solve(S a00, S a01, S a02, S a11, S a12, S a22, const S b[3], S x[3]) {
  const S d0a = tabs(a00), d1a = tabs(a11), d2a = tabs(a22);
  int p0 = 0;
  if (d1a > d0a) p0 = 1;
  if (d2a > (p0 == 0 ? d0a : d1a)) p0 = 2;
  int p1, p2;
  {
    const int q0 = (p0 == 0) ? 1 : 0, q1 = (p0 == 2) ? 1 : 2;  // remaining two, ascending
    const S dq0 = (q0 == 0) ? d0a : d1a, dq1 = (q1 == 1) ? d1a : d2a;
    // Eigen swaps k <-> biggest: the other remaining index may have moved into p0's slot; the search order of the
    // tail after the swap is (slot1, slot2).  After swapping 0 <-> p0 the slots hold: p0==1 -> (0, 2); p0==2 -> (1, 0); p0==0 -> (1, 2)
    const int s1 = (p0 == 0) ? 1 : (p0 == 1 ? 0 : 1), s2 = (p0 == 0) ? 2 : (p0 == 1 ? 2 : 0);
    const S ds1 = (s1 == 0) ? d0a : (s1 == 1 ? d1a : d2a), ds2 = (s2 == 0) ? d0a : (s2 == 1 ? d1a : d2a);
    (void)q0; (void)q1; (void)dq0; (void)dq1;
    if (ds2 > ds1) { p1 = s2; p2 = s1; } else { p1 = s1; p2 = s2; }
  }
  // permuted entries m_ij = a[p_i][p_j]
  auto pick = [&](int i, int j) -> S {
    const int lo = i < j ? i : j, hi = i < j ? j : i;
    if (lo == 0) return hi == 0 ? a00 : (hi == 1 ? a01 : a02);
    if (lo == 1) return hi == 1 ? a11 : a12;
    return a22;
  };
  const S m00 = pick(p0, p0), m10 = pick(p1, p0), m20 = pick(p2, p0), m11 = pick(p1, p1), m21 = pick(p2, p1), m22 = pick(p2, p2);
  const S c0 = b[p0 == 0 ? 0 : (p0 == 1 ? 1 : 2)], c1 = b[p1 == 0 ? 0 : (p1 == 1 ? 1 : 2)], c2 = b[p2 == 0 ? 0 : (p2 == 1 ? 1 : 2)];
  // k = 0
  const S dd0 = m00;
  const bool v0 = tabs(dd0) > S(0);
  const S l10 = v0 ? m10 / dd0 : m10, l20 = v0 ? m20 / dd0 : m20;
  // k = 1
  const S t0 = dd0 * l10;
  const S dd1 = m11 - l10 * t0;
  S l21 = m21 - l20 * t0;
  const bool v1 = tabs(dd1) > S(0);
  if (v1) l21 = l21 / dd1;
  // k = 2
  const S u0 = dd0 * l20, u1 = dd1 * l21;
  const S dd2 = m22 - (l20 * u0 + l21 * u1);
  // solve
  S y0 = c0, y1 = c1 - l10 * y0, y2 = c2 - (l20 * y0 + l21 * y1);
  y0 = (tabs(dd0) > S(0)) ? y0 / dd0 : S(0);
  y1 = (tabs(dd1) > S(0)) ? y1 / dd1 : S(0);
  y2 = (tabs(dd2) > S(0)) ? y2 / dd2 : S(0);
  y1 = y1 - l21 * y2;
  y0 = y0 - (l10 * y1 + l20 * y2);
  // un-permute
  x[0] = (p0 == 0) ? y0 : (p1 == 0 ? y1 : y2);
  x[1] = (p0 == 1) ? y0 : (p1 == 1 ? y1 : y2);
  x[2] = (p0 == 2) ? y0 : (p1 == 2 ? y1 : y2);
}

// sum over the track's observations of the reprojection cost (msckf.h:1027-1047), warp-reduced
template <class S>
__device__ __forceinline__ S track_cost(const S* rel, const S* z, int L, int lane, const S x[3]) {
  S acc = 0;
  for (int i = lane; i < L; i += 32) {
    const S* T = rel + 12 * i;
    const S h0 = T[0] * x[0] + T[1] * x[1] + T[2] + x[2] * T[9];
    const S h1 = T[3] * x[0] + T[4] * x[1] + T[5] + x[2] * T[10];
    const S h2 = T[6] * x[0] + T[7] * x[1] + T[8] + x[2] * T[11];
    const S e0 = h0 / h2 - z[2 * i], e1 = h1 / h2 - z[2 * i + 1];
    acc += e0 * e0 + e1 * e1;
  }
  return warp_sum(acc);
}

template <class S, int WPB>
__global__ void __launch_bounds__(WPB * 32) k_tri(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  pdl_launch();
  const UpdArgs<S>& a = args[blockIdx.z];
  if ((int)blockIdx.x * WPB >= a.n_tracks) return;  // (a batch launch is sized for its largest filter)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  S* poses = reinterpret_cast<S*>(smem_raw + 16);
  S* rel_all = poses + (size_t)a.M * kPoseStride;
  stage_table_tma(poses, a.poses, (unsigned)(a.M * kPoseStride * sizeof(S)), bar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * WPB + warp;
  if (t >= a.n_tracks) return;
  const int o0 = a.obs_off[t], L = a.obs_off[t + 1] - o0;
  const int* idx = a.clone_idx + o0;
  const S* zg = a.obs + 2 * (size_t)o0;
  S* rel = rel_all + (size_t)warp * a.Lmax * 14;
  S* z = rel + (size_t)a.Lmax * 12;  // observations staged in shared memory (read ~100x by the LM loops)
  for (int e = lane; e < 2 * L; e += 32) z[e] = zg[e];
  __syncwarp();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.counter_snap = a.st->num_residualized;
  if (L < 2) {  // a single observation cannot be triangulated (the reference's checkMotion is false there, msckf.h:982-984,
                // and its initial guess divides by zero): reported as rejected instead of failing the batch
    if (lane == 0) { a.pfg[3 * t] = a.pfg[3 * t + 1] = a.pfg[3 * t + 2] = S(0); a.cm_ok[t] = 0; a.tri_ok[t] = 0; }
    return;
  }
  // first clone: camera -> world
  const S* pose0 = poses + kPoseStride * idx[0];
  S C0[9];
  quat_to_rot(pose0, C0);
  const S p0[3] = {pose0[4], pose0[5], pose0[6]};
  // ---- checkMotion (msckf.h:980-1025)
  int cm = 0;
  if (L >= 2) {
    S d[3] = {z[0], z[1], S(1.0)};
    const S dn = tsqrt<S>(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    d[0] /= dn; d[1] /= dn; d[2] /= dn;
    const S dw[3] = {C0[0] * d[0] + C0[3] * d[1] + C0[6] * d[2], C0[1] * d[0] + C0[4] * d[1] + C0[7] * d[2],
                     C0[2] * d[0] + C0[5] * d[1] + C0[8] * d[2]};  // C0^T d
    S mo = 0;
    for (int i = 1 + lane; i < L; i += 32) {
      const S* ps = poses + kPoseStride * idx[i];
      const S tr[3] = {ps[4] - p0[0], ps[5] - p0[1], ps[6] - p0[2]};
      const S par = tr[0] * dw[0] + tr[1] * dw[1] + tr[2] * dw[2];
      const S o[3] = {tr[0] - par * dw[0], tr[1] - par * dw[1], tr[2] - par * dw[2]};
      const S nn = tsqrt<S>(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
      mo = nn > mo ? nn : mo;
    }
    mo = warp_max(mo);
    cm = mo > a.st->translation_threshold;
  }
  // ---- relative poses T_i^-1 * T_0 (msckf.h:1154-1168): rel = [R (9) | t (3)], first-clone frame -> clone i
  for (int i = lane; i < L; i += 32) {
    const S* ps = poses + kPoseStride * idx[i];
    S Ci[9];
    quat_to_rot(ps, Ci);
    S* T = rel + 12 * i;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)  // C_i * C_0^T
        T[3 * r + c] = Ci[3 * r] * C0[3 * c] + Ci[3 * r + 1] * C0[3 * c + 1] + Ci[3 * r + 2] * C0[3 * c + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const S a0 = Ci[3 * r] * p0[0] + Ci[3 * r + 1] * p0[1] + Ci[3 * r + 2] * p0[2];
      const S a1 = -(Ci[3 * r] * ps[4] + Ci[3 * r + 1] * ps[5] + Ci[3 * r + 2] * ps[6]);
      T[9 + r] = a0 + a1;
    }
  }
  __syncwarp();
  // ---- generateInitialGuess (msckf.h:1126-1145) from the first and the last observation
  S sol[3];
  {
    const S* T = rel + 12 * (L - 1);
    const S z1u = z[0], z1v = z[1], z2u = z[2 * (L - 1)], z2v = z[2 * (L - 1) + 1];
    const S m0 = T[0] * z1u + T[1] * z1v + T[2], m1 = T[3] * z1u + T[4] * z1v + T[5], m2 = T[6] * z1u + T[7] * z1v + T[8];
    const S A0 = m0 - z2u * m2, A1 = m1 - z2v * m2;
    const S b0 = z2u * T[11] - T[9], b1 = z2v * T[11] - T[10];
    const S depth = (S(1) / (A0 * A0 + A1 * A1)) * (A0 * b0 + A1 * b1);
    const S i0 = z1u * depth, i1 = z1v * depth, i2 = depth;
    sol[0] = i0 / i2; sol[1] = i1 / i2; sol[2] = S(1.0) / i2;
  }
  // ---- Levenberg-Marquardt (msckf.h:1178-1248); all control flow is warp-uniform
  S lambda = S(1e-3);
  int inner = 0, outer = 0;
  bool reduced = false;
  S delta_norm = 0;
  S total_cost = track_cost(rel, z, L, lane, sol);
  do {
    S s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // A00 A01 A02 A11 A12 A22 b0 b1 b2
    for (int i = lane; i < L; i += 32) {
      const S* T = rel + 12 * i;
      const S h0 = T[0] * sol[0] + T[1] * sol[1] + T[2] + sol[2] * T[9];
      const S h1 = T[3] * sol[0] + T[4] * sol[1] + T[5] + sol[2] * T[10];
      const S h2 = T[6] * sol[0] + T[7] * sol[1] + T[8] + sol[2] * T[11];
      // W = [R(:,0:2) | t]
      const S W0[3] = {T[0], T[1], T[9]}, W1[3] = {T[3], T[4], T[10]}, W2[3] = {T[6], T[7], T[11]};
      S J0[3], J1[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        J0[c] = S(1) / h2 * W0[c] - h0 / (h2 * h2) * W2[c];
        J1[c] = S(1) / h2 * W1[c] - h1 / (h2 * h2) * W2[c];
      }
      const S r0 = h0 / h2 - z[2 * i], r1 = h1 / h2 - z[2 * i + 1];
      const S e = tsqrt<S>(r0 * r0 + r1 * r1);
      const S w = (e <= S(0.01)) ? S(1.0) : S(0.01) / (S(2) * e);
      const S w2 = (w == S(1)) ? S(1) : w * w;
      s[0] += w2 * (J0[0] * J0[0] + J1[0] * J1[0]);
      s[1] += w2 * (J0[0] * J0[1] + J1[0] * J1[1]);
      s[2] += w2 * (J0[0] * J0[2] + J1[0] * J1[2]);
      s[3] += w2 * (J0[1] * J0[1] + J1[1] * J1[1]);
      s[4] += w2 * (J0[1] * J0[2] + J1[1] * J1[2]);
      s[5] += w2 * (J0[2] * J0[2] + J1[2] * J1[2]);
      s[6] += w2 * (J0[0] * r0 + J1[0] * r1);
      s[7] += w2 * (J0[1] * r0 + J1[1] * r1);
      s[8] += w2 * (J0[2] * r0 + J1[2] * r1);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) s[k] = warp_sum(s[k]);
    do {
      const S b[3] = {s[6], s[7], s[8]};
      S delta[3];
      ldlt3_solve(s[0] + lambda, s[1], s[2], s[3] + lambda, s[4], s[5] + lambda, b, delta);
      const S ns[3] = {sol[0] - delta[0], sol[1] - delta[1], sol[2] - delta[2]};
      delta_norm = tsqrt<S>(delta[0] * delta[0] + delta[1] * delta[1] + delta[2] * delta[2]);
      const S new_cost = track_cost(rel, z, L, lane, ns);
      if (new_cost < total_cost) {
        reduced = true;
        sol[0] = ns[0]; sol[1] = ns[1]; sol[2] = ns[2];
        total_cost = new_cost;
        lambda = (S)((double)(lambda / 10) > 1e-10 ? (double)(lambda / 10) : 1e-10);
      } else {
        reduced = false;
        lambda = (S)((double)(lambda * 10) < 1e12 ? (double)(lambda * 10) : 1e12);
      }
    } while (inner++ < 10 && !reduced);
    inner = 0;
  } while (outer++ < 10 && delta_norm > S(5e-7));
  const S fin[3] = {sol[0] / sol[2], sol[1] / sol[2], S(1.0) / sol[2]};
  // ---- validity (msckf.h:1255-1276)
  int bad = 0;
  for (int i = lane; i < L; i += 32) {
    const S* T = rel + 12 * i;
    const S pz = T[6] * fin[0] + T[7] * fin[1] + T[8] * fin[2] + T[11];
    if (pz <= S(0)) bad = 1;
  }
  bad = __any_sync(0xffffffffu, bad);
  const S normalized_cost = total_cost / (S)(2 * (size_t)L * (size_t)L);
  int ok = !bad;
  if (normalized_cost > a.st->max_gn_cost_norm) ok = 0;
  if (lane == 0) {
    // p_f_G = C0^T * fin + p0 (msckf.h:1282), computed even when invalid
    a.pfg[3 * t + 0] = C0[0] * fin[0] + C0[3] * fin[1] + C0[6] * fin[2] + p0[0];
    a.pfg[3 * t + 1] = C0[1] * fin[0] + C0[4] * fin[1] + C0[7] * fin[2] + p0[1];
    a.pfg[3 * t + 2] = C0[2] * fin[0] + C0[5] * fin[1] + C0[8] * fin[2] + p0[2];
    a.cm_ok[t] = cm;
    a.tri_ok[t] = ok;
  }
}

// packed lower-triangular symmetric storage
__device__ __forceinline__ int pk(int i, int j) { return i * (i + 1) / 2 + j; }  // i >= j

constexpr int JT = 128;  // most threads a CTA of k_jac has (see JGrp)

// A track is worked on by a GROUP of G threads (G = 128: the whole CTA -- lowest latency, used for a single filter;
// G = 64 / 32: two / four tracks per CTA, a warp (pair) each -- the CTA barriers between the phases of a track become
// named barriers / __syncwarp, so a track's serial sections (the QR warp, the panels of the gate Cholesky) no longer idle
// the warps of the same CTA: they belong to other tracks.  Used for device batches, where throughput is what counts.)
template <int G>
struct JGrp {
  static_assert(G == 32 || G == 64 || G == 128, "group size");
  // G = 32 runs in CTAs of 64 threads (two tracks): the finer the CTA, the more tracks fit the SM's shared memory (20 at L = 30)
  static constexpr int CT = (G == 32) ? 64 : 128, NW = G / 32, TPC = CT / G;
  __device__ static __forceinline__ void sync(int grp) {
    if (G == CT) __syncthreads();
    else if (G == 32) __syncwarp();
    else asm volatile("bar.sync %0, %1;" : : "r"(grp + 1), "r"(G) : "memory");
  }
};

// sum over the group; red: the CTA's CT/32 slots (one per warp)
template <int G, class T>
__device__ __forceinline__ T group_sum(T v, T* red, int grp) {
  v = warp_sum(v);
  if (G == 32) return v;
  const int w0 = grp * JGrp<G>::NW;
  JGrp<G>::sync(grp);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  JGrp<G>::sync(grp);
  T t = red[w0];
#pragma unroll
  for (int w = 1; w < JGrp<G>::NW; ++w) t += red[w0 + w];
  return t;
}

// Floating-point sums over a track's group, bit-identical for every group size: the terms are dealt to 128 VIRTUAL threads
// (virtual thread v = 32 w + lane owns the terms v, v + 128, ...), every virtual warp w is reduced by shuffles, and the four
// warp sums are added in the order ((s0 + s1) + s2) + s3.  A group of G threads plays 4 / (G/32) virtual warps per warp, so a
// device batch (G = 32) rounds exactly like the same filter run alone (G = 128).
// part(v, p): the K partial sums of virtual thread v;  red: [TPC][4][K] shared slots.
template <int G, int K, class T, class F>
__device__ __forceinline__ void group_vsum(T (&out)[K], F part, T* red, int grp) {
  constexpr int NW = JGrp<G>::NW, R = 4 / NW;
  const int lane = threadIdx.x & 31, gw = (threadIdx.x % G) >> 5;
  if (G == 32) {  // one warp plays all four virtual warps: ((s0 + s1) + s2) + s3 folded as they come (4 x K fewer live registers)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      T p[K];
      part(32 * q + lane, p);
#pragma unroll
      for (int k = 0; k < K; ++k) { const T s = warp_sum(p[k]); out[k] = (q == 0) ? s : out[k] + s; }
    }
    return;
  }
  T s[R][K];
#pragma unroll
  for (int q = 0; q < R; ++q) {
    T p[K];
    part(32 * (gw + NW * q) + lane, p);
#pragma unroll
    for (int k = 0; k < K; ++k) s[q][k] = warp_sum(p[k]);
  }
  JGrp<G>::sync(grp);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < R; ++q)
#pragma unroll
      for (int k = 0; k < K; ++k) red[(grp * 4 + gw + NW * q) * K + k] = s[q][k];
  }
  JGrp<G>::sync(grp);
#pragma unroll
  for (int k = 0; k < K; ++k) out[k] = ((red[(grp * 4 + 0) * K + k] + red[(grp * 4 + 1) * K + k]) + red[(grp * 4 + 2) * K + k]) + red[(grp * 4 + 3) * K + k];
}

__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const double* p, double (&v)[4]) {
  const double2 t = *reinterpret_cast<const double2*>(p), u = *reinterpret_cast<const double2*>(p + 2);
  v[0] = t.x; v[1] = t.y; v[2] = u.x; v[3] = u.y;
}
// two elements at an even offset from an aligned base
__device__ __forceinline__ void ld2(const float* p, float& a, float& b) { const float2 t = *reinterpret_cast<const float2*>(p); a = t.x; b = t.y; }
__device__ __forceinline__ void ld2(const double* p, double& a, double& b) { const double2 t = *reinterpret_cast<const double2*>(p); a = t.x; b = t.y; }
// p[0..5] of a row of P at an odd column (a clone block starts at kImuDim + 6 j; P's base and ldp are even-aligned): four
// aligned pairs from p - 1 instead of six scalar loads.  p[6] exists: the last clone block ends at column n - 1, and ldp
// rounds the odd capacity n_max >= n up to a multiple of 4.
static_assert(kImuDim % 2 == 1, "clone blocks start at odd columns");
template <class S>
__device__ __forceinline__ void ld6_odd(const S* p, S (&v)[6]) {
  S d;
  ld2(p - 1, d, v[0]); ld2(p + 1, v[1], v[2]); ld2(p + 3, v[3], v[4]); ld2(p + 5, v[5], d);
}

// ---- gate Cholesky, blocked by panels of 8 columns, all G threads of the track's group.
// The matrix is the packed-lower n x n array Y (n = 2L pivots from row 0); the kJRhs right-hand sides ride along as rows
// n .. n + 3 of the augmented matrix, stored as contiguous rows of n at rhs (row q at rhs + q n).  Only L^-1 rhs is wanted (the
// gate's quadratic forms), so the factor itself is never written back: each right-hand side row ends as L^-1 of itself.
// Per panel:  (1) every thread that owns a row loads the 8 x 8 diagonal micro-block and factorises it redundantly in registers (static
// indices, right-looking: the dependent chain of a pivot is rsqrt -> multiply -> one FMA) -- no shuffles, no barriers, no
// pivot broadcast;  (2) every thread solves its own rows of the panel against that micro-block in registers (rows >= n = the
// right-hand sides: their 8 entries are final);  (3) the solved panel goes to shared memory TRANSPOSED ([8][Rp]: neighbouring
// threads touch neighbouring words), one barrier;  (4) trailing update in 4 x 4 register tiles over the lower triangle, one
// barrier.  60 pivots cost 8 panels x 2 barriers instead of 60 dependent warp-wide steps (round 1: one warp, shuffle +
// shared-memory round trip per pivot: over a third of k_jac).
constexpr int kPW = 8;
constexpr int kJRhs = 4;  // z, U(:,0), U(:,1), U(:,2)
template <class S, int G>
__device__ __forceinline__ bool gate_chol_blocked(S* __restrict__ Y, S* __restrict__ rhs, int n, S* __restrict__ PnT, int Rp, int* s_fail, int grp) {
  const int R = n + kJRhs, tid = threadIdx.x % G;
  if (tid == 0) *s_fail = 0;
  for (int e = tid; e < kPW * Rp; e += G) PnT[e] = S(0);  // (rows R..Rp-1 of a partial tile must read as zero)
  JGrp<G>::sync(grp);
  for (int p0 = 0; p0 < n; p0 += kPW) {
    const int w = min(kPW, n - p0);
    // (1) diagonal micro-block: lower triangle in registers, identity padding beyond w -- only in the threads that own a row
    // of this panel (the others would spend a fifth of the kernel's instructions on a result they never use)
    const int q0 = p0 + w;
    if (q0 + tid < R) {
      S Lm[kPW][kPW], inv[kPW];
#pragma unroll
      for (int a = 0; a < kPW; ++a)
#pragma unroll
        for (int b = 0; b <= a; ++b) Lm[a][b] = (a < w) ? Y[pk(p0 + a, p0 + b)] : ((a == b) ? S(1) : S(0));
      bool ok = true;
#pragma unroll
      for (int j = 0; j < kPW; ++j) {
        const S d = Lm[j][j];
        if (!(d > S(0))) ok = false;
        const S iv = fast_rsqrt(d);
        inv[j] = iv;
#pragma unroll
        for (int a = j + 1; a < kPW; ++a) Lm[a][j] *= iv;
#pragma unroll
        for (int b = j + 1; b < kPW; ++b)
#pragma unroll
          for (int a = b; a < kPW; ++a) Lm[a][b] -= Lm[a][j] * Lm[b][j];
      }
      if (!ok && tid == 0) *s_fail = 1;  // (thread 0 always owns a row: the right-hand sides are rows >= n >= q0)
      // (2) rows below the micro-block, and the right-hand sides
      for (int i = q0 + tid; i < R; i += G) {
        S* row = (i < n) ? Y + pk(i, p0) : rhs + (size_t)(i - n) * n + p0;
        S x[kPW];
#pragma unroll
        for (int j = 0; j < kPW; ++j) x[j] = (j < w) ? row[j] : S(0);
#pragma unroll
        for (int j = 0; j < kPW; ++j) {
          x[j] *= inv[j];
#pragma unroll
          for (int jj = j + 1; jj < kPW; ++jj) x[jj] -= x[j] * Lm[jj][j];
        }
#pragma unroll
        for (int j = 0; j < kPW; ++j) PnT[j * Rp + i] = x[j];
        if (i >= n) {
#pragma unroll
          for (int j = 0; j < kPW; ++j) if (j < w) row[j] = x[j];  // final components of L^-1 rhs
        }
      }
    }
    JGrp<G>::sync(grp);
    if (*s_fail) return false;  // a non-positive pivot (uniform: read after the barrier)
    // (4) trailing update: rows q0..R-1, columns q0..n-1, lower triangle, 4 x 4 tiles (q0 < n: a full panel, q0 a multiple
    // of 8; after the last panel only right-hand-side rows are left, and they have no columns to update)
    if (q0 < n) {
      const int nt = (R - q0 + 3) >> 2, ntile = nt * (nt + 1) / 2;
      for (int q = tid; q < ntile; q += G) {
        int ti, tj;
        tri_tile_index(q, ti, tj);
        const int r0 = q0 + 4 * ti, c0 = q0 + 4 * tj;
        if (c0 >= n) continue;  // (the tile of the right-hand sides against themselves)
        S acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) acc[a][b] = S(0);
#pragma unroll
        for (int j = 0; j < kPW; ++j) {
          S pr[4], pc[4];
          ld4(PnT + j * Rp + r0, pr);
          ld4(PnT + j * Rp + c0, pc);
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] += pr[a] * pc[b];
        }
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const int row = r0 + a;
          if (row >= R) continue;
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const int col = c0 + b;
            if (col < n && col <= row) {
              if (row < n) Y[pk(row, col)] -= acc[a][b]; else rhs[(size_t)(row - n) * n + col] -= acc[a][b];
            }
          }
        }
      }
    }
    JGrp<G>::sync(grp);
  }
  return true;
}

// shared memory of one track's group (rounded to 16 bytes), in units of S:
//   r 2L | X 12L | V 6L (+ slack) | Ypacked L(2L+1)
// Once the compact outputs are written X is dead: the gate's right-hand sides U^T ([3][2L], U rounded to S) take its first
// 6L, right after r (which becomes z), so that the four right-hand-side rows are contiguous; and once they are built V is dead
// too: the gate Cholesky's transposed panel PnT (8 x Rp, Rp = (2L + 7) & ~3 >= 2L + 4 rows, 16-byte aligned) follows U^T, over
// the rest of X, V and the slack.  U (the first 3 columns of the feature's Q, fp64) is otherwise never stored: its rows are
// rebuilt from V where they are needed (u_row).
__host__ __device__ inline int jac_panel_rows(int L) { return (2 * L + 7) & ~3; }
template <class S>
__host__ __device__ inline size_t jac_xv_elems(int L) {
  const size_t gate = (size_t)6 * L + (16 / sizeof(S) - 1) + (size_t)kPW * jac_panel_rows(L);  // U^T | alignment | PnT
  return (size_t)18 * L > gate ? (size_t)18 * L : gate;
}
template <class S>
__host__ __device__ inline size_t jac_group_bytes(int L) {
  const size_t b = sizeof(S) * ((size_t)2 * L + jac_xv_elems<S>(L) + (size_t)L * (2 * L + 1));
  return (b + 15) & ~(size_t)15;
}
// whole CTA: groups of 64 / 128 threads: bar 16 | poses M*8 S | pad 16 | the groups; a single warp reads its few poses from
// global, so a CTA of G = 32 holds its two groups alone (sized by the launch's longest track)
template <class S>
__host__ __device__ inline size_t jac_smem_bytes(int L, int M, int g) {
  const int tpc = (g == 128) ? 1 : 2;
  return (g == 32 ? 0 : 16 + sizeof(S) * kPoseStride * (size_t)M + 16) + (size_t)tpc * jac_group_bytes<S>(L);
}

// Row `row` of U = H0 H1 H2 [I3; 0] (fp64) after the reflectors H2 .. H_kmin have been applied to [I3; 0] in that order:
// H_k changes rows >= k only, by  u -= sd_k v_k(row)  with  sd_k = tau64_k v_k^T U  (sd[3 k + q]).  The same operations in
// the same order as applying them to a stored [2L][3] array, so the values are the same bits.
template <class S>
__device__ __forceinline__ void u_row(const S* __restrict__ V, const double* sd, int row, int kmin, double (&u)[3]) {
#pragma unroll
  for (int q = 0; q < 3; ++q) u[q] = (row == q) ? 1.0 : 0.0;
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    if (k < kmin || row < k) continue;
    const double vk = (double)V[3 * row + k];
    u[0] -= sd[3 * k] * vk; u[1] -= sd[3 * k + 1] * vk; u[2] -= sd[3 * k + 2] * vk;
  }
}

// Ordered stacking (msckf.h:433-445): the exclusive prefix sum of the accepted blocks' row counts, computed by whichever
// CTA of k_jac finishes last (ticket counter) -- a separate 1-CTA kernel for 300 integers cost a launch latency.
template <class S, int CT>
__device__ __forceinline__ void jac_finish(const UpdArgs<S>& a, int n_cta /* CTAs of this filter that arrive here */) {
  __shared__ int s_last;
  __shared__ int s_part[CT / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __syncthreads();
  if (tid == 0) { __threadfence(); s_last = (atomicAdd(a.done, 1u) == (unsigned)n_cta - 1u) ? 1 : 0; }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int N = a.n_tracks, per = (N + CT - 1) / CT;
  const int b = min(N, tid * per), e = min(N, b + per);
  int sum = 0;
  for (int k = b; k < e; ++k) sum += __ldcg(a.rows + k);
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) s_part[warp] = incl;
  __syncthreads();
  int run = incl - sum;
  for (int w = 0; w < warp; ++w) run += s_part[w];
  for (int k = b; k < e; ++k) { a.row_off[k] = run; run += __ldcg(a.rows + k); }
  if (tid == CT - 1) { a.row_off[N] = run; a.m_out[0] = run; a.m_out[2] = 0; /* status: set by k_syrk / k_inject */ }
  if (tid == 0) *a.done = 0u;
}

// calcResidual + calcMeasJacobian + gatingTest for one feature per group of G threads (JT / G features per CTA), with
// loop A's bookkeeping (msckf.h:352-399: valid flags, num_feature_tracks_residualized_, and the p_f_G_vec index of :419)
// folded into the prologue.  mode 0: marginalize semantics; mode 1: every track valid at its given position.
// Inside: `tid`, `warp` are relative to the group; every barrier is the group's.
template <class S, int G>
__device__ __forceinline__ void jac_track(const UpdArgs<S>& a, const int t, const int grp, unsigned char* __restrict__ gmem_sm,
                                          const S* __restrict__ poses, double* redd, S* reds, int* redi) {
  using Gp = JGrp<G>;
  DevState<S>* st_rw = a.st;
  const int mode = (a.mode == 2) ? 1 : 0;  // MSCKF_B200_RESIDUALIZE: every track valid at its given position
  __shared__ int s_he_[Gp::TPC], s_valid_[Gp::TPC], s_src_[Gp::TPC], s_pushed_t_[Gp::TPC];
  __shared__ unsigned long long s_cnt_[Gp::TPC];
  int &s_he = s_he_[grp], &s_valid = s_valid_[grp], &s_src = s_src_[grp], &s_pushed_t = s_pushed_t_[grp];
  unsigned long long& s_cnt = s_cnt_[grp];
  const int tid = threadIdx.x % G, lane = tid & 31;
  const int N = a.n_tracks;
  const int c = 6 * a.M;
  int prof_i = 0;
  auto stamp = [&]() {
    if (a.prof && blockIdx.x == 0 && threadIdx.x == 0 && prof_i < 30) a.prof[40 + prof_i++] = globaltimer();
  };
  stamp();
  // ------------------------------------------------------------------ loop-A bookkeeping
  if (mode == 1) {
    if (tid == 0) { s_valid = 1; s_src = t; }
  } else {
    if (tid == 0) {
      unsigned long long counter = *a.counter_snap;
      int k = 0;
      for (; k < N && counter <= 3; ++k)  // checkMotion is not consulted while the counter is <= 3 (msckf.h:354)
        if (a.tri_ok[k]) counter++;
      s_he = k;
      s_cnt = counter;
    }
    Gp::sync(grp);
    const int he = s_he;
    // pushed(k): the track pushed a position into p_f_G_vec (msckf.h:374)
    int before = 0, total = 0, nvalid_tail = 0;
    for (int k = tid; k < N; k += G) {
      const int cm = a.cm_ok[k];
      const int pushed = (k < he) ? 1 : cm;
      total += pushed;
      if (k < t) before += pushed;
      if (k >= he && cm && a.tri_ok[k]) nvalid_tail++;
    }
    auto isum = [&](int v) { return group_sum<G>(v, redi, grp); };
    total = isum(total);
    before = isum(before);
    nvalid_tail = isum(nvalid_tail);
    if (tid == 0) {
      const int cm_t = a.cm_ok[t];
      const int pushed_t = (t < he) ? 1 : cm_t;
      const int valid_t = (t < he) ? a.tri_ok[t] : (cm_t && a.tri_ok[t]);
      // loop B reads p_f_G_vec[iter] (msckf.h:419): the iter-th pushed track when it exists, else (UB in the
      // reference) the track's own position
      int src = t;
      if (t < total && !(before == t && pushed_t)) {  // fast path: nothing before t was rejected -> p_f_G_vec[t] is t's own
        int seen = 0;
        for (int k = 0; k < N; ++k) {
          const int pushed = (k < he) ? 1 : a.cm_ok[k];
          if (pushed) { if (seen == t) { src = k; break; } seen++; }
        }
      }
      s_valid = valid_t; s_src = src; s_pushed_t = pushed_t;
      a.cm_eff[t] = pushed_t;
      if (valid_t) {
        if (t < total) { if (src != t) atomicAdd(&st_rw->pfg_shifted, 1ull); } else atomicAdd(&st_rw->pfg_oob, 1ull);
      }
      if (t == 0) st_rw->num_residualized = s_cnt + (unsigned long long)nvalid_tail;
    }
  }
  Gp::sync(grp);
  stamp();  // bookkeeping
  const int o0 = a.obs_off[t], L = a.obs_off[t + 1] - o0, L2 = 2 * L;
  const int valid = (L >= 2) ? s_valid : 0, src = s_src;  // fewer than two observations: no null space (2L - 3 < 1)
  double* Zr = a.Z + (size_t)3 * t * c;
  double* Yr = a.Yq + (size_t)3 * t * c;
  if (tid == 0) { a.valid[t] = valid; a.src[t] = src; }
  if (!valid) {  // not residualised: contributes nothing
    for (int k = tid; k < 3 * c; k += G) { Zr[k] = 0.0; Yr[k] = 0.0; }
    if (tid == 0) { a.accept[t] = 0; a.gamma[t] = S(0); a.rows[t] = 0; a.ur[3 * t] = a.ur[3 * t + 1] = a.ur[3 * t + 2] = 0.0; }
    return;
  }
  // ------------------------------------------------------------------ shared-memory carve-up
  S* r = reinterpret_cast<S*>(gmem_sm);
  S* X = r + L2;
  S* V = X + 12 * L;
  S* Ut = X;  // [3][2L]  U^T rounded to S, the gate's right-hand sides after z = r (X is dead by then)
  S* Y = X + jac_xv_elems<S>(L);
  S* PnT = reinterpret_cast<S*>((reinterpret_cast<uintptr_t>(Ut + 6 * L) + 15) & ~uintptr_t(15));  // [8][Rp]; V is dead by then
  const int Rp = jac_panel_rows(L);  // >= 2L + 4 rows, multiple of 4
  const int* idx = a.clone_idx + o0;
  const S* z = a.obs + 2 * (size_t)o0;
  const DevState<S>* st = a.st;
  const S g[3] = {st->g[0], st->g[1], st->g[2]};
  const S* pfsrc = mode ? (a.pfg_given + 3 * t) : (a.pfg + 3 * src);
  const S pf[3] = {pfsrc[0], pfsrc[1], pfsrc[2]};
  // ---- residual + measurement Jacobian blocks with the observability projection (msckf.h:915-950, 960-978)
  for (int i = tid; i < L; i += G) {
    const S* ps = poses + kPoseStride * idx[i];
    S C[9];
    quat_to_rot(ps, C);
    const S d[3] = {pf[0] - ps[4], pf[1] - ps[5], pf[2] - ps[6]};
    const S pc[3] = {C[0] * d[0] + C[1] * d[1] + C[2] * d[2], C[3] * d[0] + C[4] * d[1] + C[5] * d[2],
                     C[6] * d[0] + C[7] * d[1] + C[8] * d[2]};
    const S Xc = pc[0], Yc = pc[1], Zc = pc[2];
    const S r0 = z[2 * i] - Xc / Zc, r1 = z[2 * i + 1] - Yc / Zc;
    r[2 * i] = r0; r[2 * i + 1] = r1;
    a.rg[2 * (size_t)(o0 + i)] = r0; a.rg[2 * (size_t)(o0 + i) + 1] = r1;
    const S iz = S(1) / Zc;
    const S J[2][3] = {{S(1) * iz, S(0) * iz, (-Xc / Zc) * iz}, {S(0) * iz, S(1) * iz, (-Yc / Zc) * iz}};
    const S sk[3][3] = {{S(0), -pc[2], pc[1]}, {pc[2], S(0), -pc[0]}, {-pc[1], pc[0], S(0)}};
    S A[2][6];
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        A[q][b] = J[q][0] * sk[0][b] + J[q][1] * sk[1][b] + J[q][2] * sk[2][b];
        A[q][3 + b] = -(J[q][0] * C[b] + J[q][1] * C[3 + b] + J[q][2] * C[6 + b]);
      }
    S u[6];
    u[0] = C[0] * g[0] + C[1] * g[1] + C[2] * g[2];
    u[1] = C[3] * g[0] + C[4] * g[1] + C[5] * g[2];
    u[2] = C[6] * g[0] + C[7] * g[1] + C[8] * g[2];
    u[3] = -d[2] * g[1] + d[1] * g[2];  // skew(d) * g
    u[4] = d[2] * g[0] - d[0] * g[2];
    u[5] = -d[1] * g[0] + d[0] * g[1];
    S uu = 0;
#pragma unroll
    for (int b = 0; b < 6; ++b) uu += u[b] * u[b];
    const S iuu = S(1) / uu;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      S Au = 0;
#pragma unroll
      for (int b = 0; b < 6; ++b) Au += A[q][b] * u[b];
#pragma unroll
      for (int b = 0; b < 6; ++b) {
        const S hx = A[q][b] - Au * iuu * u[b];
        X[12 * i + 6 * q + b] = hx;
        a.Xg[12 * (size_t)(o0 + i) + 6 * q + b] = hx;
        if (b >= 3) V[3 * (2 * i + q) + (b - 3)] = -hx;  // H_f = -H_x(:,3:6)
      }
    }
  }
  Gp::sync(grp);
  stamp();  // X, r
  // ---- warp 0: column-pivoted Householder QR of H_f (2L x 3) -- the trailing 2L-3 columns of Q are A_j
  // (msckf.h:954-955) -- then U and U^T r, all warp-synchronous (shuffle reductions, no CTA barriers).  Warps 1..3
  // meanwhile: Y = X P_sub X^T + u_var I.
  __shared__ double s_urv_[Gp::TPC][3];
  __shared__ double s_sd_[Gp::TPC][9];
  double* s_urv = s_urv_[grp];
  double* s_sd = s_sd_[grp];
  const int warp = tid >> 5;
  if (warp == 0) {
    S tau[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      S nn[3] = {S(-1), S(-1), S(-1)};
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) {
        if (cc < k) continue;
        S sacc = 0;
        _Pragma("unroll 1") for (int row = k + lane; row < L2; row += 32) sacc += V[3 * row + cc] * V[3 * row + cc];
        nn[cc] = warp_sum_call(sacc);
      }
      int piv = k;
      S best = nn[k];
#pragma unroll
      for (int cc = 1; cc < 3; ++cc)
        if (cc > k && nn[cc] > best) { best = nn[cc]; piv = cc; }
      if (piv != k)
        _Pragma("unroll 1") for (int row = lane; row < L2; row += 32) { const S tmp = V[3 * row + k]; V[3 * row + k] = V[3 * row + piv]; V[3 * row + piv] = tmp; }
      __syncwarp();
      S tacc = 0;
      _Pragma("unroll 1") for (int row = k + 1 + lane; row < L2; row += 32) tacc += V[3 * row + k] * V[3 * row + k];
      const S tail = warp_sum_call(tacc);
      const S c0 = V[3 * k + k];
      S beta, tk;
      __syncwarp();
      if (tail <= S(sizeof(S) == 4 ? 1.17549435e-38 : 2.2250738585072014e-308)) {
        beta = c0; tk = S(0);
        _Pragma("unroll 1") for (int row = k + 1 + lane; row < L2; row += 32) V[3 * row + k] = S(0);
      } else {
        beta = tsqrt<S>(c0 * c0 + tail);
        if (c0 >= S(0)) beta = -beta;
        const S dd = c0 - beta;
        _Pragma("unroll 1") for (int row = k + 1 + lane; row < L2; row += 32) V[3 * row + k] /= dd;
        tk = (beta - c0) / beta;
      }
      tau[k] = tk;
      __syncwarp();
      if (tk != S(0)) {
#pragma unroll
        for (int cc = 1; cc < 3; ++cc) {
          if (cc <= k) continue;
          S sacc = 0;
          _Pragma("unroll 1") for (int row = k + 1 + lane; row < L2; row += 32) sacc += V[3 * row + k] * V[3 * row + cc];
          S sdot = warp_sum_call(sacc) + V[3 * k + cc];
          sdot *= tk;
          __syncwarp();
          _Pragma("unroll 1") for (int row = k + 1 + lane; row < L2; row += 32) V[3 * row + cc] -= V[3 * row + k] * sdot;
          if (lane == 0) V[3 * k + cc] -= sdot;
          __syncwarp();
        }
      }
      if (lane == 0) {
        V[3 * k + k] = S(1);                                // unit diagonal of the Householder vector
        for (int row = 0; row < k; ++row) V[3 * row + k] = S(0);  // zero above: V(:,k) is the full vector v_k
      }
      __syncwarp();
    }
    // export v_k, tau for the explicit-row kernel
    _Pragma("unroll 1") for (int e = lane; e < 3 * L2; e += 32) a.Vg[3 * 2 * (size_t)o0 + e] = V[e];
    if (lane < 3) { a.taug[3 * t + lane] = tau[lane == 0 ? 0 : (lane == 1 ? 1 : 2)]; }
    // ---- exact reflectors for the Gram stage: H_k = I - tau64_k v_k v_k^T with tau64_k = 2 / (v_k^T v_k) in fp64, so
    // that Q = H_0 H_1 H_2 is orthogonal to 1e-16 whatever the filter precision: G_j = I - U_j U_j^T is an exact
    // projector and the body Gram terms and the explicit rows (k_rows) describe the same H_o.
    double tau64[3];
    {
      double vv3[3] = {0.0, 0.0, 0.0};
      _Pragma("unroll 1") for (int row = lane; row < L2; row += 32) {  // v_k is zero above row k
        const S v0 = V[3 * row], v1 = V[3 * row + 1], v2 = V[3 * row + 2];
        vv3[0] += (double)v0 * (double)v0; vv3[1] += (double)v1 * (double)v1; vv3[2] += (double)v2 * (double)v2;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) { vv3[k] = warp_sum_call(vv3[k]); tau64[k] = (tau[k] != S(0)) ? 2.0 / vv3[k] : 0.0; }
    }
    // ---- U = Q(:,0:3) = H0 H1 H2 [I3; 0]  (fp64), kept as the nine coefficients sd_k of u_row
    double sd[9];
#pragma unroll
    for (int k = 2; k >= 0; --k) {
      double s3[3] = {0.0, 0.0, 0.0};
      _Pragma("unroll 1") for (int row = k + lane; row < L2; row += 32) {
        const double vk = (double)V[3 * row + k];
        double u[3];
        u_row(V, sd, row, k + 1, u);
        s3[0] += vk * u[0]; s3[1] += vk * u[1]; s3[2] += vk * u[2];
      }
#pragma unroll
      for (int q = 0; q < 3; ++q) sd[3 * k + q] = warp_sum_call(s3[q]) * tau64[k];
    }
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < 9; ++q) s_sd[q] = sd[q];
    }
    // U^T r in fp64 from the raw residual
    {
      double urv[3] = {0.0, 0.0, 0.0};
      _Pragma("unroll 1") for (int row = lane; row < L2; row += 32) {
        const double rr = (double)r[row];
        double u[3];
        u_row(V, sd, row, 0, u);
        urv[0] += u[0] * rr; urv[1] += u[1] * rr; urv[2] += u[2] * rr;
      }
#pragma unroll
      for (int q = 0; q < 3; ++q) urv[q] = warp_sum_call(urv[q]);
      if (lane == 0) { s_urv[0] = urv[0]; s_urv[1] = urv[1]; s_urv[2] = urv[2]; }
    }
  }
  if (G == 32 || warp != 0) {  // (a single-warp group does both, one after the other)
    // ---- gating (msckf.h:1103-1124): gamma = r_o^T (H_o P H_o^T + u_var I)^-1 r_o with H_o = (Q^T X)[3:]
    // Y = X P_sub X^T + u_var I, symmetric 2L x 2L, packed lower, by 2 x 2 blocks (i, k), k <= i.  Block rows i and L-1-i share a pass
    // of L + 1 blocks (lane e takes (i, e) for e <= i, else (L-1-i, e-i-1)): no pair decode, and the lanes of a pass read P
    // along the same two block rows.  Each block's sums run in the same order whichever thread computes it.
    const S* P = a.P;
    const int ldp = a.ldp;
    const S uvar = st->u_var;
    constexpr int YW = (G == 32) ? 1 : G / 32 - 1;  // warps on the pairs
    for (int ps = (G == 32) ? 0 : warp - 1; ps < (L + 1) / 2; ps += YW) {
      const int ilo = ps, ihi = L - 1 - ps, ne = (ilo == ihi) ? ilo + 1 : L + 1;
      for (int e = lane; e < ne; e += 32) {
        const int i = (e <= ilo) ? ilo : ihi, k = (e <= ilo) ? e : e - ilo - 1;
        const S* Pb = P + (ptrdiff_t)(kImuDim + 6 * idx[i]) * ldp + (kImuDim + 6 * idx[k]);
        const S* Xi = X + 12 * i;
        S T0[6], T1[6];
#pragma unroll
        for (int b = 0; b < 6; ++b) { T0[b] = S(0); T1[b] = S(0); }
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const S x0 = Xi[q], x1 = Xi[6 + q];
          S pv[6];
          ld6_odd(Pb + (ptrdiff_t)q * ldp, pv);
#pragma unroll
          for (int b = 0; b < 6; ++b) {
            T0[b] += x0 * pv[b];
            T1[b] += x1 * pv[b];
          }
        }
        S xk[12];
#pragma unroll
        for (int h = 0; h < 6; ++h) ld2(X + 12 * k + 2 * h, xk[2 * h], xk[2 * h + 1]);
        S y00 = 0, y01 = 0, y10 = 0, y11 = 0;
#pragma unroll
        for (int b = 0; b < 6; ++b) {
          y00 += T0[b] * xk[b]; y01 += T0[b] * xk[6 + b];
          y10 += T1[b] * xk[b]; y11 += T1[b] * xk[6 + b];
        }
        S* y0 = Y + pk(2 * i, 2 * k);
        S* y1 = y0 + 2 * i + 1;  // pk(2i + 1, 2k)
        y0[0] = (i == k) ? y00 + uvar : y00;
        y1[0] = y10;
        y1[1] = (i == k) ? y11 + uvar : y11;
        if (i != k) y0[1] = y01;
      }
    }
  }
  Gp::sync(grp);
  stamp();  // QR, U (warp 0) | Y pairs (warps 1..3)
  // ---- compact outputs for the Gram stage, written as if accepted (X's shared memory is about to become U^T); a rejected
  // track zeroes them again after the gate
  for (int k = tid; k < 3 * c; k += G) { Zr[k] = 0.0; Yr[k] = 0.0; }
  double Mm[6];  // M = U^T D U (3x3 symmetric), D = diag(u_var, v_var, u_var, ...)
  const double du = (double)st->u_var, dv = (double)st->v_var;
  group_vsum<G, 6>(Mm, [&](int v, double (&p)[6]) {
    for (int k = 0; k < 6; ++k) p[k] = 0.0;
    for (int row = v; row < L2; row += 128) {
      const double dd = (row & 1) ? dv : du;
      double u[3];
      u_row(V, s_sd, row, 0, u);
      const double u0 = u[0], u1 = u[1], u2 = u[2];
      p[0] += dd * u0 * u0; p[1] += dd * u0 * u1; p[2] += dd * u0 * u2;
      p[3] += dd * u1 * u1; p[4] += dd * u1 * u2; p[5] += dd * u2 * u2;
    }
  }, redd, grp);
  const double M3[3][3] = {{Mm[0], Mm[1], Mm[2]}, {Mm[1], Mm[3], Mm[4]}, {Mm[2], Mm[4], Mm[5]}};
  Gp::sync(grp);
  {
    for (int e = tid; e < L * 6; e += G) {
      const int i = e / 6, b = e % 6;
      const int col = 6 * idx[i] + b;
      const double xa = X[12 * i + b], xb = X[12 * i + 6 + b];
      double zb[3], yb[3], uA[3], uB[3];
      u_row(V, s_sd, 2 * i, 0, uA);
      u_row(V, s_sd, 2 * i + 1, 0, uB);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const double ua = uA[q], ub = uB[q];
        zb[q] = ua * xa + ub * xb;
        yb[q] = du * ua * xa + dv * ub * xb;
      }
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        Zr[(size_t)q * c + col] = zb[q];
        Yr[(size_t)q * c + col] = yb[q] - 0.5 * (M3[q][0] * zb[0] + M3[q][1] * zb[1] + M3[q][2] * zb[2]);
      }
    }
  }
  Gp::sync(grp);  // X is dead: U^T takes its place
  // ---- gate (msckf.h:1103-1124) without forming S = A^T Y A + u_var I: with M = Y + u_var I (SPD) and [U A] orthogonal,
  // the Schur complement of (Q^T M Q)^-1 = Q^T M^-1 Q gives
  //   gamma = r_o^T S^-1 r_o = z^T M^-1 z - (U^T M^-1 z)^T (U^T M^-1 U)^-1 (U^T M^-1 z),  z = A r_o = r - U (U^T r),
  // so with M = L L^T, a = L^-1 z, B = L^-1 U and c = B^T a:  gamma = a^T a - c^T (B^T B)^-1 c.  The right-hand sides of the
  // Cholesky of M are z (in r's place) and the three columns of U (rows of U^T).
  for (int row = tid; row < L2; row += G) {
    double u[3];
    u_row(V, s_sd, row, 0, u);
    r[row] = (S)((double)r[row] - (u[0] * s_urv[0] + u[1] * s_urv[1] + u[2] * s_urv[2]));
    Ut[row] = (S)u[0]; Ut[L2 + row] = (S)u[1]; Ut[2 * L2 + row] = (S)u[2];
  }
  Gp::sync(grp);  // V is dead: PnT takes its place
  stamp();  // compact outputs, right-hand sides
  __shared__ int s_chol_fail[Gp::TPC];
  bool chol_ok = gate_chol_blocked<S, G>(Y, r, L2, PnT, Rp, &s_chol_fail[grp], grp);
  // a^T a, c = B^T a, B^T B (00 01 02 11 12 22): r holds a, Ut holds B^T
  S qf[10];
  group_vsum<G, 10>(qf, [&](int v, S (&p)[10]) {
    for (int k = 0; k < 10; ++k) p[k] = S(0);
    for (int j = v; j < L2; j += 128) {
      const S aj = r[j], b0 = Ut[j], b1 = Ut[L2 + j], b2 = Ut[2 * L2 + j];
      p[0] += aj * aj; p[1] += b0 * aj; p[2] += b1 * aj; p[3] += b2 * aj;
      p[4] += b0 * b0; p[5] += b0 * b1; p[6] += b0 * b2; p[7] += b1 * b1; p[8] += b1 * b2; p[9] += b2 * b2;
    }
  }, reds, grp);
  // c^T (B^T B)^-1 c = |l^-1 c|^2 with B^T B = l l^T (3 x 3, in registers)
  const S l00 = tsqrt<S>(qf[4]), l10 = qf[5] / l00, l20 = qf[6] / l00;
  const S d11 = qf[7] - l10 * l10, l11 = tsqrt<S>(d11), l21 = (qf[8] - l20 * l10) / l11;
  const S d22 = qf[9] - (l20 * l20 + l21 * l21), l22 = tsqrt<S>(d22);
  const S w0 = qf[1] / l00, w1 = (qf[2] - l10 * w0) / l11, w2 = (qf[3] - (l20 * w0 + l21 * w1)) / l22;
  if (!(qf[4] > S(0) && d11 > S(0) && d22 > S(0))) chol_ok = false;
  S gam = qf[0] - ((w0 * w0 + w1 * w1) + w2 * w2);
  const int acc = chol_ok && (gam < st->chi2[L]);  // table[dof+1], dof = L-1 (msckf.h:433,:1117)
  if (!chol_ok) gam = S(1e30);
  stamp();  // Cholesky + gamma
  if (!acc) {
    for (int e = tid; e < L * 6; e += G) {
      const int col = 6 * idx[e / 6] + e % 6;
#pragma unroll
      for (int q = 0; q < 3; ++q) { Zr[(size_t)q * c + col] = 0.0; Yr[(size_t)q * c + col] = 0.0; }
    }
  }
  if (tid == 0) {
    a.accept[t] = acc;
    a.gamma[t] = gam;
    a.rows[t] = acc ? (L2 - 3) : 0;
    for (int q = 0; q < 3; ++q) a.ur[3 * t + q] = acc ? s_urv[q] : 0.0;
  }
  stamp();  // outputs
  if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) a.prof[40 + prof_i] = 0ull;
}

// (G = 32, fp32: 10 CTAs = 20 tracks per SM, the 2 640 resident tracks a batch of 8 config-B filters needs to run in one
// wave -- 96 registers and 10 x (2 x 10.3 KB) of shared memory at L = 30)
template <class S, int G>
__global__ void __launch_bounds__(JGrp<G>::CT, (G == 32) ? (sizeof(S) == 4 ? 10 : 5) : (sizeof(S) == 4 ? 5 : 3)) k_jac(const UpdArgs<S>* __restrict__ args) {
  pdl_wait();
  const UpdArgs<S>& a = args[blockIdx.z];
  constexpr int TPC = JGrp<G>::TPC, CT = JGrp<G>::CT;
  const int N = a.n_tracks;
  if ((int)blockIdx.x * TPC >= N) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const S* poses = a.poses;
  unsigned char* wp = smem_raw;
  if (G != 32) {
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
    S* ps = reinterpret_cast<S*>(smem_raw + 16);
    stage_table_tma(ps, a.poses, (unsigned)(a.M * kPoseStride * sizeof(S)), bar);
    poses = ps;
    wp += 16 + sizeof(S) * kPoseStride * (size_t)a.M;
    wp = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(wp) + 15) & ~uintptr_t(15));
  }
  // group_vsum's slots, one array per element type so that every group of the CTA owns its own bytes in both (the groups of
  // a CTA synchronise only among themselves): 6 doubles (M = U^T D U) and 10 S (the gate's quadratic forms) per virtual warp;
  // a single-warp group reduces by shuffles alone
  __shared__ double redd[(G == 32) ? 1 : TPC * 4 * 6];
  __shared__ S reds[(G == 32) ? 1 : TPC * 4 * 10];
  __shared__ int redi[CT / 32];
  const int grp = threadIdx.x / G, t = blockIdx.x * TPC + grp;
  if (t < N) jac_track<S, G>(a, t, grp, wp + (size_t)grp * jac_group_bytes<S>(a.Lmax), poses, redd, reds, redi);
  jac_finish<S, CT>(a, (N + TPC - 1) / TPC);
}

}  // namespace mb
