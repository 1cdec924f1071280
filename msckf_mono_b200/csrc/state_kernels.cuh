// msckf_mono_b200/csrc/state_kernels.cuh
// Device-resident rest of the MSCKF<_S> surface so the covariance never leaves the GPU:
//   k_propagate : msckf.h:101-145 (calcF :874-890, calcG :892-903, propogateImuStateRK :1425-1467,
//                 Phi = exp(F dT) with Eigen's Pade degree selection, observability constraints :116-132)
//   k_augment   : msckf.h:148-212
//   k_gather    : covariance slicing of pruneEmptyStates / pruneRedundantStates (matrix_utils.h:58-87)
// Each runs one filter or, with the filter index in the block index, a device batch of filters (msckf_b200_batch_*).
// Arithmetic is carried out in the filter precision _S like the reference.
#pragma once
#include "common.cuh"

namespace mb {

template <class S> struct ExpmPick;
template <> struct ExpmPick<float> {
  __device__ static int pick(double l1, int& sq) {
    sq = 0;
    if (l1 < 4.258730016922831e-001) return 3;
    if (l1 < 1.880152677804762e+000) return 5;
    frexp(l1 / 3.925724783138660, &sq);
    if (sq < 0) sq = 0;
    return 7;
  }
};
template <> struct ExpmPick<double> {
  __device__ static int pick(double l1, int& sq) {
    sq = 0;
    if (l1 < 1.495585217958292e-002) return 3;
    if (l1 < 2.539398330063230e-001) return 5;
    if (l1 < 9.504178996162932e-001) return 7;
    if (l1 < 2.097847961257068e+000) return 9;
    frexp(l1 / 5.371920351148152, &sq);
    if (sq < 0) sq = 0;
    return 13;
  }
};

// 15x15 helpers on shared-memory matrices (row-major, ld 15); all 256 threads call them.
template <class S>
__device__ __forceinline__ void mm15(S* C, const S* A, const S* B) {  // C = A*B  (C must not alias)
  const int t = threadIdx.x;
  if (t < 225) {
    const int i = t / 15, j = t % 15;
    S s = 0;
#pragma unroll
    for (int k = 0; k < 15; ++k) s += A[15 * i + k] * B[15 * k + j];
    C[t] = s;
  }
  __syncthreads();
}
template <class S>
__device__ __forceinline__ void mm15_nt(S* C, const S* A, const S* B) {  // C = A*B^T
  const int t = threadIdx.x;
  if (t < 225) {
    const int i = t / 15, j = t % 15;
    S s = 0;
#pragma unroll
    for (int k = 0; k < 15; ++k) s += A[15 * i + k] * B[15 * j + k];
    C[t] = s;
  }
  __syncthreads();
}
// C = sum_k coef[k] * M[k]   (nterm <= 5)
template <class S>
__device__ __forceinline__ void lin15(S* C, int nterm, const double* coef, const S* const* Ms) {
  const int t = threadIdx.x;
  if (t < 225) {
    S s = 0;
    for (int k = 0; k < nterm; ++k) s += (S)coef[k] * Ms[k][t];
    C[t] = s;
  }
  __syncthreads();
}

// first lane (among `active` ones) holding the largest non-negative value: two / three REDUX instructions instead of a
// five-level shuffle tree (the pivot search was 40 % of k_propagate's LU step)
__device__ __forceinline__ int warp_argmax_first(float v, bool active, int lane) {
  const unsigned b = active ? __float_as_uint(v) : 0u;  // non-negative floats order like their bit patterns
  const unsigned m = __reduce_max_sync(0xffffffffu, b);
  return (int)__reduce_min_sync(0xffffffffu, (active && b == m) ? (unsigned)lane : 31u);
}
__device__ __forceinline__ int warp_argmax_first(double v, bool active, int lane) {
  const unsigned hi = active ? (unsigned)__double2hiint(v) : 0u, lo = (unsigned)__double2loint(v);
  const unsigned mhi = __reduce_max_sync(0xffffffffu, hi);
  const bool c1 = active && hi == mhi;
  const unsigned mlo = __reduce_max_sync(0xffffffffu, c1 ? lo : 0u);
  return (int)__reduce_min_sync(0xffffffffu, (c1 && lo == mlo) ? (unsigned)lane : 31u);
}

// The state kernels take their per-filter arguments by value, so that a call needs no staging buffer and no synchronisation.
// One body serves a single filter (NM = 1) and a device batch (NM = kBatchMembers): the member is the block index (k_propagate,
// k_augment: one CTA per member) or the grid row (k_gather).  A batch of more members runs as one launch per kBatchMembers.
constexpr int kBatchMembers = 32;  // 32 fp64 propagate members are 29 952 B: under sm_90's 32 764 B of kernel parameters
template <class T, int NM>
struct Members { T m[NM]; };

// Up to kPropMax IMU readings per launch and member (msckf_b200_propagate_n: the shim queues the readings between two images).
// The readings are applied one after the other with exactly the arithmetic of a single propagate() each.
constexpr int kPropMax = 16;
template <class S>
struct PropBatch {
  DevState<S>* st;
  S* P;
  int ldp, M, k, pad_;
  unsigned long long* prof;  // optional %globaltimer stamps of the first reading's phases (profiling aid)
  S r[kPropMax][7];  // omega[3], a[3], dT
};
static_assert(sizeof(Members<PropBatch<double>, kBatchMembers>) <= 32764, "k_propagate's batched arguments exceed the parameter limit");

template <class S, int NM>
__global__ void __launch_bounds__(256) k_propagate(const Members<PropBatch<S>, NM> a) {
  // The IMU state, the 15 x 15 IMU block of P and (for windows up to 85 clones) the thread's columns of P_IC stay on chip
  // across the readings of the batch: one global round trip per launch instead of one per reading and serial section.
  // (Fields are read from the parameter bank one at a time: a reference to a.m[f] would copy the member to local memory.)
  const int f = NM == 1 ? 0 : blockIdx.x;
  DevState<S>* gst = a.m[f].st;
  int prof_i = 0;
  auto stamp = [&]() {
    if (a.m[f].prof && threadIdx.x == 0 && prof_i < 16) a.m[f].prof[prof_i++] = globaltimer();
  };
  stamp();
  __shared__ DevState<S> s_state;
  DevState<S>* st = &s_state;
  S* __restrict__ P = a.m[f].P;
  const int ldp = a.m[f].ldp, M = a.m[f].M;
  {
    static_assert(sizeof(DevState<S>) % 4 == 0, "DevState is copied word-wise");
    const unsigned* src = reinterpret_cast<const unsigned*>(gst);
    unsigned* dst = reinterpret_cast<unsigned*>(&s_state);
    for (int e = threadIdx.x; e < (int)(sizeof(DevState<S>) / 4); e += 256) dst[e] = src[e];
  }
  __shared__ S PII[225];
  if (threadIdx.x < 225) PII[threadIdx.x] = P[(size_t)(threadIdx.x / 15) * ldp + threadIdx.x % 15];
  const int c_all = 6 * M;
  const bool cols_in_regs = c_all <= 512;
  S vcol[2][15];
  if (cols_in_regs) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int col = threadIdx.x + 256 * u;
#pragma unroll
      for (int k = 0; k < 15; ++k) vcol[u][k] = (col < c_all) ? P[(size_t)k * ldp + 15 + col] : S(0);
    }
  }
  __shared__ S F[225], Phi[225], A2[225], A4[225], A6[225], A8[225], Um[225], Vm[225], Tm[225], Id[225];
  __shared__ S G[15 * 12], GQ[15 * 12];
  __shared__ S CT[9];            // C_IG^T
  __shared__ S prop_q[4], prop_v[3], prop_p[3];
  __shared__ int s_deg, s_sq;
  __shared__ S colsum[15];
  const int t = threadIdx.x;
  stamp();  // state, P_II and P_IC columns on chip
  for (int ir = 0; ir < a.m[f].k; ++ir) {
  const S wx = a.m[f].r[ir][0], wy = a.m[f].r[ir][1], wz = a.m[f].r[ir][2], ax = a.m[f].r[ir][3], ay = a.m[f].r[ir][4],
          az = a.m[f].r[ir][5], dT = a.m[f].r[ir][6];
  __syncthreads();
  if (t < 225) { F[t] = S(0); Id[t] = ((t / 15) == (t % 15)) ? S(1) : S(0); }
  if (t < 180) G[t] = S(0);
  __syncthreads();
  if (t == 0) {
    // ---- calcF / calcG
    const S oh[3] = {wx - st->b_g[0], wy - st->b_g[1], wz - st->b_g[2]};
    const S ah[3] = {ax - st->b_a[0], ay - st->b_a[1], az - st->b_a[2]};
    S C[9];
    quat_to_rot(st->q_IG, C);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) CT[3 * i + j] = C[3 * j + i];
    const S so[9] = {S(0), -oh[2], oh[1], oh[2], S(0), -oh[0], -oh[1], oh[0], S(0)};
    const S sa[9] = {S(0), -ah[2], ah[1], ah[2], S(0), -ah[0], -ah[1], ah[0], S(0)};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        F[15 * i + j] = -so[3 * i + j];
        S s = 0;
        for (int k = 0; k < 3; ++k) s += CT[3 * i + k] * sa[3 * k + j];
        F[15 * (6 + i) + j] = -s;
        F[15 * (6 + i) + 9 + j] = -CT[3 * i + j];
        G[12 * (6 + i) + 6 + j] = -CT[3 * i + j];
      }
    for (int i = 0; i < 3; ++i) {
      F[15 * i + 3 + i] = S(-1);
      F[15 * (12 + i) + 6 + i] = S(1);
      G[12 * i + i] = S(-1);
      G[12 * (3 + i) + 3 + i] = S(1);
      G[12 * (9 + i) + 9 + i] = S(1);
    }
    // ---- propogateImuStateRK (msckf.h:1425-1467)
    S O[4][4];
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) O[i][j] = S(0);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) O[i][j] = S(0.5) * (-so[3 * i + j]);
      O[i][3] = S(0.5) * oh[i];
      O[3][i] = S(0.5) * (-oh[i]);
    }
    const S y0[4] = {-st->q_IG[0], -st->q_IG[1], -st->q_IG[2], st->q_IG[3]};
    S k0[4], k1[4], k2[4], k3[4], k4[4], k5[4], y[4];
#define MB_MV(dst, src) for (int i_ = 0; i_ < 4; ++i_) dst[i_] = O[i_][0] * src[0] + O[i_][1] * src[1] + O[i_][2] * src[2] + O[i_][3] * src[3];
    MB_MV(k0, y0);
    for (int i = 0; i < 4; ++i) y[i] = y0[i] + (k0[i] / S(4.)) * dT;
    MB_MV(k1, y);
    for (int i = 0; i < 4; ++i) y[i] = y0[i] + (k0[i] / S(8.) + k1[i] / S(8.)) * dT;
    MB_MV(k2, y);
    for (int i = 0; i < 4; ++i) y[i] = y0[i] + (-k1[i] / S(2.) + k2[i]) * dT;
    MB_MV(k3, y);
    for (int i = 0; i < 4; ++i) y[i] = y0[i] + (k0[i] * S(3.) / S(16.) + k3[i] * S(9.) / S(16.)) * dT;
    MB_MV(k4, y);
    for (int i = 0; i < 4; ++i)
      y[i] = y0[i] + (-k0[i] * S(3.) / S(7.) + k1[i] * S(2.) / S(7.) + k2[i] * S(12.) / S(7.) - k3[i] * S(12.) / S(7.) + k4[i] * S(8.) / S(7.)) * dT;
    MB_MV(k5, y);
#undef MB_MV
    S yt[4];
    for (int i = 0; i < 4; ++i) yt[i] = y0[i] + (S(7.) * k0[i] + S(32.) * k2[i] + S(12.) * k3[i] + S(32.) * k4[i] + S(7.) * k5[i]) * dT / S(90.);
    S q[4] = {-yt[0], -yt[1], -yt[2], yt[3]};
    quat_normalize(q);
    for (int i = 0; i < 4; ++i) prop_q[i] = q[i];
    for (int i = 0; i < 3; ++i) {
      const S acc = CT[3 * i] * ah[0] + CT[3 * i + 1] * ah[1] + CT[3 * i + 2] * ah[2] + st->g[i];
      prop_v[i] = st->v_I_G[i] + acc * dT;
      prop_p[i] = st->p_I_G[i] + st->v_I_G[i] * dT;
    }
  }
  __syncthreads();
  stamp();  // calcF / calcG / RK
  // ---- F *= dT ; Phi = exp(F)  (unsupported/Eigen MatrixExponential restated)
  if (t < 225) F[t] *= dT;
  __syncthreads();
  if (t < 15) {
    double s = 0;
    for (int i = 0; i < 15; ++i) s += fabs((double)F[15 * i + t]);
    colsum[t] = (S)s;
  }
  __syncthreads();
  if (t == 0) {
    double l1 = 0;
    for (int j = 0; j < 15; ++j) l1 = fmax(l1, (double)colsum[j]);
    int sq;
    s_deg = ExpmPick<S>::pick(l1, sq);
    s_sq = sq;
  }
  __syncthreads();
  const int deg = s_deg, sq = s_sq;
  if (sq > 0) {
    if (t < 225) F[t] *= (S)ldexp(1.0, -sq);
    __syncthreads();
  }
  mm15(A2, F, F);
  if (deg == 3) {
    const double cu[2] = {1.0, 60.0}, cv[2] = {12.0, 120.0};
    const S* ms[2] = {A2, Id};
    lin15(Tm, 2, cu, ms);
    mm15(Um, F, Tm);
    lin15(Vm, 2, cv, ms);
  } else if (deg == 5) {
    mm15(A4, A2, A2);
    const double cu[3] = {1.0, 420.0, 15120.0}, cv[3] = {30.0, 3360.0, 30240.0};
    const S* ms[3] = {A4, A2, Id};
    lin15(Tm, 3, cu, ms);
    mm15(Um, F, Tm);
    lin15(Vm, 3, cv, ms);
  } else if (deg == 7) {
    mm15(A4, A2, A2);
    mm15(A6, A4, A2);
    const double cu[4] = {1.0, 1512.0, 277200.0, 8648640.0}, cv[4] = {56.0, 25200.0, 1995840.0, 17297280.0};
    const S* ms[4] = {A6, A4, A2, Id};
    lin15(Tm, 4, cu, ms);
    mm15(Um, F, Tm);
    lin15(Vm, 4, cv, ms);
  } else if (deg == 9) {
    mm15(A4, A2, A2);
    mm15(A6, A4, A2);
    mm15(A8, A6, A2);
    const double cu[5] = {1.0, 3960.0, 2162160.0, 302702400.0, 8821612800.0};
    const double cv[5] = {90.0, 110880.0, 30270240.0, 2075673600.0, 17643225600.0};
    const S* ms[5] = {A8, A6, A4, A2, Id};
    lin15(Tm, 5, cu, ms);
    mm15(Um, F, Tm);
    lin15(Vm, 5, cv, ms);
  } else {
    mm15(A4, A2, A2);
    mm15(A6, A4, A2);
    const double b[14] = {64764752532480000.0, 32382376266240000.0, 7771770303897600.0, 1187353796428800.0,
                          129060195264000.0, 10559470521600.0, 670442572800.0, 33522128640.0, 1323241920.0,
                          40840800.0, 960960.0, 16380.0, 182.0, 1.0};
    {
      const double c1[3] = {b[13], b[11], b[9]};
      const S* ms[3] = {A6, A4, A2};
      lin15(Vm, 3, c1, ms);
    }
    mm15(Tm, A6, Vm);
    {
      const double c2[5] = {1.0, b[7], b[5], b[3], b[1]};
      const S* ms[5] = {Tm, A6, A4, A2, Id};
      lin15(A8, 5, c2, ms);
    }
    mm15(Um, F, A8);
    {
      const double c3[3] = {b[12], b[10], b[8]};
      const S* ms[3] = {A6, A4, A2};
      lin15(Tm, 3, c3, ms);
    }
    mm15(A8, A6, Tm);
    {
      const double c4[5] = {1.0, b[6], b[4], b[2], b[0]};
      const S* ms[5] = {A8, A6, A4, A2, Id};
      lin15(Vm, 5, c4, ms);
    }
  }
  // (V - U) Phi = (V + U): partial-pivot LU on the 15x30 augmented system [den | num]
  if (t < 225) { Tm[t] = Vm[t] - Um[t]; Phi[t] = Vm[t] + Um[t]; }
  __syncthreads();
  stamp();  // Pade numerator / denominator
  // partial-pivot LU of the 15 x 30 system [den | num] and the back substitution on ONE warp, __syncwarp only (the CTA-wide
  // form cost five block barriers per pivot).  Same operations as before (first largest |pivot|, multiplier by division,
  // multiply-subtract), arranged for a SHORT instruction stream -- this kernel's body is ~90 KB of SASS and whatever runs once
  // per reading is fetched cold: the pivot is a warp arg-max (5 shuffle steps), lane = ROW for the elimination (one division
  // per lane, a rolled loop along the row; stride 15 words: conflict-free), lane = column for the row swap and the back
  // substitution (rolled).  (Measured: unrolled per-column register forms of this were slower.)
  if (t < 32) {
    S* Mx = (t < 15) ? Tm : Phi;
    const int j = (t < 15) ? t : ((t < 30) ? t - 15 : 0);
#pragma unroll 1
    for (int k = 0; k < 15; ++k) {
      const bool cand = t >= k && t < 15;
      const int p = warp_argmax_first(cand ? tabs(Tm[15 * t + k]) : S(0), cand, t);  // first largest |entry| of column k, diagonal down
      if (p != k && t < 30) { const S tmp = Mx[15 * k + j]; Mx[15 * k + j] = Mx[15 * p + j]; Mx[15 * p + j] = tmp; }
      __syncwarp();
      {  // lanes 0..14: row t of den; lanes 16..30: row t - 16 of num.  Every load of the step in flight before the first store
         // (a rolled read-modify-write loop serialises on shared-memory latency: the stores may alias the loads)
        const int row = t & 15;
        if (row > k && row < 15) {
          const S l = Tm[15 * row + k] / Tm[15 * k + k];
          S* Mr = (t < 16) ? Tm : Phi;
          S pr[15], mr[15];
#pragma unroll
          for (int c = 0; c < 15; ++c) { pr[c] = Mr[15 * k + c]; mr[c] = Mr[15 * row + c]; }
          __syncwarp(__activemask());
#pragma unroll
          for (int c = 0; c < 15; ++c)
            if (t >= 16 || c > k) Mr[15 * row + c] = mr[c] - l * pr[c];
          if (t < 16) Tm[15 * row + k] = S(0);
        }
      }
      __syncwarp();
    }
    // back substitution: column t of Phi per lane, the solved entries in registers (static indices)
    if (t < 15) {
      S x[15];
#pragma unroll
      for (int i = 14; i >= 0; --i) {
        S sacc = Phi[15 * i + t];
#pragma unroll
        for (int k = i + 1; k < 15; ++k) sacc -= Tm[15 * i + k] * x[k];
        x[i] = sacc / Tm[15 * i + i];
      }
#pragma unroll
      for (int i = 0; i < 15; ++i) Phi[15 * i + t] = x[i];
    }
  }
  __syncthreads();
  stamp();  // LU + back substitution
  for (int sgn = 0; sgn < sq; ++sgn) {
    mm15(Tm, Phi, Phi);
    if (t < 225) Phi[t] = Tm[t];
    __syncthreads();
  }
  // ---- observability constraints (msckf.h:116-132)
  if (t == 0) {
    S Rn[9], Rp[9];
    quat_to_rot(st->q_IG_null, Rn);
    quat_to_rot(prop_q, Rp);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Phi[15 * i + j] = Rp[3 * i] * Rn[3 * j] + Rp[3 * i + 1] * Rn[3 * j + 1] + Rp[3 * i + 2] * Rn[3 * j + 2];
    S u[3];
    for (int i = 0; i < 3; ++i) u[i] = Rn[3 * i] * st->g[0] + Rn[3 * i + 1] * st->g[1] + Rn[3 * i + 2] * st->g[2];
    const S uu = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
    const S s[3] = {(S(1) / uu) * u[0], (S(1) / uu) * u[1], (S(1) / uu) * u[2]};
    for (int blk = 0; blk < 2; ++blk) {
      const int r0 = blk == 0 ? 6 : 12;
      S tmp[3];
      for (int i = 0; i < 3; ++i)
        tmp[i] = blk == 0 ? (st->v_I_G_null[i] - prop_v[i]) : (dT * st->v_I_G_null[i] + st->p_I_G_null[i] - prop_p[i]);
      const S* g = st->g;
      const S w[3] = {-tmp[2] * g[1] + tmp[1] * g[2], tmp[2] * g[0] - tmp[0] * g[2], -tmp[1] * g[0] + tmp[0] * g[1]};
      S Ab[9];
      for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Ab[3 * i + j] = Phi[15 * (r0 + i) + j];
      for (int i = 0; i < 3; ++i) {
        const S d = Ab[3 * i] * u[0] + Ab[3 * i + 1] * u[1] + Ab[3 * i + 2] * u[2] - w[i];
        for (int j = 0; j < 3; ++j) Phi[15 * (r0 + i) + j] = Ab[3 * i + j] - d * s[j];
      }
    }
  }
  __syncthreads();
  stamp();  // observability constraints
  // ---- covariance: P_II <- sym(Phi (P_II + G Q G^T dT) Phi^T), P_IC <- Phi P_IC (msckf.h:134-144)
  if (t < 180) {  // GQ = G * Q_imu
    const int i = t / 12, j = t % 12;
    S s = 0;
    for (int k = 0; k < 12; ++k) s += G[12 * i + k] * st->Q_imu[12 * k + j];
    GQ[t] = s;
  }
  __syncthreads();
  if (t < 225) {
    const int i = t / 15, j = t % 15;
    S s = 0;
    for (int k = 0; k < 12; ++k) s += GQ[12 * i + k] * G[12 * j + k];
    A2[t] = PII[t] + s * dT;
  }
  __syncthreads();
  mm15(A4, Phi, A2);
  mm15_nt(A6, A4, Phi);
  if (t < 225) {
    const int i = t / 15, j = t % 15;
    PII[t] = (A6[15 * i + j] + A6[15 * j + i]) / S(2.0);
  }
  if (cols_in_regs) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (t + 256 * u < c_all) {
        S nv[15];
#pragma unroll
        for (int i = 0; i < 15; ++i) {
          S sacc = 0;
#pragma unroll
          for (int k = 0; k < 15; ++k) sacc += Phi[15 * i + k] * vcol[u][k];
          nv[i] = sacc;
        }
#pragma unroll
        for (int i = 0; i < 15; ++i) vcol[u][i] = nv[i];
      }
    }
  } else {
    for (int col = t; col < c_all; col += 256) {
      S v[15];
#pragma unroll
      for (int k = 0; k < 15; ++k) v[k] = P[(size_t)k * ldp + 15 + col];
#pragma unroll
      for (int i = 0; i < 15; ++i) {
        S sacc = 0;
#pragma unroll
        for (int k = 0; k < 15; ++k) sacc += Phi[15 * i + k] * v[k];
        P[(size_t)i * ldp + 15 + col] = sacc;
        P[(size_t)(15 + col) * ldp + i] = sacc;
      }
    }
  }
  __syncthreads();
  if (t == 0) {
    for (int i = 0; i < 4; ++i) { st->q_IG[i] = prop_q[i]; st->q_IG_null[i] = prop_q[i]; }
    for (int i = 0; i < 3; ++i) {
      st->v_I_G[i] = prop_v[i]; st->v_I_G_null[i] = prop_v[i];
      st->p_I_G[i] = prop_p[i]; st->p_I_G_null[i] = prop_p[i];
    }
  }
  __syncthreads();  // the next reading starts from the state and covariance written above
  stamp();  // covariance
  }
  // ---- write back: IMU state, P_II, P_IC (and its transpose)
  if (t == 0) {
    for (int i = 0; i < 4; ++i) { gst->q_IG[i] = st->q_IG[i]; gst->q_IG_null[i] = st->q_IG_null[i]; }
    for (int i = 0; i < 3; ++i) {
      gst->v_I_G[i] = st->v_I_G[i]; gst->v_I_G_null[i] = st->v_I_G_null[i];
      gst->p_I_G[i] = st->p_I_G[i]; gst->p_I_G_null[i] = st->p_I_G_null[i];
    }
  }
  if (t < 225) P[(size_t)(t / 15) * ldp + t % 15] = PII[t];
  if (cols_in_regs) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int col = t + 256 * u;
      if (col < c_all) {
#pragma unroll
        for (int i = 0; i < 15; ++i) {
          P[(size_t)i * ldp + 15 + col] = vcol[u][i];
          P[(size_t)(15 + col) * ldp + i] = vcol[u][i];
        }
      }
    }
  }
}

// augmentState (msckf.h:148-212): clone the IMU pose through the extrinsics and append 6 rows/columns to P.
template <class S>
struct AugArgs {
  DevState<S>* st;
  S* P;
  S* poses;
  int ldp, M;
};
template <class S, int NM>
__global__ void __launch_bounds__(256) k_augment(const Members<AugArgs<S>, NM> a) {
  const int f = NM == 1 ? 0 : blockIdx.x;
  DevState<S>* const st = a.m[f].st;
  S* __restrict__ const P = a.m[f].P;
  S* __restrict__ const poses = a.m[f].poses;
  const int ldp = a.m[f].ldp, M = a.m[f].M;
  __shared__ S J[6][6];  // the 6 nonzero columns of J: state columns {0,1,2,12,13,14}
  __shared__ S JP6[6][6];
  const int t = threadIdx.x;
  const int n = 15 + 6 * M;
  if (t == 0) {
    S q[4];
    quat_mul(st->q_CI, st->q_IG, q);
    quat_normalize(q);
    S lever[3];
    quat_inv_rotate(st->q_IG, st->p_C_I, lever);
    S* ps = poses + kPoseStride * M;
    ps[0] = q[0]; ps[1] = q[1]; ps[2] = q[2]; ps[3] = q[3];
    ps[4] = st->p_I_G[0] + lever[0]; ps[5] = st->p_I_G[1] + lever[1]; ps[6] = st->p_I_G[2] + lever[2];
    ps[7] = S(0);
    S R[9];
    quat_to_rot(st->q_CI, R);
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) J[i][j] = S(0);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) J[i][j] = R[3 * i + j];
    J[3][0] = S(0); J[3][1] = -lever[2]; J[3][2] = lever[1];
    J[4][0] = lever[2]; J[4][1] = S(0); J[4][2] = -lever[0];
    J[5][0] = -lever[1]; J[5][1] = lever[0]; J[5][2] = S(0);
    J[3][3] = S(1); J[4][4] = S(1); J[5][5] = S(1);
  }
  __syncthreads();
  const int kc[6] = {0, 1, 2, 12, 13, 14};
  for (int b = t; b < n; b += 256) {
    S pk_[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) pk_[k] = P[(size_t)kc[k] * ldp + b];
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      S s = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k) s += J[a][k] * pk_[k];
      P[(size_t)(n + a) * ldp + b] = s;
      P[(size_t)b * ldp + n + a] = s;
      for (int k = 0; k < 6; ++k)
        if (b == kc[k]) JP6[a][k] = s;
    }
  }
  __syncthreads();
  if (t < 36) {
    const int a = t / 6, a2 = t % 6;
    S c1 = 0, c2 = 0;
    for (int k = 0; k < 6; ++k) { c1 += JP6[a][k] * J[a2][k]; c2 += JP6[a2][k] * J[a][k]; }
    P[(size_t)(n + a) * ldp + n + a2] = (c1 + c2) / S(2.0);
  }
}

// P_new = P_old(map, map) with map = [0..14, kept clone blocks]; poses gathered likewise.  The keep list travels as a
// kernel argument: prune() needs no staging copy and no synchronisation.
constexpr int kMaxKeep = 192;
struct KeepList { int n; int idx[kMaxKeep]; };
template <class S>
struct GatherArgs {
  const S* Pold;
  S* Pnew;
  const S* poses_old;
  S* poses_new;
  int n_new, ldp;
  KeepList kl;
};
static_assert(sizeof(Members<GatherArgs<double>, kBatchMembers>) <= 32764, "k_gather's batched arguments exceed the parameter limit");
template <class S, int NM>
__global__ void __launch_bounds__(256) k_gather(const Members<GatherArgs<S>, NM> g) {
  const int f = NM == 1 ? 0 : blockIdx.y;
  const int* keep_clones = g.m[f].kl.idx;
  const int n_keep = g.m[f].kl.n, n_new = g.m[f].n_new, ldp = g.m[f].ldp;
  const S* __restrict__ const Pold = g.m[f].Pold;
  S* __restrict__ const Pnew = g.m[f].Pnew;
  const S* __restrict__ const poses_old = g.m[f].poses_old;
  S* __restrict__ const poses_new = g.m[f].poses_new;
  const size_t total = (size_t)n_new * n_new;
  for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
    const int a = (int)(e / n_new), b = (int)(e % n_new);
    const int sa = a < 15 ? a : 15 + 6 * keep_clones[(a - 15) / 6] + (a - 15) % 6;
    const int sb = b < 15 ? b : 15 + 6 * keep_clones[(b - 15) / 6] + (b - 15) % 6;
    Pnew[(size_t)a * ldp + b] = Pold[(size_t)sa * ldp + sb];
  }
  if (blockIdx.x == 0)
    for (int e = threadIdx.x; e < n_keep * kPoseStride; e += 256)
      poses_new[e] = poses_old[kPoseStride * keep_clones[e / kPoseStride] + e % kPoseStride];
}

}  // namespace mb
