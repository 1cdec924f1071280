"""A dense numpy fp64 reference of the engine's state calls (propagate, augment, prune) on a fetched engine state, the
descriptor of an IMU reading as k_propagate sees it (which Pade branch, how far from a threshold, whether the LU pivots), and
the inputs that tests/test_state_kernels_gpu.py drives the kernels with.

State layout (msckf_b200_get_state): imu [29] p, v, b_g, b_a, g, q_IG, p_null, v_null, q_null; clone poses [M, 7] p_C_G, q_CG.
A reading is (omega [3], a [3], dT).

The reference is not the kernels' block form written again:
  * propagate builds F and G like msckf_numpy, steps the state with msckf_numpy's own Runge-Kutta scheme (msckf.h:1425-1467: at
    dT of a second its truncation error is far above rounding, so the exact rotation would not do), takes Phi = expm(F dT) from
    scipy (an algorithm other than Eigen's Pade), applies the observability changes of msckf.h:116-132 against the null state,
    and forms P+ = Phi_full (P + Q_full) Phi_full^T with Phi_full = blkdiag(Phi, I_6M), Q_full = blkdiag(G Q G^T dT, 0),
    symmetrising the IMU block only (as the filter does);
  * augment is P+ = T P T^T with the dense (n + 6) x n matrix T = [I; J] of msckf_numpy.augmentState;
  * prune is numpy indexing of P and the poses by the kept clone blocks."""
from math import factorial

import numpy as np
import scipy.linalg as sla

from msckf_mono_b200 import synth
from oracle.msckf_numpy import MSCKF as NumpyMSCKF, quat_mul, quat_normalized, quat_to_rot, skew

# Eigen's degree selection (matrix_exp_computeUV<float / double>): degree d while ||A||_1 < the threshold, else the top degree
# after `squarings` halvings, where frexp(||A||_1 / maxnorm) gives the count
PADE = {"float32": ([(3, 4.258730016922831e-001), (5, 1.880152677804762e+000)], 7, 3.925724783138660),
        "float64": ([(3, 1.495585217958292e-002), (5, 2.539398330063230e-001), (7, 9.504178996162932e-001),
                     (9, 2.097847961257068e+000)], 13, 5.371920351148152)}


# ----------------------------------------------------------------------------------------------------------- reference
def _view(imu):
    """a msckf_numpy filter object holding just the IMU state its Runge-Kutta step reads, in fp64"""
    f = NumpyMSCKF(np.float64)
    f.imu = {"q_IG": imu[15:19].copy(), "v_I_G": imu[3:6].copy(), "p_I_G": imu[0:3].copy(), "b_g": imu[6:9].copy(),
             "b_a": imu[9:12].copy(), "g": imu[12:15].copy()}
    return f


def F_and_G(imu, omega, a):
    """calcF / calcG (msckf.h:874-903) at the state imu and the reading (omega, a), fp64"""
    C = quat_to_rot(imu[15:19])
    F = np.zeros((15, 15))
    F[0:3, 0:3] = -skew(omega - imu[6:9])
    F[0:3, 3:6] = -np.eye(3)
    F[6:9, 0:3] = -C.T @ skew(a - imu[9:12])
    F[6:9, 9:12] = -C.T
    F[12:15, 6:9] = np.eye(3)
    G = np.zeros((15, 12))
    G[0:3, 0:3] = -np.eye(3)
    G[3:6, 3:6] = np.eye(3)
    G[6:9, 6:9] = -C.T
    G[9:12, 9:12] = np.eye(3)
    return F, G


def propagate(P, imu, reading, Q):
    """(P+, imu+) after one IMU reading, fp64.  The clone poses do not change."""
    P, imu, Q = (np.asarray(x, np.float64) for x in (P, imu, Q))
    omega, a, dT = np.asarray(reading[0:3], np.float64), np.asarray(reading[3:6], np.float64), float(reading[6])
    F, G = F_and_G(imu, omega, a)
    prop = _view(imu)._propagate_imu_state_rk(omega, a, np.float64(dT))
    Phi = sla.expm(F * dT)
    # observability constraints (msckf.h:116-132), against the null state
    Rn = quat_to_rot(imu[25:29])
    g = imu[12:15]
    Phi[0:3, 0:3] = quat_to_rot(prop["q_IG"]) @ Rn.T
    u = Rn @ g
    s = u / (u @ u)
    for rows, tmp in ((slice(6, 9), imu[22:25] - prop["v_I_G"]),
                      (slice(12, 15), dT * imu[22:25] + imu[19:22] - prop["p_I_G"])):
        A = Phi[rows, 0:3].copy()
        Phi[rows, 0:3] = A - np.outer(A @ u - skew(tmp) @ g, s)
    n = P.shape[0]
    Phi_full = np.eye(n)
    Phi_full[:15, :15] = Phi
    Q_full = np.zeros((n, n))
    Q_full[:15, :15] = G @ Q @ G.T * dT
    Pn = Phi_full @ (P + Q_full) @ Phi_full.T
    Pn[:15, :15] = (Pn[:15, :15] + Pn[:15, :15].T) / 2
    out = imu.copy()
    out[0:3], out[3:6], out[15:19] = prop["p_I_G"], prop["v_I_G"], prop["q_IG"]
    out[19:22], out[22:25], out[25:29] = prop["p_I_G"], prop["v_I_G"], prop["q_IG"]
    return Pn, out


def propagate_n(P, imu, readings, Q):
    """k readings as k single steps in sequence"""
    for r in readings:
        P, imu = propagate(P, imu, r, Q)
    return P, imu


def augment(P, imu, poses, q_CI, p_C_I):
    """(P+, poses+) after appending the camera clone of the IMU pose, fp64 (msckf_numpy.augmentState, not symmetrised)"""
    P, imu, q_CI, p_C_I = (np.asarray(x, np.float64) for x in (P, imu, q_CI, p_C_I))
    n = P.shape[0]
    C = quat_to_rot(imu[15:19])
    lever = C.T @ p_C_I
    T = np.zeros((n + 6, n))
    T[:n, :n] = np.eye(n)
    T[n:n + 3, 0:3] = quat_to_rot(q_CI)
    T[n + 3:, 0:3] = skew(lever)
    T[n + 3:, 12:15] = np.eye(3)
    pose = np.concatenate([imu[0:3] + lever, quat_normalized(quat_mul(q_CI, imu[15:19]))])
    return T @ P @ T.T, np.vstack([np.asarray(poses, np.float64).reshape(-1, 7), pose])


def prune_map(keep):
    """the rows / columns of P that a prune keeping clones `keep` keeps"""
    return np.concatenate([np.arange(15)] + [np.arange(15 + 6 * k, 21 + 6 * k) for k in keep]).astype(int)


def prune(P, poses, keep):
    m = prune_map(keep)
    return P[np.ix_(m, m)], np.asarray(poses).reshape(-1, 7)[np.asarray(keep, dtype=int)]


# ---------------------------------------------------------------------------------------------------------- descriptor
def pick(l1, dtype):
    """(degree, squarings) that ExpmPick<dtype> takes at ||F dT||_1 = l1"""
    lower, top, maxnorm = PADE[np.dtype(dtype).name]
    for d, thr in lower:
        if l1 < thr:
            return d, 0
    return top, max(int(np.frexp(l1 / maxnorm)[1]), 0)


def thresholds(dtype, upto=1e4):
    """every ||A||_1 at which the degree or the squaring count changes"""
    lower, _, maxnorm = PADE[np.dtype(dtype).name]
    t = [thr for _, thr in lower]
    k = 0
    while maxnorm * 2.0 ** k < upto:
        t.append(maxnorm * 2.0 ** k)
        k += 1
    return np.array(t)


def pade_uv(A, deg):
    """U (odd terms) and V (even terms) of the [deg / deg] Pade approximant of exp(A), from the closed form of its
    coefficients c_k = (2d - k)! d! / ((2d)! k! (d - k)!) (Eigen's b are these times a constant, which changes no pivot)"""
    c = [factorial(2 * deg - k) * factorial(deg) / (factorial(2 * deg) * factorial(k) * factorial(deg - k)) for k in range(deg + 1)]
    pw = [np.eye(A.shape[0])]
    for _ in range(deg):
        pw.append(pw[-1] @ A)
    U = sum(c[k] * pw[k] for k in range(1, deg + 1, 2))
    V = sum(c[k] * pw[k] for k in range(0, deg + 1, 2))
    return U, V


def pivot_gap(A):
    """largest |chosen pivot| / |diagonal candidate| over the steps of a partial-pivot LU of A (1: no row is exchanged); a gap
    well above 1 exchanges the row whatever the rounding of A"""
    A = np.array(A, dtype=np.float64)
    gap = 1.0
    for k in range(A.shape[0]):
        p = k + int(np.argmax(np.abs(A[k:, k])))
        if p != k:
            gap = max(gap, abs(A[p, k]) / abs(A[k, k]))
            A[[k, p]] = A[[p, k]]
        A[k + 1:] -= np.outer(A[k + 1:, k] / A[k, k], A[k])
    return gap


def describe(imu, reading, dtype):
    """the reading as k_propagate of a `dtype` engine sees it at the (fetched) state imu: dict l1 = ||F dT||_1 (F and F dT
    formed in dtype, column sums in double rounded back to dtype), deg, sq (ExpmPick), margin (smallest |l1 / threshold - 1|),
    swap (whether scipy's partial-pivot LU of V - U, at that degree and scaling, exchanges a row) and gap (pivot_gap of V - U)"""
    S = np.dtype(dtype).type
    st = np.asarray(imu).astype(dtype)
    r = np.asarray(reading).astype(dtype)
    C = quat_to_rot(st[15:19])
    F = np.zeros((15, 15), dtype=dtype)
    F[0:3, 0:3] = -skew(r[0:3] - st[6:9])
    F[0:3, 3:6] = -np.eye(3, dtype=dtype)
    F[6:9, 0:3] = -C.T @ skew(r[3:6] - st[9:12])
    F[6:9, 9:12] = -C.T
    F[12:15, 6:9] = np.eye(3, dtype=dtype)
    Fd = (F * r[6]).astype(dtype)
    l1 = float(max(S(np.abs(Fd.astype(np.float64)).sum(axis=0)[j]) for j in range(15)))
    deg, sq = pick(l1, dtype)
    A = Fd.astype(np.float64) * 2.0 ** -sq
    U, V = pade_uv(A, deg)
    piv = sla.lu_factor(V - U)[1]
    return {"l1": l1, "deg": deg, "sq": sq, "margin": float(np.min(np.abs(l1 / thresholds(dtype) - 1))),
            "swap": bool(np.any(piv != np.arange(15))), "gap": pivot_gap(V - U)}


# -------------------------------------------------------------------------------------------------------------- inputs
CAMERA = synth.euroc_camera()  # the EuRoC extrinsics: a lever arm of 6.5 cm
# a dense SPD Q_imu at the EuRoC scales (gyro / gyro-bias / accelerometer / accelerometer-bias variances): a random correlation
# matrix between them, so that every entry of Q_imu and every stride into it counts
_QD = np.sqrt(np.array([1e-4] * 3 + [3.6733e-5] * 3 + [1e-2] * 3 + [7e-2] * 3))
_B = np.random.default_rng(11).normal(size=(12, 12))
_CORR = _B @ _B.T + 2 * np.eye(12)
_CORR /= np.sqrt(np.outer(np.diag(_CORR), np.diag(_CORR)))
Q_IMU = _QD[:, None] * _CORR * _QD[None, :]
# a non-identity attitude, nonzero biases and velocity
IMU0 = {"p_I_G": np.array([1.2, -0.7, 0.4]), "v_I_G": np.array([0.6, -0.4, 0.15]), "b_g": np.array([0.05, -0.04, 0.03]),
        "b_a": np.array([0.3, -0.25, 0.2]), "g": np.array([0.0, 0.0, -9.81]),
        "q_IG": quat_normalized(np.array([0.3, -0.2, 0.5, 0.8]))}


def setup():
    """(camera, noise, params, imu_state) of the engines under test"""
    noise = dict(synth.euroc_noise(), Q_imu=Q_IMU)
    return CAMERA, noise, synth.euroc_params(max_cam_states=192), IMU0


def imu_vector(s=IMU0):
    """the state dict as the engine's imu [29] (null state = state), fp64"""
    v = [s[k] for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG")]
    return np.concatenate(v + [s["p_I_G"], s["v_I_G"], s["q_IG"]]).astype(np.float64)


def reading(rng, dT):
    """one reading of dT: a rotation rate of ~0.3 rad/s and a specific force near 1 g, both off the axes"""
    w = np.array([0.25, -0.15, 0.3]) + 0.05 * rng.normal(size=3)
    a = np.array([0.8, -0.6, 9.6]) + 0.3 * rng.normal(size=3)
    return np.concatenate([w, a, [dT]])


def readings(rng, k, dT=0.005):
    return np.array([reading(rng, dT) for _ in range(k)]).reshape(-1, 7)


# Pade branches the tests cover, by the ||F dT||_1 they aim at (the middle of each branch's band): (degree, squarings, l1)
BRANCHES = {"float64": [(3, 0, 0.0075), (5, 0, 0.06), (7, 0, 0.5), (9, 0, 1.4), (13, 0, 3.5), (13, 1, 8.0), (13, 3, 30.0)],
            "float32": [(3, 0, 0.2), (5, 0, 0.9), (7, 0, 2.8), (7, 2, 11.0)]}
# readings whose LU of V - U exchanges rows at IMU0, the chosen pivot 1.6 and 2.1 times the diagonal candidate (found with
# `describe`): the pivoting depends on the direction of the specific force against the attitude, and takes a long dT
SWAP_READINGS = {"float64": (13, 3, np.array([0.187, -0.02, 0.014, 2.066, 9.172, 9.338, 2.574])),
                 "float32": (7, 2, np.array([0.194, 0.04, 0.024, 1.609, 3.699, 4.078, 2.332]))}


def branch_readings(dtype, imu=None):
    """[(degree, squarings, reading)] of `dtype`: one reading per branch of BRANCHES, its dT scaled so that ||F dT||_1 hits
    the branch's target at the state imu (||F dT||_1 is linear in dT), then the dtype's reading whose LU swaps a row"""
    imu = imu_vector() if imu is None else imu
    name = np.dtype(dtype).name
    out = []
    rng = np.random.default_rng(3)
    for deg, sq, target in BRANCHES[name]:
        r = reading(rng, 1.0)
        r[6] = target / describe(imu, r, np.float64)["l1"]
        out.append((deg, sq, r))
    return out + [SWAP_READINGS[name]]
