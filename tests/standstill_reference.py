"""numpy fp64 reference of the standstill update (msckf_b200_standstill_update, DESIGN.md 4.18).

A window of k IMU readings (omega_j, a_j, dT_j) taken at rest has, for every j, r_j = [omega_j - b_g; a_j - (b_a - C(q_IG) g)]
= H dx + n_j with one H for every reading and n_j ~ N(0, s^2 R0 / dT_j), R0 the gyro (0..2) and accelerometer (6..8) blocks of
Q_imu.  `dense_update` fuses all 6k reading rows and a zero-velocity row block as one EKF update; `stats` forms what the host
forms from the readings (the dT-weighted means, T, R = s^2 R0 / T and the scatter, in the host's arithmetic order, so that z
and R are the engine's bit for bit); `mean_update` fuses the 9 rows VELOCITY, GYRO_AT_REST, ACCEL_AT_REST.  The scatter rows
have H = 0, so the two updates agree and NIS_dense = scatter sigma + NIS_mean."""
from types import SimpleNamespace

import numpy as np

from oracle.msckf_numpy import MSCKF as NumpyMSCKF, quat_mul, quat_normalized, quat_to_rot

GYRO_AT_REST, ACCEL_AT_REST, VELOCITY = 15, 16, 0


def skew(u):
    return np.array([[0.0, -u[2], u[1]], [u[2], 0.0, -u[0]], [-u[1], u[0], 0.0]])


def r0_blocks(Q):
    """(R0_g, R0_a): the gyro and accelerometer blocks of the 12 x 12 Q_imu"""
    Q = np.asarray(Q, dtype=np.float64).reshape(12, 12)
    return Q[0:3, 0:3].copy(), Q[6:9, 6:9].copy()


def stats(readings, Q, noise_scale=1.0, sigma_v=0.01, weights="dT"):
    """The host's statistics of a window: T, the dT-weighted means w, a (z of the at-rest items), Rg = s^2 R0_g / T,
    Ra = s^2 R0_a / T, Rv = sigma_v^2 I, sigma (the scatter's chi-square, 6 (k - 1) dof) and scatter = sigma / (6 (k - 1)).
    Sums run in reading order in fp64 like the engine's, so w, a, Rg and Ra are its bits.  weights="count": the unweighted
    mean (what the engine must NOT do; the mutation tests use it)."""
    r = np.asarray(readings, dtype=np.float64).reshape(-1, 7)
    k = len(r)
    T, sw, sa = 0.0, [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]
    for j in range(k):
        dT = float(r[j, 6]) if weights == "dT" else 1.0
        T += dT
        for i in range(3):
            sw[i] += dT * float(r[j, i])
            sa[i] += dT * float(r[j, 3 + i])
    w = np.array([x / T for x in sw])
    a = np.array([x / T for x in sa])
    if weights != "dT":
        T = float(sum(float(x) for x in r[:, 6]))
    Rg0, Ra0 = r0_blocks(Q)
    s2 = noise_scale * noise_scale
    Rg, Ra = s2 * Rg0 / T, s2 * Ra0 / T
    ybar = np.r_[w, a]
    R0i = np.linalg.inv(np.block([[Rg0, np.zeros((3, 3))], [np.zeros((3, 3)), Ra0]]))
    sig = sum(float(r[j, 6]) * (r[j, 0:6] - ybar) @ R0i @ (r[j, 0:6] - ybar) for j in range(k)) / s2
    return {"T": T, "w": w, "a": a, "Rg": Rg, "Ra": Ra, "Rv": sigma_v * sigma_v * np.eye(3), "sigma": sig,
            "scatter": sig / (6.0 * (k - 1)), "k": k}


def items(st):
    """the 9-row stack of a window's statistics, as item dicts (capi.aid_items)"""
    return [{"model": VELOCITY, "z": np.zeros(3), "R": st["Rv"]},
            {"model": GYRO_AT_REST, "z": st["w"], "R": st["Rg"]},
            {"model": ACCEL_AT_REST, "z": st["a"], "R": st["Ra"]}]


def predicted(imu):
    """h(x) = [b_g; b_a - C(q_IG) g] of an imu vector (p, v, b_g, b_a, g, q_IG, ...)"""
    imu = np.asarray(imu, dtype=np.float64)
    return np.r_[imu[6:9], imu[9:12] - quat_to_rot(imu[15:19]) @ imu[12:15]]


def rest_jacobian(imu, n, theta_sign=1.0):
    """H (6 x n) of the two at-rest models: GYRO rows over db_g; ACCEL rows -[C g]x over dtheta and I over db_a.
    theta_sign = -1 flips H_theta (a mutation the tests must catch)."""
    imu = np.asarray(imu, dtype=np.float64)
    u = quat_to_rot(imu[15:19]) @ imu[12:15]
    H = np.zeros((6, n))
    H[0:3, 3:6] = np.eye(3)
    H[3:6, 0:3] = -theta_sign * skew(u)
    H[3:6, 9:12] = np.eye(3)
    return H


def velocity_rows(n):
    H = np.zeros((3, n))
    H[:, 6:9] = np.eye(3)
    return H


def joseph(P, imu, poses, H, r, R):
    """Joseph form, the injection of oracle/msckf_numpy.py (msckf.h:1373-1391) and the NIS; all fp64"""
    S = H @ P @ H.T + R
    K = np.linalg.solve(S, H @ P).T
    dx = K @ r
    A = np.eye(P.shape[0]) - K @ H
    Pn = A @ P @ A.T + K @ R @ K.T
    buq = lambda d: NumpyMSCKF._build_update_quat(SimpleNamespace(S=np.float64, dt=np.float64), d)  # noqa: E731
    imu, poses = np.array(imu, dtype=np.float64), np.array(poses, dtype=np.float64).reshape(-1, 7)
    imu[15:19] = quat_mul(buq(dx[0:3]), imu[15:19])  # not renormalised
    imu[6:9] += dx[3:6]; imu[3:6] += dx[6:9]; imu[9:12] += dx[9:12]; imu[0:3] += dx[12:15]
    for k in range(len(poses)):
        poses[k, 3:7] = quat_normalized(quat_mul(buq(dx[15 + 6 * k:18 + 6 * k]), poses[k, 3:7]))
        poses[k, 0:3] += dx[18 + 6 * k:21 + 6 * k]
    return {"P": Pn, "imu": imu, "poses": poses, "nis": float(r @ np.linalg.solve(S, r)), "dx": dx,
            "dx_norm": float(np.linalg.norm(dx))}


def dense_system(readings, Q, imu, n, noise_scale=1.0, sigma_v=0.01):
    """(H, r, R) of the dense update: the zero-velocity rows, then the 6 rows of every reading"""
    r = np.asarray(readings, dtype=np.float64).reshape(-1, 7)
    Rg0, Ra0 = r0_blocks(Q)
    R0 = np.block([[Rg0, np.zeros((3, 3))], [np.zeros((3, 3)), Ra0]]) * noise_scale ** 2
    Hr, h = rest_jacobian(imu, n), predicted(imu)
    Hs, rs, Rs = [velocity_rows(n)], [-np.asarray(imu, dtype=np.float64)[3:6]], [sigma_v ** 2 * np.eye(3)]
    for j in range(len(r)):
        Hs.append(Hr); rs.append(r[j, 0:6] - h); Rs.append(R0 / r[j, 6])
    R = np.zeros((sum(x.shape[0] for x in Rs),) * 2)
    o = 0
    for x in Rs:
        R[o:o + len(x), o:o + len(x)] = x
        o += len(x)
    return np.vstack(Hs), np.concatenate(rs), R


def dense_update(P, imu, poses, readings, Q, noise_scale=1.0, sigma_v=0.01):
    H, r, R = dense_system(readings, Q, imu, P.shape[0], noise_scale, sigma_v)
    return joseph(P, imu, poses, H, r, R)


def mean_system(st, imu, n, theta_sign=1.0):
    """(H, r, R) of the 9-row stack of a window's statistics"""
    H = np.vstack([velocity_rows(n), rest_jacobian(imu, n, theta_sign)])
    r = np.r_[-np.asarray(imu, dtype=np.float64)[3:6], np.r_[st["w"], st["a"]] - predicted(imu)]
    R = np.zeros((9, 9))
    R[0:3, 0:3], R[3:6, 3:6], R[6:9, 6:9] = st["Rv"], st["Rg"], st["Ra"]
    return H, r, R


def mean_update(P, imu, poses, st, theta_sign=1.0):
    H, r, R = mean_system(st, imu, P.shape[0], theta_sign)
    return joseph(P, imu, poses, H, r, R)


def rest_readings(rng, imu, k, Q, noise_scale=1.0, dT=None, bias=None):
    """k readings taken at rest by a filter whose state is imu: omega = b_g + n, a = b_a - C g + n, n ~ N(0, s^2 R0 / dT)
    (plus an optional bias on the mean); dT non-uniform around 5 ms unless given"""
    Rg0, Ra0 = r0_blocks(Q)
    Lg, La = np.linalg.cholesky(Rg0), np.linalg.cholesky(Ra0)
    h = predicted(imu)
    dts = rng.uniform(0.003, 0.007, size=k) if dT is None else np.full(k, dT)
    out = np.zeros((k, 7))
    for j in range(k):
        out[j, 0:3] = h[0:3] + noise_scale * Lg @ rng.normal(size=3) / np.sqrt(dts[j])
        out[j, 3:6] = h[3:6] + noise_scale * La @ rng.normal(size=3) / np.sqrt(dts[j])
        out[j, 6] = dts[j]
    if bias is not None:
        out[:, 0:6] += bias
    return out
