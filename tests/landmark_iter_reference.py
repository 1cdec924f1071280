"""Dense fp64 reference of the iterated mapped-landmark update (an iterated EKF, msckf_b200_landmark_update with max_iter >= 2).

With the prior x^ (IMU state and clone poses) and P, delta_0 = 0 and the iterate x_i = x^ [+] delta_i on the clone poses (the
engine's injection: q <- normalise(buildUpdateQuat(dtheta) * q), p <- p + dp), linearisation i builds the uncompressed stacked
system (H_i, r_i) of the observations used at linearisation 0 (tests/test_landmark_gpu.py's model), and
delta_{i+1} = K_i (r_i + H_i delta_i) with K_i = P H_i^T (H_i P H_i^T + R)^-1, always against the prior P.  It stops when
max |delta_{i+1} - delta_i| <= tol, after max_iter linearisations, or when a used observation is behind the camera at the next
iterate (then the previous linearisation is applied).  The last linearisation is applied as one dense EKF update with the
residual r_i + H_i delta_i (test_aid_gpu.numpy_update: Joseph form and the injection of oracle/msckf_numpy.py).  Flags, gamma,
NIS and dof are linearisation 0's.  max_iter <= 1 is exactly the single dense update of tests/test_landmark_gpu.py."""
from types import SimpleNamespace

import numpy as np

from oracle.msckf_numpy import MSCKF as NumpyMSCKF, quat_mul, quat_normalized
from tests.test_aid_gpu import numpy_update
from tests.test_landmark_gpu import dense, jacobian, project


def build_update_quat(d):
    return NumpyMSCKF._build_update_quat(SimpleNamespace(S=np.float64, dt=np.float64), np.asarray(d, dtype=np.float64))


def boxplus(poses, delta):
    """clone poses [M, 7] (p_C_G, q_CG xyzw) moved by the clone part of delta (n = 15 + 6 M), the engine's injection in fp64"""
    out = np.array(poses, dtype=np.float64, copy=True)
    for k in range(len(out)):
        out[k, 3:7] = quat_normalized(quat_mul(build_update_quat(delta[15 + 6 * k:18 + 6 * k]), out[k, 3:7]))
        out[k, 0:3] = out[k, 0:3] + delta[18 + 6 * k:21 + 6 * k]
    return out


def boxminus(a, b):
    """the clone error e with a = b [+] e (rotation: buildUpdateQuat inverted exactly, |dtheta| < 2)"""
    e = np.zeros(6 * len(a))
    for k in range(len(a)):
        qb = b[k, 3:7]
        qe = quat_mul(a[k, 3:7], np.array([-qb[0], -qb[1], -qb[2], qb[3]]) / (qb @ qb))
        qe = qe * np.sign(qe[3]) / np.linalg.norm(qe)
        e[6 * k:6 * k + 3] = -2.0 * qe[0:3]
        e[6 * k + 3:6 * k + 6] = a[k, 0:3] - b[k, 0:3]
    return e


def linearise(n, poses, clone, z, p_L, used):
    """(H, r) of the used observations at clone poses `poses`, or None when one of them is behind the camera / not finite"""
    H, r = [], []
    for k, zi, pl in zip(np.asarray(clone)[used], np.asarray(z)[used], np.asarray(p_L)[used]):
        pc, zh = project(poses[k], pl)
        if not (pc[0, 2] > 0 and np.all(np.isfinite(zh))):
            return None
        row = np.zeros((2, n))
        row[:, 15 + 6 * k:21 + 6 * k] = jacobian(poses[k], pl)
        H.append(row)
        r.append(zi - zh[0])
    return np.vstack(H), np.concatenate(r)


def iekf(P, imu, poses, clone, z, p_L, R, chi2=0.0, max_iter=1, tol=1e-10):
    """the iterated update on (P, imu, poses): a dict with the updated P, imu, poses, the result fields of
    msckf_b200_landmark_result (nis, dof, used, applied, iterations, converged, step), gamma, flag, and the last linearisation
    (H, r, delta_lin: the delta it was taken at) with the applied delta dx"""
    P = np.asarray(P, dtype=np.float64)
    n = P.shape[0]
    H, r, Rb, gam, flag = dense(P, poses, clone, z, p_L, R, chi2)
    used = flag == 0
    out = {"gamma": gam, "flag": flag, "used": int(used.sum()), "dof": len(r), "iterations": 0, "converged": 0, "step": 0.0}
    if not used.any():
        return dict(out, P=P.copy(), imu=np.array(imu, float), poses=np.array(poses, float), nis=0.0, applied=0)
    out["nis"] = float(r @ np.linalg.solve(H @ P @ H.T + Rb, r))
    delta = np.zeros(n)
    it = 1
    while True:
        K = np.linalg.solve(H @ P @ H.T + Rb, H @ P).T
        new = K @ (r + H @ delta)
        if it >= max_iter:
            break
        out["step"] = float(np.abs(new - delta).max())
        if out["step"] <= tol:
            out["converged"] = 1
            break
        nxt = linearise(n, boxplus(poses, new), clone, z, p_L, used)
        if nxt is None:  # a used observation fails at the next iterate: the current linearisation is applied
            break
        delta = new
        H, r = nxt
        it += 1
    Pn, imun, posesn, _, _ = numpy_update(P, np.array(imu, float), np.array(poses, float), H, r + H @ delta, Rb)
    return dict(out, P=Pn, imu=imun, poses=posesn, applied=1, iterations=it, H=H, r=r, delta_lin=delta, dx=new, Rb=Rb)


def stationarity(P, H, r, Rb, dx):
    """|P^-1 dx - H^T R^-1 r| relative to |H^T R^-1 r|: zero at a fixed point of the iteration (Gauss-Newton)"""
    g = H.T @ np.linalg.solve(Rb, r)
    return float(np.abs(np.linalg.solve(P, dx) - g).max() / np.abs(g).max())


def relocalisation_trial(rng, M, per, drift_pos, drift_yaw, sigma, max_iter, P=None):
    """one draw of the relocalisation toy: M clones whose error shares a drift (position drift_pos, yaw drift_yaw, roll and
    pitch drift_yaw / 5) plus a small per-clone part, drawn from P; `per` landmarks per clone at 3-15 m depth, pixel noise
    sigma.  Returns (NEES of the updated clone poses over 6 M dof, mean squared clone position error)."""
    n = 15 + 6 * M
    if P is None:
        P = relocalisation_prior(M, drift_pos, drift_yaw)
    est = np.zeros((M, 7))
    for k in range(M):
        est[k, 3:7] = quat_normalized(np.concatenate([rng.normal(size=3) * 0.15, [1.0]]))
        est[k, 0:3] = [0.3 * k, 0.0, 0.0]
    e = np.linalg.cholesky(P) @ rng.normal(size=n)
    truth = boxplus(est, e)
    clone, z, p_L = [], [], []
    for k in range(M):
        for _ in range(per):
            d = rng.uniform(3, 15)
            pc = np.array([rng.uniform(-0.4, 0.4) * d, rng.uniform(-0.3, 0.3) * d, d])
            pl = np.linalg.inv(_rot(truth[k])) @ pc + truth[k, 0:3]
            clone.append(k); z.append(pc[:2] / d + sigma * rng.normal(size=2)); p_L.append(pl)
    R = sigma ** 2 * np.eye(2)
    out = iekf(P, np.zeros(29), est, np.array(clone), np.array(z), np.array(p_L), R, max_iter=max_iter, tol=1e-10)
    er = boxminus(truth, out["poses"])
    Pc = out["P"][15:, 15:]
    return float(er @ np.linalg.solve(Pc, er)), float(np.sum(er.reshape(M, 6)[:, 3:] ** 2) / M)


def relocalisation_prior(M, drift_pos, drift_yaw):
    n = 15 + 6 * M
    Jc = np.vstack([np.eye(6)] * M)
    Sc = np.diag([(drift_yaw / 5) ** 2, (drift_yaw / 5) ** 2, drift_yaw ** 2, drift_pos ** 2, drift_pos ** 2, drift_pos ** 2])
    P = np.eye(n) * 1e-4
    P[15:, 15:] = Jc @ Sc @ Jc.T + np.diag(np.tile([1e-6] * 3 + [1e-4] * 3, M))
    return P


def _rot(pose):
    from oracle.msckf_numpy import quat_to_rot
    return quat_to_rot(pose[3:7])
