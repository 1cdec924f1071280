"""Dense fp64 reference of the iterated stacked aided update (an iterated EKF, msckf_b200_aid_stack_update_iter /
_fde_iter, include/msckf_b200.h), on a fetched state, built on tests/aid_fde_reference.py's linearise and joseph and the
injection of montecarlo.perturb.

With the prior x^ (imu 19: p, v, b_g, b_a, g, q_IG; poses [M, 7]: p, q) and P, delta_0 = 0 and the iterate x_i = x^ [+] delta_i
(montecarlo.perturb, with clone quaternions renormalised as the engine's injection does), linearisation i stacks the items'
(H_i, r_i) at x_i and delta_{i+1} = K_i (r_i + H_i delta_i), K_i = P H_i^T (H_i P H_i^T + R)^-1, always against the prior P.
It stops when max |delta_{i+1} - delta_i| <= tol (NaN: infinite), after max_iter linearisations, or when an item is
degenerate at the next iterate (then the current linearisation is applied).  The last linearisation is applied as one
Joseph-form update with the residual r_i + H_i delta_i and the injection of oracle/msckf_numpy.py.  The NIS is linearisation
0's.  max_iter <= 1 is aid_fde_reference.joseph exactly."""
import numpy as np
from scipy.linalg import block_diag

from msckf_mono_b200 import montecarlo as mc
from tests.aid_fde_reference import joseph, linearise

HEADING_MIN_HORIZ = 1e-6  # the kernel's kAidHeadingMinHoriz, kAidRangeMin, kAidPlaneMinBeamZ
RANGE_MIN = 1e-6
PLANE_MIN_BEAM_Z = 1e-6


def boxplus(imu, poses, delta):
    """(imu, poses) of x^ [+] delta: montecarlo's injection, clone quaternions renormalised"""
    s = mc.perturb({"imu": np.asarray(imu, dtype=np.float64), "poses": np.asarray(poses, dtype=np.float64)}, delta)
    poses = s["poses"]
    poses[:, 3:7] /= np.linalg.norm(poses[:, 3:7], axis=1, keepdims=True)
    return s["imu"], poses


def degenerate(item, imu, poses):
    """the item cannot be linearised at the state (what ends a plain stack with status 2)"""
    m = item["model"]
    if m in (mc.AID_HEADING, mc.AID_CLONE_HEADING):
        q, _, _, _ = mc._gnss_frame(item, imu, poses)
        f = np.asarray(item["z"][1:4], dtype=np.float64)
        d = mc.quat_to_rot(q).T @ f
        return not (d[0] ** 2 + d[1] ** 2 > HEADING_MIN_HORIZ * (f @ f))
    if m in (mc.AID_RANGE, mc.AID_CLONE_RANGE):
        q, p, _ = mc._range_frame(item, imu, poses)
        z = np.asarray(item["z"], dtype=np.float64)
        return not (mc.range_of(p, q, z[4:7], z[1:4]) > RANGE_MIN)
    if m in (mc.AID_PLANE_RANGE, mc.AID_CLONE_PLANE_RANGE):
        q, p, _ = mc._range_frame(item, imu, poses)
        z = np.asarray(item["z"], dtype=np.float64)
        b = mc.quat_to_rot(q).T @ (z[5:8] / np.linalg.norm(z[5:8]))
        return not (b[2] ** 2 > PLANE_MIN_BEAM_Z) or not (mc.plane_range_of(p, q, z[1], z[2:5], z[5:8]) > 0.0)
    return False


def stacked(items, imu, poses, n):
    """(H, r) of the stack at the state, or None when an item is degenerate there"""
    if any(degenerate(it, imu, poses) for it in items):
        return None
    lin = linearise(items, imu, poses, n)
    return np.vstack([h for h, _ in lin]), np.concatenate([v for _, v in lin])


def iekf(items, imu, poses, P, max_iter=1, tol=0.0):
    """the iterated update of the (applied) stack on (P, imu, poses): a dict with the updated P, imu, poses, nis and dof of
    linearisation 0, iterations, converged, step (steps: every step taken), dx_norm, and the last linearisation (H, r, delta_lin: the delta it was
    taken at; dx: the applied delta)"""
    P = np.asarray(P, dtype=np.float64)
    imu, poses = np.asarray(imu, dtype=np.float64), np.asarray(poses, dtype=np.float64)
    n = P.shape[0]
    R = block_diag(*[it["R"] for it in items])
    H, r = stacked(items, imu, poses, n)
    nis = float(r @ np.linalg.solve(H @ P @ H.T + R, r))
    delta = np.zeros(n)
    it, step, converged, steps = 1, 0.0, 0, []
    while True:
        new = np.linalg.solve(H @ P @ H.T + R, H @ P).T @ (r + H @ delta)
        if it >= max_iter:
            break
        d = np.abs(new - delta)
        step = float(np.inf if np.isnan(d).any() else d.max())
        steps.append(step)
        if step <= tol:
            converged = 1
            break
        nxt = stacked(items, *boxplus(imu, poses, new), n)
        if nxt is None:
            break
        delta = new
        H, r = nxt
        it += 1
    from tests.test_aid_gpu import numpy_update
    Pn, imun, posesn, _, dx_norm = numpy_update(P, imu, poses, H, r + H @ delta, R)
    return {"P": Pn, "imu": imun, "poses": posesn, "nis": nis, "dof": len(r), "iterations": it, "converged": converged,
            "step": step, "steps": steps, "dx_norm": dx_norm, "H": H, "r": r, "R": R, "delta_lin": delta, "dx": new}


def one_linearisation(items, imu, poses, P):
    """joseph's (P, dx, nis): what max_iter 1 must give"""
    return joseph(items, np.asarray(imu, dtype=np.float64), np.asarray(poses, dtype=np.float64), np.asarray(P, dtype=np.float64))


def stationarity(P, H, r, R, dx):
    """|P^-1 dx - H^T R^-1 r| relative to |H^T R^-1 r| (H, r at the last iterate): zero at a fixed point (Gauss-Newton)"""
    g = H.T @ np.linalg.solve(R, r)
    return float(np.abs(np.linalg.solve(P, dx) - g).max() / np.abs(g).max())


def anchor_toy(rng, sigma_p, max_iter, draws=2000, sigma=0.1):
    """ANEES over 3 dof of the position after one range stack to montecarlo.ANCHORS (range sigma m) with a position-only
    prior P = sigma_p^2 I: truth near the origin, the estimate drawn as truth + N(0, P)"""
    total = 0.0
    for _ in range(draws):
        truth = rng.normal(size=3) * 0.5
        est = truth + sigma_p * rng.normal(size=3)
        imu = np.zeros(19)
        imu[0:3], imu[18] = est, 1.0
        items = [{"model": mc.AID_RANGE, "a": 0, "b": 0, "R": np.array([[sigma ** 2]]),
                  "z": np.r_[np.linalg.norm(truth - a) + sigma * rng.normal(), a, 0.0, 0.0, 0.0]} for a in mc.ANCHORS]
        P = np.eye(15) * 1e-6
        P[12:15, 12:15] = sigma_p ** 2 * np.eye(3)
        out = iekf(items, imu, np.zeros((0, 7)), P, max_iter=max_iter, tol=1e-12)
        e = truth - out["imu"][0:3]
        total += float(e @ np.linalg.solve(out["P"][12:15, 12:15], e))
    return total / draws


def drift_prior(rng, M, drift):
    """a dense SPD prior over 15 + 6M states whose position blocks have a standard deviation of about `drift` m and whose
    attitude blocks about drift / 5 rad"""
    n = 15 + 6 * M
    s = np.r_[np.full(3, drift / 5), np.full(3, 0.01), np.full(3, drift / 2), np.full(3, 0.01), np.full(3, drift),
              np.tile(np.r_[np.full(3, drift / 5), np.full(3, drift)], M)]
    A = rng.normal(size=(n, n))
    return (s[:, None] * (A @ A.T / n + np.eye(n)) * s[None, :]) / 2


def scene(rng, imu, poses, M, kinds=("range", "plane", "antenna", "heading", "body", "relative", "clone_range")):
    """items of the kinds named, measured at the state (imu, poses) with their noise: two ranges, a plane range, a GNSS
    antenna fix with a 0.5 m lever, a heading, a body velocity, a relative pose between clones 0 and M - 1 (M >= 2) and a range
    at clone M - 1 (M >= 1)"""
    from tests.test_gnss_gpu import antenna_item, heading_item
    from tests.test_odometry_gpu import body_item, rel_item
    from tests.test_range_gpu import plane_item, range_item
    items = []
    for k in kinds:
        if k == "range":
            items += [range_item(rng, imu, poses) for _ in range(2)]
        elif k == "plane":
            items.append(plane_item(rng, imu, poses))
        elif k == "antenna":
            items.append(antenna_item(rng, imu, poses, 7, lever=np.array([0.5, 0.0, 0.0])))
        elif k == "heading":
            items.append(heading_item(rng, imu, poses, axis=np.array([1.0, 0.2, 0.1])))
        elif k == "body":
            items.append(body_item(rng, imu, 7))
        elif k == "relative" and M >= 2:
            items.append(rel_item(rng, poses, 0, M - 1))
        elif k == "clone_range" and M >= 1:
            items.append(range_item(rng, imu, poses, clone=M - 1))
    return items
