"""Dense numpy fault detection and exclusion over the items of a stacked aided update (the rounds of
msckf_b200_aid_stack_update_fde, include/msckf_b200.h), in fp64, built on montecarlo.odometry_residual / odometry_jacobian,
with the Joseph-form update of the kept items, and the scenes the tests draw: stacks of side_shapes recipes with faults of a
chosen size."""
import numpy as np
from scipy.linalg import block_diag

from msckf_mono_b200 import montecarlo as mc


def linearise(items, imu, poses, n):
    """[(H_j [d_j, n], r_j [d_j])] of the items at the state (the models of montecarlo; VELOCITY, POSITION, POSE and CLONE_POSE
    as test_odometry_gpu.H_r)"""
    from tests.test_range_gpu import H_r
    return [H_r(it, imu, poses, n) for it in items]


def set_nis(S, r, rows):
    """r_A^T S_AA^-1 r_A over the stack rows `rows`"""
    return float(r[rows] @ np.linalg.solve(S[np.ix_(rows, rows)], r[rows]))


def exclusion_tests(S, r, blocks):
    """t_j = y_j^T B_j^-1 y_j (y = S_AA^-1 r_A, B_j = (S_AA^-1)_jj) of each item block (a list of index arrays into A's
    rows), over the rows of A in order"""
    rows = np.concatenate(blocks)
    Si = np.linalg.inv(S[np.ix_(rows, rows)])
    y = Si @ r[rows]
    out, k = [], 0
    for b in blocks:
        s = slice(k, k + len(b))
        out.append(float(y[s] @ np.linalg.solve(Si[s, s], y[s])))
        k += len(b)
    return out


def fde(items, imu, poses, P, chi2, max_exclude, dropped=()):
    """The rounds over the items not in `dropped` (degenerate): a dict with outcome (0 passed, 1 after exclusions, 2 at
    max_exclude, 3 not identifiable), kept (item indices of A at the end), excluded [(item, round)], nis / dof of the last set
    gated, item_nis [n_items] (NaN: dropped), tests [n_items] (t_j of the last round the item took part in, NaN: none)"""
    n = P.shape[0]
    lin = linearise([it for k, it in enumerate(items) if k not in dropped], imu, poses, n)
    idx = [k for k in range(len(items)) if k not in dropped]
    H = np.vstack([h for h, _ in lin])
    r = np.concatenate([v for _, v in lin])
    S = H @ P @ H.T + block_diag(*[items[k]["R"] for k in idx])
    first = np.cumsum([0] + [len(v) for _, v in lin])
    rows_of = {k: np.arange(first[i], first[i + 1]) for i, k in enumerate(idx)}
    item_nis = [np.nan] * len(items)
    tests = [np.nan] * len(items)
    for k in idx:
        item_nis[k] = set_nis(S, r, rows_of[k])
    A, excluded = list(idx), []
    margin = [np.inf]  # the smallest relative distance of a decision from its threshold or from a tie
    for rnd in range(len(items) + 1):
        rows = np.concatenate([rows_of[k] for k in A])
        g = set_nis(S, r, rows)
        margin.append(abs(g / chi2[len(rows) - 1] - 1.0))
        if g <= chi2[len(rows) - 1]:
            outcome = 1 if excluded else 0
            break
        if len(excluded) >= max_exclude:
            outcome = 2
            break
        if len(A) == 1:
            outcome = 3
            break
        t = exclusion_tests(S, r, [rows_of[k] for k in A])
        ratio = []
        for k, tk in zip(A, t):
            tests[k] = tk
            ratio.append(tk / chi2[len(rows_of[k]) - 1])
        j = int(np.argmax(ratio))  # (the first maximum: the lowest item index on a tie)
        margin.append(abs(ratio[j] - 1.0))
        if len(ratio) > 1:
            margin.append(1.0 - sorted(ratio)[-2] / ratio[j] if ratio[j] > 0 else 0.0)
        if not ratio[j] > 1.0:
            outcome = 3
            break
        excluded.append((A[j], rnd))
        del A[j]
    return {"outcome": outcome, "kept": A, "excluded": excluded, "nis": g, "dof": len(rows), "item_nis": item_nis,
            "tests": tests, "margin": min(margin)}


def joseph(items, imu, poses, P):
    """(P, dx, nis) of the Joseph-form update with the items, in fp64"""
    lin = linearise(items, imu, poses, P.shape[0])
    H = np.vstack([h for h, _ in lin])
    r = np.concatenate([v for _, v in lin])
    R = block_diag(*[it["R"] for it in items])
    S = H @ P @ H.T + R
    K = np.linalg.solve(S, H @ P).T
    A = np.eye(P.shape[0]) - K @ H
    return A @ P @ A.T + K @ R @ K.T, K @ r, float(r @ np.linalg.solve(S, r))


def range_scene(rng, imu, poses, n_ranges=4, sigma=0.1, faults=(), bias=2.0, gnss=False, jump=0.0, odometry=False, clone=None):
    """Items at the state (imu 19+, poses [M, 7]): n_ranges ranges (sigma m) to anchors 3..8 m away, made `bias` m long where
    their index is in `faults`; with gnss, an antenna fix (0.05 m) moved `jump` m horizontally; with odometry, a body velocity
    (0.02 m/s) and, with clone, a range at that clone"""
    p, q = imu[0:3], imu[15:19]
    items = []
    for k in range(n_ranges):
        lever = rng.normal(size=3) * 0.2
        u = rng.normal(size=3)
        anchor = p + (3.0 + 5.0 * rng.random()) * u / np.linalg.norm(u)
        rho = mc.range_of(p, q, lever, anchor) + sigma * rng.normal() + (bias if k in faults else 0.0)
        items.append({"model": mc.AID_RANGE, "a": 0, "b": 0, "z": np.r_[rho, anchor, lever], "R": np.array([[sigma ** 2]])})
    if gnss:
        lever = rng.normal(size=3) * 0.3
        d = rng.normal(size=2)
        z = mc.antenna_position(p, q, lever) + 0.05 * rng.normal(size=3) + jump * np.r_[d / np.linalg.norm(d), 0.0]
        items.append({"model": mc.AID_ANTENNA_POSITION, "a": 7, "b": 0, "z": np.r_[z, lever], "R": 0.05 ** 2 * np.eye(3)})
    if odometry:
        items.append({"model": mc.AID_BODY_VELOCITY, "a": 7, "b": 0, "z": mc.body_velocity(imu) + 0.02 * rng.normal(size=3),
                      "R": 0.02 ** 2 * np.eye(3)})
    if clone is not None:
        pc, qc = poses[clone, 0:3], poses[clone, 3:7]
        lever = rng.normal(size=3) * 0.2
        u = rng.normal(size=3)
        anchor = pc + 4.0 * u / np.linalg.norm(u)
        items.append({"model": mc.AID_CLONE_RANGE, "a": clone, "b": 0,
                      "z": np.r_[mc.range_of(pc, qc, lever, anchor) + sigma * rng.normal(), anchor, lever], "R": np.array([[sigma ** 2]])})
    return items


def recipe_items(rng, recipe, imu, poses, M):
    """the items of a recipe of tests/side_shapes.py ((model, rows, clone), clone -1: M - 1) near their predictions"""
    from msckf_mono_b200 import capi
    from tests.side_shapes import FDE_MASK
    from tests.test_aid_gpu import make_spec
    from tests.test_gnss_gpu import antenna_item
    from tests.test_odometry_gpu import body_item, rel_item
    from tests.test_range_gpu import plane_item, range_item
    items = []
    for model, rows, clone in recipe:
        k = None if clone is None else (M - 1 if clone == -1 else clone)
        if model in ("RANGE", "CLONE_RANGE"):
            it = range_item(rng, imu, poses, clone=k)
        elif model in ("PLANE_RANGE", "CLONE_PLANE_RANGE"):
            it = plane_item(rng, imu, poses, clone=k)
        elif model in ("ANTENNA_POSITION", "CLONE_ANTENNA_POSITION"):
            it = antenna_item(rng, imu, poses, FDE_MASK[rows], clone=k)
        elif model == "BODY_VELOCITY":
            it = body_item(rng, imu, FDE_MASK[rows])
        elif model == "RELATIVE_POSE":
            it = rel_item(rng, poses, 0, M - 1)
        else:  # POSE, CLONE_POSE
            it = dict(make_spec(rng, getattr(capi, "AID_" + model), imu, poses, 15 + 6 * M, k or 0)[0])
            it["a"] = it.pop("clone")
        assert len(it["R"]) == rows and it["model"] == getattr(capi, "AID_" + model), (model, rows)
        items.append(it)
    return items


def fault_rows(item):
    """(indices into z, rows of r) that a fault moves (r = z - h(x) on them): a range, an antenna fix's or a body velocity's
    masked coordinates, a pose's or a relative pose's position"""
    m = item["model"]
    if m in mc.RANGE_MODELS:
        return [0], [0]
    mask = {mc.AID_ANTENNA_POSITION: item.get("a"), mc.AID_CLONE_ANTENNA_POSITION: item.get("b"), mc.AID_BODY_VELOCITY: item.get("a")}
    if m in mask:
        rows = [j for j in range(3) if (mask[m] >> j) & 1]
        return rows, list(range(len(rows)))
    assert len(item["R"]) == 6, m  # POSE, CLONE_POSE, RELATIVE_POSE: r = [dtheta, z_p - p]
    return [0, 1, 2], [3, 4, 5]


def with_faults(rng, items, faults, ratios, imu, poses, P, chi2):
    """copies of the items with item faults[i] moved along a random direction of its fault rows by b, where b^2 e^T S_jj^-1 e =
    ratios[i] chi2[d_j - 1] (e the unit move in r, S_jj = H_j P H_j^T + R_j): the fault alone is that many thresholds"""
    out = [dict(it, z=np.array(it["z"], dtype=np.float64)) for it in items]
    for j, ratio in zip(faults, ratios):
        H, _ = linearise([out[j]], imu, poses, P.shape[0])[0]
        S = H @ P @ H.T + out[j]["R"]
        zi, ri = fault_rows(out[j])
        u = rng.normal(size=len(zi))
        u /= np.linalg.norm(u)
        e = np.zeros(len(S))
        e[ri] = u
        b = np.sqrt(ratio * chi2[len(S) - 1] / (e @ np.linalg.solve(S, e)))
        out[j]["z"][zi] += b * u
    return out
