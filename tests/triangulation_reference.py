"""A plain numpy reference of what MARGINALIZE does before the update proper, with a trace of every decision taken on the way:
  * check_motion: checkMotion (msckf.h:980-1025);
  * initialize_position: initializePosition (msckf.h:1147-1285) with generateInitialGuess (:1126-1145), cost (:1027-1047),
    jacobian (:1287-1323) and the 3x3 Eigen::LDLT solve of :1222 (ldlt3: Eigen's unblocked LDLT picks, at step k, the largest
    |diagonal| of the not yet eliminated and not yet updated entries, the first index winning a tie, and divides by a pivot
    only when it is non-zero);
  * minimiser: the least-squares answer by an independent route (scipy's trust-region solver on the plain reprojection
    residuals in the same inverse-depth parameters), to which initialize_position must agree wherever its trace says the LM
    converged and no observation sits on the Huber branch (there the LM's fixed point sum w^2 J^T r = 0 is the plain minimum);
  * loop_ab: the bookkeeping of marginalize()'s two loops (msckf.h:352-399 and :419) on flags alone: which tracks are valid,
    which pushed a position into p_f_G_vec, and which track's position loop B reads for track `iter` (p_f_G_vec[iter]: shifted
    by the rejections before it, or out of bounds);
  * designed_tracks: tracks on the trajectory of tests/vision_reference.py built to take each branch with a margin.
Everything runs in the scalar type S it is given (np.float64: the reference; np.float32: which flags an fp32 filter may
legitimately decide otherwise, see fp32_excluded).

What the designed set reaches on this trajectory (a 30 m circle with a wobble, the camera looking outward), from the algebra and
from a sweep of 4000 random geometries (lengths 2 .. 70, any clone subset, landmarks 0.5 .. 40 m):
  * the elimination order of the first solve: the (alpha, alpha) and (beta, beta) entries of the normal matrix are both ~L and
    differ by the clones' rotation times the landmark's bearing only, the (rho, rho) entry is the sum of the squared baselines
    across the bearing: below both for short tracks, above both for long ones and between them at about 34 observations.  All
    six orders occurred in the sweep (the two with rho in the middle in 33 of 4000), and the designed set takes all six;
  * a tie needs two of those sums equal to the last bit, and a zero pivot a positive semi-definite matrix plus lambda >= 1e-10
    on its diagonal with a vanishing pivot: neither occurred in the sweep, so both are exercised on ldlt3 directly (matrices,
    not tracks) and asserted absent from the designed set;
  * a landmark behind exactly one clone lies in the wedge between that clone's image plane and its neighbours': for clones
    5 cm apart the wedge is micrometres thin, so the clone in question is ten or more clones from the others of its track.  With
    that it can be the first, the last or one in the middle, handled by lane 0, 8, 11 or 31, in the first or the second
    32-stride pass (a 70-clone window has no room for one in the third);
  * the clones are 5 cm apart and a long track's path is curved by more than the threshold, so checkMotion is taken 20 % below
    and above the threshold by tracks of 2, 3 and 4 observations (the deciding clone is the last one); longer tracks pass it
    by far."""
import numpy as np
import scipy.optimize as sopt

from oracle.msckf_numpy import quat_to_rot

ORDERS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


# ---------------------------------------------------------------------------------------------------------------- the solve
def ldlt3(A, b, S=np.float64):
    """(x, order, tie, zero) of Eigen's A.ldlt().solve(b) for a symmetric 3 x 3 A: the elimination order, whether a pivot
    search met two equal candidates, and whether a pivot was zero (its row of the solve is then skipped)"""
    A = np.array(A, dtype=S)
    b = np.array(b, dtype=S)
    perm = [0, 1, 2]
    tie = False
    for k in range(2):  # pivot search on the original diagonal (left-looking: nothing is updated before its own step)
        d = [abs(A[i, i]) for i in range(k, 3)]
        j = k + int(np.argmax(d))  # argmax returns the first of equal maxima, as maxCoeff does
        tie |= sorted(d)[-1] == sorted(d)[-2]
        if j != k:
            A[[k, j]] = A[[j, k]]
            A[:, [k, j]] = A[:, [j, k]]
            b[[k, j]] = b[[j, k]]
            perm[k], perm[j] = perm[j], perm[k]
    Lm = np.eye(3, dtype=S)
    D = np.zeros(3, dtype=S)
    zero = False
    for k in range(3):
        D[k] = A[k, k] - sum((Lm[k, j] * Lm[k, j] * D[j] for j in range(k)), S(0))
        for i in range(k + 1, 3):
            v = A[i, k] - sum((Lm[i, j] * Lm[k, j] * D[j] for j in range(k)), S(0))
            Lm[i, k] = v / D[k] if abs(D[k]) > 0 else v
        zero |= not abs(D[k]) > 0
    y = np.zeros(3, dtype=S)
    for k in range(3):
        y[k] = b[k] - sum((Lm[k, j] * y[j] for j in range(k)), S(0))
    y = np.array([y[k] / D[k] if abs(D[k]) > 0 else S(0) for k in range(3)], dtype=S)
    for k in (1, 0):
        y[k] = y[k] - sum((Lm[j, k] * y[j] for j in range(k + 1, 3)), S(0))
    x = np.zeros(3, dtype=S)
    x[perm] = y
    return x, tuple(perm), bool(tie), bool(zero)


# ------------------------------------------------------------------------------------------------------------- checkMotion
def check_motion(poses, idx, obs0, threshold, S=np.float64):
    """(flag, trace): trace has the largest orthogonal translation, its margin to the threshold (ortho / threshold - 1), the
    track position of the clone that has it and how many clones exceed the threshold"""
    if len(idx) < 2:
        return False, {"ortho": 0.0, "margin": -1.0, "decider": -1, "above": 0}
    P = np.asarray(poses, dtype=S)
    first = P[idx[0]]
    d = np.array([obs0[0], obs0[1], 1.0], dtype=S)
    d = d / np.sqrt(d @ d)
    d = (quat_to_rot(first[3:7]).T.astype(S) @ d).astype(S)
    ortho = []
    for k in idx[1:]:
        t = P[k, 0:3] - first[0:3]
        o = t - (t @ d) * d
        ortho.append(np.sqrt(o @ o))
    ortho = np.array(ortho, dtype=S)
    thr = S(threshold)
    return bool(ortho.max() > thr), {"ortho": float(ortho.max()), "margin": float(ortho.max() / thr - 1),
                                     "decider": 1 + int(np.argmax(ortho)), "above": int((ortho > thr).sum())}


# ------------------------------------------------------------------------------------------------------ initializePosition
def relative_poses(poses, idx, S=np.float64):
    """(R [L, 3, 3], t [L, 3]): T_i^-1 T_0, taking a point of the first clone's frame to clone i's (msckf.h:1154-1168)"""
    P = np.asarray(poses, dtype=S)
    C = [quat_to_rot(P[k, 3:7]).astype(S) for k in idx]
    R = np.array([Ci @ C[0].T for Ci in C], dtype=S)
    t = np.array([Ci @ (P[idx[0], 0:3] - P[k, 0:3]) for Ci, k in zip(C, idx)], dtype=S)
    return R, t


def _h(R, t, x, S):
    return (R @ np.array([x[0], x[1], 1.0], dtype=S) + x[2] * t).astype(S)


def _cost(R, t, z, x, S):
    tot = S(0)
    for i in range(len(z)):
        h = _h(R[i], t[i], x, S)
        e = np.array([h[0] / h[2], h[1] / h[2]], dtype=S) - z[i]
        tot = tot + e @ e
    return tot


def initialize_position(poses, idx, obs, max_cost, S=np.float64):
    """(valid, p_f_G, trace) of a track of two or more observations.  trace: outer (passes), inner (attempts per pass), lambdas
    (after every attempt), accepted (per attempt), exit ("cap" or "delta"), converged (ended on delta_norm with the last step
    accepted), huber (observations on the Huber branch, per pass), orders / tie / zero (of every solve), min_depth and its
    observation, cost (normalized_cost) and its margin to max_cost (cost / max_cost - 1), sol (alpha, beta, rho)"""
    L = len(idx)
    R, t = relative_poses(poses, idx, S)
    z = np.asarray(obs, dtype=S).reshape(L, 2)
    # generateInitialGuess from the first and the last observation
    m = R[-1] @ np.array([z[0, 0], z[0, 1], 1.0], dtype=S)
    A = np.array([m[0] - z[-1, 0] * m[2], m[1] - z[-1, 1] * m[2]], dtype=S)
    b = np.array([z[-1, 0] * t[-1, 2] - t[-1, 0], z[-1, 1] * t[-1, 2] - t[-1, 1]], dtype=S)
    depth = (S(1) / (A @ A)) * (A @ b)
    p = np.array([z[0, 0] * depth, z[0, 1] * depth, depth], dtype=S)
    sol = np.array([p[0] / p[2], p[1] / p[2], S(1) / p[2]], dtype=S)
    lam, delta_norm, reduced = S(1e-3), S(0), False
    total = _cost(R, t, z, sol, S)
    tr = {"inner": [], "lambdas": [], "accepted": [], "huber": [], "orders": [], "tie": False, "zero": False}
    outer = 0
    while True:
        A3, b3, nh = np.zeros((3, 3), dtype=S), np.zeros(3, dtype=S), 0
        for i in range(L):
            h = _h(R[i], t[i], sol, S)
            W = np.column_stack([R[i][:, 0], R[i][:, 1], t[i]]).astype(S)
            J = np.array([S(1) / h[2] * W[0] - h[0] / (h[2] * h[2]) * W[2], S(1) / h[2] * W[1] - h[1] / (h[2] * h[2]) * W[2]], dtype=S)
            r = np.array([h[0] / h[2], h[1] / h[2]], dtype=S) - z[i]
            e = np.sqrt(r @ r)
            if e <= S(0.01):
                A3 += J.T @ J
                b3 += J.T @ r
            else:
                w = S(0.01) / (S(2) * e)
                nh += 1
                A3 += w * w * (J.T @ J)
                b3 += w * w * (J.T @ r)
        tr["huber"].append(nh)
        inner = 0
        while True:
            delta, order, tie, zero = ldlt3(A3 + lam * np.eye(3, dtype=S), b3, S)
            tr["orders"].append(order)
            tr["tie"] |= tie
            tr["zero"] |= zero
            new = (sol - delta).astype(S)
            delta_norm = np.sqrt(delta @ delta)
            c = _cost(R, t, z, new, S)
            if c < total:
                reduced, sol, total = True, new, c
                lam = S(lam / 10) if float(lam / 10) > 1e-10 else S(1e-10)
            else:
                reduced = False
                lam = S(lam * 10) if float(lam * 10) < 1e12 else S(1e12)
            tr["lambdas"].append(float(lam))
            tr["accepted"].append(reduced)
            go = inner < 10 and not reduced
            inner += 1
            if not go:
                break
        tr["inner"].append(inner)
        go = outer < 10 and delta_norm > S(5e-7)
        outer += 1
        if not go:
            break
    final = np.array([sol[0] / sol[2], sol[1] / sol[2], S(1) / sol[2]], dtype=S)
    pz = np.array([(R[i] @ final + t[i])[2] for i in range(L)], dtype=S)
    cost = total / S(2 * L * L)
    valid = bool(not (pz <= 0).any() and not cost > S(max_cost))
    C0 = quat_to_rot(np.asarray(poses, dtype=S)[idx[0], 3:7]).astype(S)
    pfg = (C0.T @ final + np.asarray(poses, dtype=S)[idx[0], 0:3]).astype(S)
    tr.update(outer=outer, exit="delta" if not delta_norm > S(5e-7) else "cap", converged=bool(not delta_norm > S(5e-7) and reduced),
              min_depth=float(pz.min()), min_depth_obs=int(np.argmin(pz)), behind=int((pz <= 0).sum()), cost=float(cost),
              cost_margin=float(cost / S(max_cost) - 1), sol=sol.astype(np.float64))
    return valid, pfg, tr


def minimiser(poses, idx, obs, x0):
    """p_f_G of the least-squares minimum of the reprojection residuals, by scipy's trust-region solver from x0 = (alpha, beta,
    rho)"""
    R, t = relative_poses(poses, idx)
    z = np.asarray(obs, dtype=np.float64).reshape(-1, 2)

    def res(x):
        h = R @ np.array([x[0], x[1], 1.0]) + x[2] * t
        return (h[:, 0:2] / h[:, 2:3] - z).ravel()

    x = sopt.least_squares(res, np.asarray(x0, np.float64), xtol=1e-15, ftol=1e-15, gtol=1e-15).x
    P = np.asarray(poses, np.float64)
    return quat_to_rot(P[idx[0], 3:7]).T @ np.array([x[0] / x[2], x[1] / x[2], 1.0 / x[2]]) + P[idx[0], 0:3]


def triangulate(poses, tracks, params, S=np.float64):
    """dict cm [N], ok [N] (bool), pfg [N, 3] (fp64; zero for a track of one observation, which is reported as rejected) and
    the traces cm_trace, tri_trace [N] (None for a track of one observation) of tracks {idx, obs} on clone poses [M, 7]"""
    N = len(tracks)
    out = {"cm": np.zeros(N, bool), "ok": np.zeros(N, bool), "pfg": np.zeros((N, 3)), "cm_trace": [None] * N, "tri_trace": [None] * N}
    for j, tk in enumerate(tracks):
        idx = [int(k) for k in tk["idx"]]
        if len(idx) < 2:
            continue
        obs = np.asarray(tk["obs"], dtype=S)
        out["cm"][j], out["cm_trace"][j] = check_motion(poses, idx, obs[0], params["translation_threshold"], S)
        out["ok"][j], pfg, out["tri_trace"][j] = initialize_position(poses, idx, obs, params["max_gn_cost_norm"], S)
        out["pfg"][j] = pfg.astype(np.float64)
    return out


# -------------------------------------------------------------------------------------------------------------- loops A, B
def loop_ab(cm, tri, counter0):
    """marginalize()'s bookkeeping on flags: cm[k], tri[k] what checkMotion and initializePosition return for track k, counter0
    num_feature_tracks_residualized_ before the call.  Returns dict valid, pushed [N] (bool), src [N] (the track whose position
    loop B uses for track k: p_f_G_vec[k]'s owner, or k itself where that read is out of bounds or k is not valid),
    pfg_shifted, pfg_oob (counts over the valid tracks) and counter (after)"""
    N = len(cm)
    counter = int(counter0)
    valid, pushed, vec = np.zeros(N, bool), np.zeros(N, bool), []
    for k in range(N):  # :352-399
        if counter > 3 and not cm[k]:
            continue
        pushed[k] = True
        vec.append(k)  # p_f_G_vec.push_back: whether valid or not (:374)
        if tri[k]:
            valid[k] = True
            counter += 1
    src = np.arange(N)
    shifted = oob = 0
    for it in range(N):  # :414-419
        if not valid[it]:
            continue
        if it < len(vec):
            src[it] = vec[it]
            shifted += int(vec[it] != it)
        else:
            oob += 1
    return {"valid": valid, "pushed": pushed, "src": src, "pfg_shifted": shifted, "pfg_oob": oob, "counter": counter}


# ---------------------------------------------------------------------------------------------------------- designed tracks
def _observe(poses, idx, p):
    """(obs [L, 2], depths [L]) of the point p in the clones idx"""
    out, pz = np.empty((len(idx), 2)), np.empty(len(idx))
    for i, k in enumerate(idx):
        pc = quat_to_rot(poses[k, 3:7]) @ (p - poses[k, 0:3])
        out[i], pz[i] = pc[0:2] / pc[2], pc[2]
    return out, pz


def _ahead(poses, k, lateral, depth):
    """the point at (lateral * depth, 0.1 * depth, depth) in clone k's frame"""
    return quat_to_rot(poses[k, 3:7]).T @ np.array([lateral * depth, 0.1 * depth, depth]) + poses[k, 0:3]


def motion_track(poses, idx, factor, threshold):
    """a track whose largest orthogonal translation is factor * threshold: the bearing of its first observation is tilted from
    the direction of travel towards the first clone's optical axis by the angle that makes it so (found by bisection: the
    orthogonal translation grows with the tilt); the landmark is 6 m along that bearing, in front of every clone"""
    p0 = poses[idx[0], 0:3]
    C0 = quat_to_rot(poses[idx[0], 3:7])
    tang = poses[idx[-1], 0:3] - p0
    tang = tang / np.linalg.norm(tang)
    axis = C0[2] - (C0[2] @ tang) * tang
    axis = axis / np.linalg.norm(axis)

    def ortho(theta):
        d = np.cos(theta) * tang + np.sin(theta) * axis
        T = poses[idx[1:], 0:3] - p0
        return np.linalg.norm(T - np.outer(T @ d, d), axis=1).max()

    lo, hi = 0.0, np.pi / 2
    assert ortho(lo) < factor * threshold < ortho(hi), (ortho(lo), ortho(hi))
    theta = sopt.brentq(lambda th: ortho(th) - factor * threshold, lo, hi, xtol=1e-14)
    p = p0 + 6.0 * (np.cos(theta) * tang + np.sin(theta) * axis)
    obs, pz = _observe(poses, idx, p)
    assert pz.min() > 0.05, pz.min()
    return obs


def grazing_track(poses, idx, behind):
    """a track whose landmark is behind exactly the clone at track position `behind`: it lies 3 m to the side of that clone, half
    way between its image plane and the nearest of the other clones' image planes"""
    C = quat_to_rot(poses[idx[behind], 3:7])
    for ang in np.arange(16) * np.pi / 8:  # the wedge between the image planes opens on the side the other clones turned to
        base = poses[idx[behind], 0:3] + 3.0 * (np.cos(ang) * C[0] + np.sin(ang) * C[1])
        a = np.array([(quat_to_rot(poses[k, 3:7]) @ (base - poses[k, 0:3]))[2] for k in idx])
        b = np.array([(quat_to_rot(poses[k, 3:7]) @ C[2])[2] for k in idx])
        roots = np.delete(-a / b, behind)  # depth along the axis at which clone k sees the point at depth zero
        if roots.max() < -1e-3:
            break
    else:
        return None  # no such wedge: the other clones' image planes leave no room on any side
    obs, pz = _observe(poses, idx, base + 0.5 * roots.max() * C[2])
    assert (pz <= 0).sum() == 1 and pz[behind] < 0, pz
    return obs


def noisy_track(poses, seed):
    """3 .. 8 observations of a landmark 2 .. 30 m away under 5 .. 50 milli-units of noise (15 .. 150 pixels): the LM converges
    slowly on such tracks, so they are where its loop limits and the damping's floor are met (NOISY_SEEDS)"""
    rng = np.random.default_rng(seed)
    L = int(rng.integers(3, 9))
    idx = np.sort(rng.choice(70, L, replace=False))
    obs, _ = _observe(poses, idx, _ahead(poses, idx[L // 2], 0.2, float(rng.uniform(2, 30))))
    return idx, obs + rng.uniform(0.005, 0.05) * rng.normal(size=obs.shape)


def designed_tracks(poses, threshold, seed=0):
    """[{name, kind, idx, obs}] on clone poses [M >= 70, 7] (fp64) for a filter whose translation_threshold is `threshold`
    (DESIGN_THRESHOLD: above the 5 cm between clones, so that short tracks can be made to fail).  kind is what the track is built
    for: "clean", "motion-" / "motion+" (checkMotion 20 % below / above the threshold), "behind" (cheirality), "cost" (gross
    outliers), "huber" (mild outliers, accepted), "parallax" (5 cm of baseline at 8 m), "noisy" (slow LM), "order" (an elimination order)."""
    rng = np.random.default_rng(seed)
    M = len(poses)
    assert M >= 70
    out = []

    def add(name, kind, idx, obs):
        out.append({"name": name, "kind": kind, "idx": np.asarray(idx, np.int32), "obs": np.asarray(obs, np.float64)})

    sigma = 3e-4  # a tenth of a pixel, in normalised coordinates
    for L in (2, 3, 4):
        for sign, factor in (("-", 0.8), ("+", 1.2)):
            idx = np.arange(M - L, M) if L > 2 else np.array([M - 3, M - 1])
            add(f"motion{sign}{L}", "motion" + sign, idx, motion_track(poses, idx, factor, threshold))
    # the clone behind which the landmark lies is 19 or more clones from the others of its track: the wedge between their
    # image planes is then wide enough for observations of a few tens (normalised), not thousands
    head = list(range(31))
    # (clones before, clones after, track position of the clone behind which the landmark lies): that clone is the first
    # of those between the two groups that leaves a wedge
    for before, after in (([0], [69]), ([], list(range(30, 61))), (head + [40], []), (head, []), (list(range(40)), []),
                          (list(range(11)), list(range(49, 70)))):
        lo, hi = (before[-1] + 10 if before else 0), (after[0] - 10 if after else M)
        got = [(k, grazing_track(poses, np.array(before + [k] + after), len(before))) for k in range(lo, hi)]
        k, obs = next((k, o) for k, o in got if o is not None)
        add(f"behind{len(before) + 1 + len(after)}@{len(before)}", "behind", before + [k] + after, obs)
    for L, every in ((3, 1), (6, 3), (12, 3), (24, 3)):
        idx = np.sort(rng.choice(M, L, replace=False))
        obs, _ = _observe(poses, idx, _ahead(poses, idx[L // 2], 0.2, 5.0))
        obs[1::every] += 0.3 * rng.choice([-1.0, 1.0], size=obs[1::every].shape)
        add(f"cost{L}", "cost", idx, obs)
    for L in (4, 10, 40, 66):
        idx = np.sort(rng.choice(M, L, replace=False))
        obs, _ = _observe(poses, idx, _ahead(poses, idx[L // 2], -0.2, 4.0))
        obs += sigma * rng.normal(size=obs.shape)
        obs[L // 2] += [0.02, -0.015]
        add(f"huber{L}", "huber", idx, obs)
    for k, noise in ((5, 0.0), (40, sigma), (68, 3 * sigma)):
        idx = np.array([k, k + 1])
        obs, _ = _observe(poses, idx, _ahead(poses, k, 0.1, 8.0))
        add(f"parallax{k}", "parallax", idx, obs + noise * rng.normal(size=obs.shape))
    for sd in NOISY_SEEDS:
        add(f"noisy{sd}", "noisy", *noisy_track(poses, sd))
    # elimination orders of the first solve: the landmark's side (alpha's sign) orders the alpha and beta entries, the track's
    # length and the landmark's depth place the rho entry below, between or above them
    for name, idx, lateral, depth in ORDER_TRACKS:
        idx = np.asarray(idx)
        obs, pz = _observe(poses, idx, _ahead(poses, idx[0], lateral, depth))
        assert pz.min() > 0.5
        add(name, "order", idx, obs + sigma * rng.normal(size=obs.shape))
    for j, L in enumerate((2, 3, 31, 32, 33, 63, 64, 65, 70)):
        idx = np.arange(L) if j % 2 else np.sort(rng.choice(M, L, replace=False))
        obs, _ = _observe(poses, idx, _ahead(poses, idx[L // 2], 0.3 * (-1) ** j, 3.0 + j))
        add(f"clean{L}", "clean", idx, obs + sigma * rng.normal(size=obs.shape))
    return out


DESIGN_THRESHOLD = 0.0625
# (name, clones, lateral offset / depth, depth in the first clone) of the tracks that take the elimination orders of
# ORDERS_REACHED in their first solve
ORDER_TRACKS = [("order021", range(26, 60), 0.146, 1.7), ("order120", range(7, 42), -0.433, 22.3)]
ORDERS_REACHED = list(ORDERS)
# noisy_track seeds whose LM stops on the 11-pass cap (17, 24, 25, 33: the first three with lambda at its floor, 25 rejected
# on cost) or takes seven accepted steps in a row to the floor 1e-10 and then ends on delta_norm (1, 8)
NOISY_SEEDS = (1, 8, 17, 24, 25, 33)


def fp32_excluded(poses, tracks, params):
    """names of the tracks of which an fp32 run of this reference decides a flag otherwise than the fp64 run (on the poses and
    observations rounded to fp32): an fp32 filter may legitimately decide them either way"""
    p32 = np.asarray(poses, np.float32).astype(np.float64)
    t32 = [dict(t, obs=np.asarray(t["obs"], np.float32).astype(np.float64)) for t in tracks]
    a, b = triangulate(p32, t32, params, np.float64), triangulate(p32, t32, params, np.float32)
    return [t["name"] for j, t in enumerate(tracks) if a["cm"][j] != b["cm"][j] or a["ok"][j] != b["ok"][j]]
FP32_EXCLUDED = ()
