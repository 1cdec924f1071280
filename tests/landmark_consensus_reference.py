"""numpy restatement of the consensus on mapped-landmark matches (msckf_b200_landmark_update_consensus, DESIGN.md 4.17):
sampling, minimal fit, scoring, selection and refit, in fp64 and in input order.

A hypothesis th = (psi, t0, t1, t2) is a rigid correction of the window about G's z axis, applied to the map:
p_L' = Rz(psi)^T (p_L - c - t) + c, with the pivot c the mean p_C_G of the clones the observations name (window order).  Observation
i (clone k, z, p_L) is an inlier of th when p_C = C_k (p_L' - p_C_G,k) has depth > 0 and e = r^T R^-1 r <= thresh, r = z - p_C[0:2] /
p_C[2].  Poses are [M, 7]: p_C_G (3), q_CG (x, y, z, w)."""
import numpy as np

from oracle.msckf_numpy import quat_to_rot

MASK = (1 << 64) - 1
STEPS = 8        # Gauss-Newton steps of the minimal fit and of the refit
STEP_TOL = 1e-12  # stop when max |step| <= this
PIVOT_REL = 1e-12  # a Cholesky pivot must be > this x its diagonal entry


def splitmix64(x):
    """splitmix64's output for state x (the state advanced by the golden gamma first)"""
    z = (x + 0x9E3779B97F4A7C15) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def sample_pairs(seed, hypotheses, n):
    """[hypotheses, 2] input-order observation pairs: i = u mod n, j = v mod (n - 1), j += 1 when j >= i, with
    u = splitmix64(seed + 2h), v = splitmix64(seed + 2h + 1) (all mod 2^64).  None when n < 2 (no pair can be drawn)."""
    if n < 2:
        return None
    out = np.zeros((hypotheses, 2), dtype=np.int64)
    for h in range(hypotheses):
        u = splitmix64((seed + 2 * h) & MASK)
        v = splitmix64((seed + 2 * h + 1) & MASK)
        i = u % n
        j = v % (n - 1)
        j += j >= i
        out[h] = i, j
    return out


def pivot(poses, clone):
    """the mean p_C_G of the clones named (ascending clone order, summed in that order)"""
    ks = sorted(set(int(k) for k in clone))
    s = np.zeros(3)
    for k in ks:
        s = s + poses[k, 0:3]
    return s / len(ks)


def weight(R):
    """R^-1 of a 2 x 2 R"""
    return np.linalg.inv(np.asarray(R, dtype=np.float64))


def model(th, c, poses, clone, z, p_L, W, jac=False):
    """per observation: front (depth > 0 and z^ finite), r [n, 2], e [n] (inf where not front) and (jac) dz^/dth [n, 2, 4]"""
    clone = np.asarray(clone)
    sn, cs = np.sin(th[0]), np.cos(th[0])
    d = np.asarray(p_L, dtype=np.float64) - c - th[1:4]
    u = np.stack([cs * d[:, 0] + sn * d[:, 1], -sn * d[:, 0] + cs * d[:, 1], d[:, 2]], axis=1) + c - poses[clone, 0:3]
    Cs = np.array([quat_to_rot(poses[k, 3:7]) for k in range(len(poses))])[clone]
    p = np.einsum("nij,nj->ni", Cs, u)
    with np.errstate(divide="ignore", invalid="ignore"):
        zh = p[:, 0:2] / p[:, 2:3]
    front = (p[:, 2] > 0) & np.all(np.isfinite(zh), axis=1)
    r = np.asarray(z, dtype=np.float64) - zh
    e = np.where(front, np.einsum("ni,ij,nj->n", np.where(front[:, None], r, 0.0), W, np.where(front[:, None], r, 0.0)), np.inf)
    if not jac:
        return front, r, e
    zero, one = np.zeros(len(d)), np.ones(len(d))
    D = np.stack([np.stack([-sn * d[:, 0] + cs * d[:, 1], -cs * one, -sn * one, zero], axis=1),
                  np.stack([-cs * d[:, 0] - sn * d[:, 1], sn * one, -cs * one, zero], axis=1),
                  np.stack([zero, zero, zero, -one], axis=1)], axis=1)  # [n, 3, 4]: dp_L'/dth
    with np.errstate(divide="ignore", invalid="ignore"):
        iz = 1.0 / p[:, 2]
        J = np.stack([np.stack([iz, zero, -zh[:, 0] * iz], axis=1), np.stack([zero, iz, -zh[:, 1] * iz], axis=1)], axis=1)
    return front, r, e, np.einsum("nij,njk,nkl->nil", J, Cs, D)


def gauss_newton(th0, c, poses, clone, z, p_L, W):
    """at most STEPS Gauss-Newton steps from th0 over all the given observations; (th, ok): ok is False when a point leaves the
    front or a pivot of the 4 x 4 Cholesky is not > PIVOT_REL x its diagonal entry"""
    th = np.array(th0, dtype=np.float64)
    for _ in range(STEPS):
        front, r, e, Jz = model(th, c, poses, clone, z, p_L, W, jac=True)
        if not front.all():
            return th, False
        H = np.einsum("nai,ab,nbj->ij", Jz, W, Jz)
        g = np.einsum("nai,ab,nb->i", Jz, W, r)
        L = np.zeros((4, 4))
        for j in range(4):
            dj = H[j, j] - L[j, :j] @ L[j, :j]
            if not dj > PIVOT_REL * H[j, j]:
                return th, False
            L[j, j] = np.sqrt(dj)
            for i in range(j + 1, 4):
                L[i, j] = (H[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
        x = np.linalg.solve(L.T, np.linalg.solve(L, g))
        th = th + x
        if np.max(np.where(np.isnan(x), np.inf, np.abs(x))) <= STEP_TOL:
            break
    return th, True


def consensus(poses, clone, z, p_L, R, hypotheses, thresh, min_inliers, seed):
    """the whole consensus of one call: a dict with pairs, th [H, 4], valid [H], scores [H] (inliers, -1 when not valid),
    e [H, n] (each hypothesis's e_i; inf behind the camera), best (-1: none valid), refit, th_final, inliers [n] (final),
    e_best / e_refit (the e_i the final choice was made on), status (0 found, 1 fewer than min_inliers) and pre [n] (0, or 3:
    excluded by consensus; k_lmk_clone keeps flag 2 first)"""
    poses = np.asarray(poses, dtype=np.float64)
    clone = np.asarray(clone)
    z = np.asarray(z, dtype=np.float64).reshape(-1, 2)
    p_L = np.asarray(p_L, dtype=np.float64).reshape(-1, 3)
    n = len(clone)
    W = weight(R)
    c = pivot(poses, clone)
    pairs = sample_pairs(seed, hypotheses, n)
    H = 0 if pairs is None else hypotheses
    th = np.zeros((hypotheses, 4))
    valid = np.zeros(hypotheses, bool)
    scores = np.full(hypotheses, -1, np.int64)
    E = np.full((hypotheses, n), np.inf)
    for h in range(H):
        i, j = pairs[h]
        sel = [i, j]
        t, ok = gauss_newton(np.zeros(4), c, poses, clone[sel], z[sel], p_L[sel], W)
        th[h] = t
        if not ok:
            continue
        _, _, e = model(t, c, poses, clone, z, p_L, W)
        E[h] = e
        if e[i] <= thresh and e[j] <= thresh:
            valid[h] = True
            scores[h] = int((e <= thresh).sum())
    out = dict(pairs=pairs, th=th, valid=valid, scores=scores, e=E, pivot=c, best=-1, refit=0, th_final=np.zeros(4),
               inliers=np.zeros(n, bool), e_best=None, e_refit=None)
    if valid.any():
        best = int(np.argmax(np.where(valid, scores, -1)))  # first maximum: the lowest index
        in0 = E[best] <= thresh
        t, ok = gauss_newton(th[best], c, poses, clone[in0], z[in0], p_L[in0], W)
        ok = ok and np.all(np.isfinite(t))
        e1 = model(t, c, poses, clone, z, p_L, W)[2] if ok else np.full(n, np.inf)
        in1 = e1 <= thresh
        refit = bool(ok and in1.sum() >= in0.sum())
        out.update(best=best, refit=int(refit), th_final=t if refit else th[best], inliers=in1 if refit else in0,
                   e_best=E[best], e_refit=e1)
    out["status"] = 0 if out["best"] >= 0 and out["inliers"].sum() >= min_inliers else 1
    out["pre"] = np.where(out["inliers"] & (out["status"] == 0), 0, 3)
    return out


def final_flags(pre, flag_plain):
    """the call's flags from the consensus's pre-set flags and the plain call's (2 first, then 3, then the gate's 1 / 0)"""
    flag_plain = np.asarray(flag_plain)
    return np.where(flag_plain == 2, 2, np.where(np.asarray(pre) == 3, 3, flag_plain))


def rz(psi):
    c, s = np.cos(psi), np.sin(psi)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def planted(rng, poses, counts, th, outlier_rate, noise=0.002, depth=(3.0, 15.0)):
    """matches whose map positions p_L are off from what the clones see by the correction th = (psi, t) about the pivot:
    the clones see p_L' = Rz(psi)^T (p_L - c - t) + c.  counts: clone -> observations (shuffled input order).  Each match is
    wrong with probability outlier_rate: its p_L is swapped for another match's.  (clone, z, p_L, wrong [n] bool)"""
    clone = np.concatenate([np.full(c, k) for k, c in counts.items()]).astype(np.int32)
    rng.shuffle(clone)
    n = len(clone)
    c = pivot(poses, clone)
    seen = np.zeros((n, 3))
    for i, k in enumerate(clone):
        d = rng.uniform(*depth)
        pc = np.array([rng.uniform(-0.4, 0.4) * d, rng.uniform(-0.3, 0.3) * d, d])
        seen[i] = quat_to_rot(poses[k, 3:7]).T @ pc + poses[k, 0:3]
    p_L = (rz(th[0]) @ (seen - c).T).T + c + np.asarray(th[1:4])  # the inverse of the correction
    z = np.array([(quat_to_rot(poses[k, 3:7]) @ (s - poses[k, 0:3])) for k, s in zip(clone, seen)])
    z = z[:, 0:2] / z[:, 2:3] + noise * rng.normal(size=(n, 2))
    wrong = rng.uniform(size=n) < outlier_rate
    for i in np.flatnonzero(wrong):
        p_L[i] = p_L[(i + 1 + rng.integers(n - 1)) % n]
    return clone, z, p_L, wrong
