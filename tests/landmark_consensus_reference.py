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
    ks, inv = np.unique(clone, return_inverse=True)  # (the rotations of the clones named only)
    Cs = np.array([quat_to_rot(poses[k, 3:7]) for k in ks]).reshape(-1, 3, 3)[inv.ravel()]
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


def set_counts(sets):
    """{clone set (tuple): landmarks} of a list with one clone set per landmark (tests/side_shapes.py's MAP_* lists)"""
    out = {}
    for cs in sets:
        out[tuple(cs)] = out.get(tuple(cs), 0) + 1
    return out


def planted_map(rng, poses, sets, th, swap=(), move=(), push=(), sigma=0.05, noise=0.002, outlier_rate=0.0):
    """matches of landmarks seen from several clones, as planted() draws them: sets maps a clone set (tuple, <= 8 clones) to
    its number of landmarks; landmark l has one p_L shared by all its observations, off by the correction th from what the
    clones see, and a random Sigma_L.  Wrong matches, each passing the host's map checks (one p_L per landmark, one observation
    per clone, <= 8 clones):
      swap: landmarks whose p_L is another landmark's (every observation of the landmark wrong);
      move: (landmark, clone) observations moved to another landmark id that is not seen from that clone (p_L follows the id);
      push: (landmark, clone) observations whose z is 0.05 off (the match found the wrong keypoint);
      outlier_rate: each landmark swapped with this probability, on top of `swap`.
    Landmark ids follow the order of `sets` (set by set).  (clone, z, p_L, landmark, Sigma_L [L, 6], wrong [n] bool), shuffled."""
    from tests.landmark_map_reference import landmarks_seen_from, tri
    cs_of, pts, Sig = [], [], []
    for cs, count in sets.items():
        for _ in range(count):
            cs_of.append(tuple(cs))
            pts.append(landmarks_seen_from(rng, poses, list(cs)))
            B = rng.normal(size=(3, 3)) * sigma
            Sig.append(tri(B @ B.T + sigma ** 2 * np.eye(3)))
    L = len(pts)
    c = pivot(poses, [k for cs in cs_of for k in cs])
    seen = np.array(pts)
    p_map = (rz(th[0]) @ (seen - c).T).T + c + np.asarray(th[1:4])  # each landmark's map position
    swap = set(swap) | {l for l in range(L) if rng.uniform() < outlier_rate}
    lm_pL = p_map.copy()
    for l in sorted(swap):
        lm_pL[l] = p_map[(l + 1 + rng.integers(L - 1)) % L]
    clone, z, p_L, lm, wrong = [], [], [], [], []
    members = {l: set(cs_of[l]) for l in range(L)}
    moved = {}
    for (l, k) in move:  # to the next landmark (cyclically) that k does not see and that stays within 8 clones
        for d in range(1, L):
            l2 = (l + d) % L
            if k not in members[l2] and len(members[l2]) < 8 and l2 not in swap:
                members[l2].add(k)
                members[l].discard(k)
                moved[(l, k)] = l2
                break
        else:
            raise ValueError(("no landmark to move to", l, k))
    for l in range(L):
        for k in cs_of[l]:
            pc = quat_to_rot(poses[k, 3:7]) @ (seen[l] - poses[k, 0:3])
            zz = pc[0:2] / pc[2] + noise * rng.normal(size=2) + (0.05 if (l, k) in push else 0.0)
            lid = moved.get((l, k), l)
            clone.append(k); z.append(zz); lm.append(lid); p_L.append(lm_pL[lid])
            wrong.append(l in swap or (l, k) in moved or (l, k) in push)
    o = rng.permutation(len(clone))
    return (np.array(clone, np.int32)[o], np.array(z)[o], np.array(p_L)[o], np.array(lm, np.int32)[o], np.array(Sig),
            np.array(wrong)[o])


def map_checks(clone, p_L, landmark, n_landmarks):
    """the host's checks of a map call (lmk_map_plan): ids in range, one p_L per landmark, no landmark seen twice from a
    clone, at most 8 clones per landmark; raises AssertionError"""
    clone, p_L, landmark = np.asarray(clone), np.asarray(p_L), np.asarray(landmark)
    assert landmark.min() >= 0 and landmark.max() < n_landmarks
    for l in np.unique(landmark):
        sel = landmark == l
        assert np.all(p_L[sel] == p_L[sel][0]), l
        assert len(np.unique(clone[sel])) == sel.sum() <= 8, l


def pairs_fast(seed, hypotheses, n):
    """sample_pairs for many hypotheses at once (numpy uint64; the same values)"""
    with np.errstate(over="ignore"):
        h = np.arange(hypotheses, dtype=np.uint64)
        s = np.uint64(seed % 2 ** 64)

        def sm(x):
            z = x + np.uint64(0x9E3779B97F4A7C15)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            return z ^ (z >> np.uint64(31))
        u, v = sm(s + np.uint64(2) * h), sm(s + np.uint64(2) * h + np.uint64(1))
    i = (u % np.uint64(n)).astype(np.int64)
    j = (v % np.uint64(n - 1)).astype(np.int64)
    j += j >= i
    return np.stack([i, j], axis=1)


def first_valid_layout(first, hypotheses, n, min_later=0, seeds=range(1, 10000)):
    """a seed and the observations to plant as degenerate ([n] bool) such that a hypothesis is fittable exactly when neither of
    its pair is degenerate, and the first such hypothesis is `first`: the good observations are hypothesis `first`'s pair plus,
    greedily in input order, every observation that closes no pair of an earlier hypothesis.  Searched over `seeds` until at
    least min_later hypotheses after `first` are fittable too (their ties then meet hypothesis `first` at every level of the
    arg-max).  (seed, degenerate)"""
    for seed in seeds:
        pr = pairs_fast(seed, hypotheses, n)
        a, b = pr[first]
        if any({int(x), int(y)} == {int(a), int(b)} for x, y in pr[:first]):
            continue
        adj = [set() for _ in range(n)]
        for x, y in pr[:first]:
            adj[x].add(int(y)); adj[y].add(int(x))
        good = {int(a), int(b)}
        for o in range(n):
            if o not in good and not (adj[o] & good):
                good.add(o)
        deg = np.ones(n, bool)
        deg[list(good)] = False
        ok = ~deg[pr[:, 0]] & ~deg[pr[:, 1]]
        assert np.flatnonzero(ok)[0] == first
        if ok[first + 1:].sum() >= min_later:
            return seed, deg
    raise ValueError(("no seed", first, hypotheses, n))


TIE_THRESH = 1e8  # thresh of tied(): every observation in front is an inlier of every valid hypothesis


def tied(rng, poses, counts, th, degenerate):
    """noise-free matches (planted() with noise 0, no wrong match) of the correction th, with the observations marked in
    `degenerate` moved behind their clone: a pair with one of them has no minimal fit.  At thresh TIE_THRESH every valid
    hypothesis counts the same inliers, all the observations in front (a few minimal fits of 2 points converge elsewhere
    or not at all in 8 steps; a tighter thresh would split their counts).  (clone, z, p_L)"""
    clone = np.concatenate([np.full(c, k) for k, c in sorted(counts.items())]).astype(np.int32)  # input order: clone by clone
    c = pivot(poses, clone)
    seen = np.zeros((len(clone), 3))
    for i, k in enumerate(clone):
        d = rng.uniform(3.0, 15.0)
        pc = np.array([rng.uniform(-0.4, 0.4) * d, rng.uniform(-0.3, 0.3) * d, d])
        seen[i] = quat_to_rot(poses[k, 3:7]).T @ pc + poses[k, 0:3]
    p_L = (rz(th[0]) @ (seen - c).T).T + c + np.asarray(th[1:4])
    z = np.array([(quat_to_rot(poses[k, 3:7]) @ (s - poses[k, 0:3])) for k, s in zip(clone, seen)])
    z = z[:, 0:2] / z[:, 2:3]
    for i in np.flatnonzero(degenerate):
        k = clone[i]
        p_L[i] = 2 * poses[k, 0:3] - p_L[i]  # mirrored through the camera centre: behind it under any small correction
    return clone, z, p_L


def refit_rejected(rng, poses, R, thresh, tries=4000):
    """a seeded search for a call whose best hypothesis's refit is finite but keeps fewer inliers (c1 < c0), so the
    hypothesis's own fit stays: 12 matches on clones 2 and 9 (20 % wrong, pixel noise 0.004), 8 hypotheses, consensus seed =
    the try.  Every e_i of every hypothesis and of the refit lies at least 1e-6 relative from thresh.  (clone, z, p_L, seed,
    the reference's consensus)"""
    for seed in range(tries):
        clone, z, p_L, _ = planted(rng, poses, {2: 6, 9: 6}, [0.02, 0.3, -0.2, 0.1], 0.2, noise=0.004)
        rf = consensus(poses, clone, z, p_L, R, 8, thresh, 2, seed=seed)
        if rf["best"] < 0 or rf["refit"] or not np.isfinite(rf["e_refit"]).any():  # (all inf: the refit's fit failed)
            continue
        es = np.concatenate([rf["e"].ravel(), rf["e_refit"]])
        es = es[np.isfinite(es)]
        if np.any(np.abs(es - thresh) <= 1e-6 * thresh):
            continue
        assert (rf["e_refit"] <= thresh).sum() < (rf["e_best"] <= thresh).sum()
        return clone, z, p_L, seed, rf
    raise AssertionError("no rejected refit in the search")


def map_exclusions(sets, pattern):
    """planted_map's (swap, move, push) that make the consensus exclude, from a map call over `sets` (one clone set per
    landmark, tests/side_shapes.py's MAP_* lists; ids in set_counts order):
      one_observation: one observation of landmark 0 pushed (and, where landmark 1 is seen from 2 clones, one of its
                       observations moved to another landmark);
      landmark:        every observation of landmark 1 (its p_L swapped);
      clone_set:       every landmark of the last clone set (swapped); swap None when that set is the whole call;
      clone:           every observation of one clone (the first clone of the middle landmark), pushed."""
    lms = []
    for cs, count in set_counts(sets).items():
        lms += [cs] * count
    if pattern == "one_observation":
        return (), ([(1, lms[1][0])] if len(lms[1]) == 2 else []), [(0, lms[0][0])]
    if pattern == "landmark":
        return [1], [], []
    if pattern == "clone_set":
        group = [l for l, cs in enumerate(lms) if cs == lms[-1]]
        return (None if len(group) == len(lms) else group), [], []
    assert pattern == "clone", pattern
    k = lms[len(lms) // 2][0]
    return (), [], [(l, k) for l, cs in enumerate(lms) if k in cs]
