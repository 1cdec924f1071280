"""The consensus on mapped-landmark matches (k_lmk_hyp, k_lmk_cons, k_lmk_clone's CONS form) at every window, observation,
hypothesis and map-group shape its kernels dispatch on (tests/side_shapes.py, CONS_*), in fp64 and fp32:
  (a) windows 91 .. 192 with clones 0, M / 2 and M - 1 observed, all 192 clones touched, 255 and 256 observations of one
      clone, 4096 of one member (every inlier bit of a k_lmk_cons thread) and 4097 refused, each with 30 % wrong matches;
  (b) 1, 7, 8, 9, 1023 and 1024 hypotheses (k_lmk_hyp's CTA edges), and 1024 hypotheses over 2 observations;
  (c) ties: the first valid hypothesis at 0 .. 1023 with every valid hypothesis tied, resolved to its index at every level
      of k_lmk_cons's arg-max;
  (d) degenerate pairs, a refit rejected for having fewer inliers, min_inliers at and one above the final count;
  (e) map uncertainty with landmarks seen from 2 .. 8 clones, the consensus excluding one observation of a landmark, all of
      a landmark, every landmark of a clone set and every observation of a clone, single and iterated, against the dense
      marginal EKF (tests/landmark_map_reference.py) and the plain map call on the kept matches;
  (f) consensus-excluded rows below k_lmk_gain's planned stride and across its panel edges;
  (g) one device batch of 40 members, every member bit for bit its single call.
The consensus is held to tests/landmark_consensus_reference.py (a count or flag may differ only through an observation within
1e-9 relative of thresh, see test_landmark_consensus_gpu.check_against_reference); every designed case asserts on the
device's outputs that it took the path it names.  Floating-point differences to the dense references are held to the side
updates' ceilings and to 10 x the measurement below."""
import json

import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import landmark_consensus_reference as ref, landmark_map_reference as mref, side_shapes as ss
from tests.test_aid_gpu import assert_unchanged, numpy_update, snapshot
from tests.test_batch_stream_gpu import Member
from tests.test_landmark_consensus_gpu import KEYS, R_PIX, THRESH, check_against_reference, cons, correction, near
from tests.test_landmark_gpu import dense, state_of
from tests.test_side_shapes_gpu import CONTRACT, lmk_checked

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
# worst relative differences to the dense references, measured on an H100 80GB HBM3 (700 W power limit) by this file; asserted
# at 10 x
MEASURED = {
    "lmk": {"float32": {"P": 5.83e-8, "state": 5.09e-8, "nis": 9.53e-12, "dx": 7.77e-12, "gamma": 5.46e-16},
            "float64": {"P": 2.21e-14, "state": 5.05e-12, "nis": 1.78e-11, "dx": 4.51e-12, "gamma": 3.65e-14}},
    "map": {"float32": {"P": 5.61e-8, "state": 5.12e-8, "nis": 5.98e-11, "dx": 4.51e-11, "gamma": 6.84e-16},
            "float64": {"P": 5.20e-12, "state": 5.27e-12, "nis": 1.04e-10, "dx": 3.63e-11, "gamma": 4.02e-14}},
    "map_iter": {"float32": {"P": 5.59e-8, "state": 5.07e-8, "nis": 6.15e-11, "gamma": 1.49e-14},
                 "float64": {"P": 2.97e-12, "state": 3.70e-12, "nis": 5.23e-11, "gamma": 6.07e-14}},
    # the consensus call against the plain call on the kept matches where that call regroups (both on the device; fp32: the
    # state rounds to the same float32 values)
    "regroup": {"float32": {"P": 2.63e-10, "state": 0.0, "nis": 3.73e-12},
                "float64": {"P": 6.26e-12, "state": 4.93e-13, "nis": 4.97e-12}},
}
REFIT_THRESH = 6.0
QUIET = 0.0005  # pixel noise of the designed cases: every right match far inside thresh, every pushed one far outside
_BASE = {}


def fresh(dtype, M):
    """a copy of one engine per (dtype, window), built once"""
    key = (np.dtype(dtype).name, M)
    cap = min(M + 2, ss.K["kMaxKeep"])
    if key not in _BASE:
        _BASE[key] = Member(dtype, M, seed=700 + M, max_clones=cap)
    return _BASE[key].twin(dtype, max_clones=cap)


def settle(worst, rel, name, where):
    for k, v in rel.items():
        assert v <= CONTRACT[name], (where, k, v)
        worst[k] = max(worst.get(k, 0.0), v)


def assert_measured(group, name, worst):
    print(f"MEASURED {group} {name} " + json.dumps({k: float(f"{v:.3g}") for k, v in worst.items()}))
    for k, v in worst.items():
        assert v <= 10 * MEASURED[group][name][k], (group, k, v, MEASURED[group][name][k])


def same_call(got, want, keep):
    """the consensus call `got` is the plain call `want` on the observations `keep`, bit for bit"""
    for k in KEYS:
        assert got[k] == want[k], (k, got[k], want[k])
    assert np.array_equal(got["gamma"][keep], want["gamma"], equal_nan=True) and np.array_equal(got["flag"][keep], want["flag"])


def same_state(a, b):
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)


def pushed(rng, poses, counts, wrong):
    """planted() matches of correction(0.3) at pixel noise QUIET over counts + wrong (clone -> observations); of clone k,
    wrong[k] observations have z 0.05 off.  (clone, z, p_L, wrong [n] bool)"""
    allc = {k: counts.get(k, 0) + wrong.get(k, 0) for k in sorted(set(counts) | set(wrong))}
    clone, z, p_L, _ = ref.planted(rng, poses, allc, correction(0.3), 0.0, noise=QUIET)
    bad = np.zeros(len(clone), bool)
    for k, w in wrong.items():
        bad[np.flatnonzero(clone == k)[:w]] = True
    z = z + 0.05 * bad[:, None]
    return clone, z, p_L, bad


# ---- (a) windows and sizes ------------------------------------------------------------------------------------------------
def size_cases():
    out = [(M, {0: 12, M // 2: 12, M - 1: 12}) for M in ss.CONS_WINDOWS]
    out.append((192, dict(ss.CONS_ALL)))
    out += [(192, {191: c, 0: 8}) for c in ss.CONS_PER_CLONE]
    out.append((192, dict(ss.CONS_FULL)))
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_windows_and_sizes(dtype):
    rng = np.random.default_rng(101)
    for M, counts in size_cases():
        a, b, c = fresh(dtype, M), fresh(dtype, M), fresh(dtype, M)
        _, poses = state_of(a.e)
        clone, z, p_L, wrong = ref.planted(rng, poses, counts, correction(0.3), 0.3)
        n = len(clone)
        seed, mi = M + n, n // 2
        res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(64, seed=seed, min_inliers=mi))
        plain = b.e.landmark_update(clone, z, p_L, R=R_PIX)
        rf = ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, mi, seed=seed)
        check_against_reference(res, rf, plain["flag"])
        assert res["consensus"]["status"] == 0 and not np.any((res["flag"] == 0) & wrong), (M, n)
        assert np.mean(res["flag"][~wrong] == 0) > 0.95
        if n == ss.K["kLmkMaxObs"]:  # the last bit-row of every k_lmk_cons thread (packed: by clone, stable) is kept in part
            last = np.argsort(clone, kind="stable")[n - ss.K["kLmkThreads"]:]
            assert np.any(res["flag"][last] == 0) and np.any(res["flag"][last] == 3)
        keep = res["flag"] != 3
        same_call(res, c.e.landmark_update(clone[keep], z[keep], p_L[keep], R=R_PIX), keep)
        same_state(a, c)
    # one observation past kLmkMaxObs: refused before anything is written
    m = fresh(dtype, 192)
    _, poses = state_of(m.e)
    counts = dict(ss.CONS_FULL)
    counts[next(k for k in range(192) if k not in counts)] = 1
    clone, z, p_L, _ = ref.planted(rng, poses, counts, correction(0.3), 0.3)
    assert len(clone) == ss.K["kLmkMaxObs"] + 1
    before = snapshot(m.e)
    with pytest.raises(RuntimeError, match="rc=-3"):
        m.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(64))
    assert b"n_obs" in capi.lib().msckf_b200_last_error()
    assert_unchanged(snapshot(m.e), before)


# ---- (b) hypothesis counts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_hypothesis_counts(dtype):
    rng = np.random.default_rng(102)
    M = 12
    for H in ss.CONS_HYP:
        a, b = fresh(dtype, M), fresh(dtype, M)
        _, poses = state_of(a.e)
        clone, z, p_L, wrong = ref.planted(rng, poses, {0: 20, 5: 20, 11: 20}, correction(0.3), 0.3)
        res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(H, seed=H))
        plain = b.e.landmark_update(clone, z, p_L, R=R_PIX)
        rf = ref.consensus(poses, clone, z, p_L, R_PIX, H, THRESH, 2, seed=H)
        assert len(res["consensus"]["scores"]) == H
        check_against_reference(res, rf, plain["flag"])
    # 2 observations, 1024 hypotheses: every pair is (0, 1) or (1, 0), each fits both exactly
    a = fresh(dtype, M)
    _, poses = state_of(a.e)
    clone, z, p_L, _ = ref.planted(rng, poses, {3: 1, 8: 1}, correction(0.3), 0.0)
    rf = ref.consensus(poses, clone, z, p_L, R_PIX, 1024, THRESH, 2, seed=5)
    assert {tuple(sorted(p)) for p in rf["pairs"].tolist()} == {(0, 1)} and rf["valid"].all()
    c = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(1024, seed=5))["consensus"]
    assert (c["status"], c["best"], c["valid"], c["inliers"]) == (0, 0, 1024, 2) and np.all(c["scores"] == 2)


# ---- (c) ties -------------------------------------------------------------------------------------------------------------
TIE_COUNTS = {0: 32, 4: 32, 8: 32, 11: 32}


def tie_case(rng, poses, first):
    """(seed, clone, z, p_L, degenerate) whose first valid hypothesis of 1024 is `first`, every valid one tied"""
    seed, deg = ref.first_valid_layout(first, ss.K["kLmkMaxHyp"], ss.CONS_TIE_OBS, min_later=0 if first == 1023 else 8)
    clone, z, p_L = ref.tied(rng, poses, TIE_COUNTS, correction(0.3), deg)
    return seed, clone, z, p_L, deg


@pytest.mark.parametrize("dtype", DTYPES)
def test_ties_resolve_to_the_first_valid_hypothesis(dtype):
    rng = np.random.default_rng(103)
    H = ss.K["kLmkMaxHyp"]
    for first in ss.CONS_FIRST:
        a = fresh(dtype, 12)
        _, poses = state_of(a.e)
        seed, clone, z, p_L, deg = tie_case(rng, poses, first)
        rf = ref.consensus(poses, clone, z, p_L, R_PIX, H, ref.TIE_THRESH, 2, seed=seed)
        valid = np.flatnonzero(rf["valid"])
        assert valid[0] == first and rf["best"] == first and np.all(rf["scores"][valid] == (~deg).sum())
        if first < 1023:  # a tie in another warp of k_lmk_cons, and one in another pass of its stride (but for 257)
            assert len({(h % 256) // 32 for h in valid}) > 1
        res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(H, seed=seed, thresh=ref.TIE_THRESH))
        c = res["consensus"]
        assert c["best"] == first, (first, c["best"])
        assert np.array_equal(c["scores"], rf["scores"]) and c["valid"] == len(valid)
        assert c["refit"] == 1 == rf["refit"] and c["inliers"] == (~deg).sum() and c["status"] == 0
        assert np.array_equal(res["flag"], np.where(deg, 2, 0))  # the degenerate ones are behind their clone


# ---- (d) branches ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_degenerate_pairs_are_not_valid(dtype):
    rng = np.random.default_rng(104)
    a, b = fresh(dtype, 12), fresh(dtype, 12)
    _, poses = state_of(a.e)
    clone, z, p_L, _ = ref.planted(rng, poses, {2: 10, 9: 10}, correction(0.3), 0.0)
    clone[1], z[1], p_L[1] = clone[0], z[0], p_L[0]  # one observation twice: a pair of the two has rank 2 of 4
    rf = ref.consensus(poses, clone, z, p_L, R_PIX, 1024, THRESH, 2, seed=11)
    hs = [h for h, p in enumerate(rf["pairs"].tolist()) if sorted(p) == [0, 1]]
    assert hs
    W, c = ref.weight(R_PIX), ref.pivot(poses, clone)
    assert ref.model(np.zeros(4), c, poses, clone[:2], z[:2], p_L[:2], W)[0].all()  # in front: the Cholesky fails the fit
    assert not ref.gauss_newton(np.zeros(4), c, poses, clone[:2], z[:2], p_L[:2], W)[1]
    res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(1024, seed=11))
    assert np.all(res["consensus"]["scores"][hs] == -1) and not rf["valid"][hs].any()
    check_against_reference(res, rf, b.e.landmark_update(clone, z, p_L, R=R_PIX)["flag"])
    # every pair degenerate (2 and 5 copies of one observation): no valid hypothesis, nothing written
    m = fresh(dtype, 12)
    before = snapshot(m.e)
    for copies in (2, 5):
        r = m.e.landmark_update(np.repeat(clone[:1], copies), np.repeat(z[:1], copies, 0), np.repeat(p_L[:1], copies, 0), R=R_PIX,
                                consensus=cons(16))
        c = r["consensus"]
        assert (c["status"], c["valid"], c["best"], r["applied"], r["used"]) == (1, 0, -1, 0, 0)
        assert np.all(c["scores"] == -1) and np.all(r["flag"] == 3)
        assert_unchanged(snapshot(m.e), before)


@pytest.mark.parametrize("dtype", DTYPES)
def test_refit_with_fewer_inliers_is_rejected(dtype):
    rng = np.random.default_rng(105)
    a, b = fresh(dtype, 12), fresh(dtype, 12)
    _, poses = state_of(a.e)
    clone, z, p_L, seed, rf = ref.refit_rejected(rng, poses, R_PIX, REFIT_THRESH)
    res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(8, seed=seed, thresh=REFIT_THRESH))
    c = res["consensus"]
    assert c["refit"] == 0 and c["best"] == rf["best"] and c["inliers"] == (rf["e_best"] <= REFIT_THRESH).sum()
    assert np.allclose([c["yaw"], *c["t"]], rf["th"][rf["best"]], rtol=1e-9, atol=1e-12)  # the hypothesis's own fit
    check_against_reference(res, rf, b.e.landmark_update(clone, z, p_L, R=R_PIX)["flag"])


@pytest.mark.parametrize("dtype", DTYPES)
def test_min_inliers_at_and_above_the_final_count(dtype):
    rng = np.random.default_rng(106)
    a, b = fresh(dtype, 12), fresh(dtype, 12)
    _, poses = state_of(a.e)
    clone, z, p_L, wrong = ref.planted(rng, poses, {0: 15, 6: 15, 11: 15}, correction(0.3), 0.3, noise=QUIET)
    rf = ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, 2, seed=3)
    k = int(rf["inliers"].sum())
    assert not near(rf["e_best"]).any() and not near(rf["e_refit"]).any() and k == (~wrong).sum()
    res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(64, seed=3, min_inliers=k))
    assert (res["consensus"]["status"], res["consensus"]["inliers"], res["applied"], res["used"]) == (0, k, 1, k)
    before = snapshot(b.e)
    res = b.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(64, seed=3, min_inliers=k + 1))
    assert (res["consensus"]["status"], res["consensus"]["inliers"], res["applied"], res["used"]) == (1, k, 0, 0)
    assert np.all(res["flag"] == 3)
    assert_unchanged(snapshot(b.e), before)  # P, the state and the launch count


# ---- (e) map uncertainty with multi-clone landmarks -----------------------------------------------------------------------
def map_reference(P, imu, poses, clone, z, p_L, lm, Sig, used, max_iter):
    """the dense marginal EKF on the used observations (landmark ids remapped): (update tuple, gamma of every observation)"""
    ids = np.unique(lm[used])
    remap = np.searchsorted(ids, lm[used]).astype(np.int32)
    gam = mref.dense(P, poses, clone, z, p_L, lm, Sig, R_PIX)[5]
    if max_iter <= 1:
        H, r, Rb = mref.dense(P, poses, clone[used], z[used], p_L[used], remap, Sig[ids], R_PIX)[0:3]
        return numpy_update(P, imu, poses, H, r, Rb), gam, remap, ids
    w = mref.iekf(P, imu, poses, clone[used], z[used], p_L[used], remap, Sig[ids], R_PIX, max_iter=max_iter, tol=0.0)
    assert w["iterations"] == max_iter
    return (w["P"], w["imu"], w["poses"], w["nis"], None), gam, remap, ids


def rel(a, b):
    return np.abs(a.astype(np.float64) - b.astype(np.float64)).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("dtype", DTYPES)
def test_map_uncertainty_with_multi_clone_landmarks(dtype):
    rng = np.random.default_rng(107)
    name = np.dtype(dtype).name
    worst = {"map": {}, "map_iter": {}, "regroup": {}}
    M = 192
    for shape, sets in ss.CONS_MAP.items():
        cases = [(p, 0) for p in ss.CONS_MAP_PATTERNS] + [("all", 8)]
        for pattern, mi in cases:
            if pattern == "all":  # the iterated update with every pattern at once
                pats = [ref.map_exclusions(sets, p) for p in ss.CONS_MAP_PATTERNS]
                pats = [p for p in pats if p is not None and p[0] is not None]
                swap = sorted({l for p in pats for l in p[0]})
                move = [m for p in pats for m in p[1]]
                push = [m for p in pats for m in p[2]]
            else:
                got = ref.map_exclusions(sets, pattern)
                if got[0] is None:
                    continue
                swap, move, push = got
            a, b = fresh(dtype, M), fresh(dtype, M)
            imu, poses = state_of(a.e)
            P = a.e.covariance().astype(np.float64)
            clone, z, p_L, lm, Sig, wrong = ref.planted_map(rng, poses, ref.set_counts(sets), correction(0.3), swap=swap, move=move,
                                                            push=push, noise=QUIET)
            ref.map_checks(clone, p_L, lm, len(Sig))
            res = a.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=mi, tol=0.0, landmark=lm, Sigma_L=Sig,
                                      consensus=cons(64, seed=len(clone)))
            where = (shape, pattern, mi)
            assert res["consensus"]["status"] == 0, where
            used = res["flag"] == 0
            assert np.array_equal(used, ~wrong), where  # every wrong match out (3, or 2 behind its clone), every right one in
            assert np.all(res["flag"][wrong] != 0) and np.all(np.isin(res["flag"][wrong], (2, 3)))
            partial = [l for l in np.unique(lm) if 0 < used[lm == l].sum() < (lm == l).sum()]
            assert bool(partial) == (pattern in ("one_observation", "clone", "all")), where
            refu, gam, remap, ids = map_reference(P, imu, poses, clone, z, p_L, lm, Sig, used, mi)
            if mi > 1:
                assert res["iterations"] == mi and res["converged"] == 0
                refu = refu[:4] + (res["dx_norm"],)
            r = lmk_checked(res, a.e, refu, gam, res["flag"], imu, mref.rows(clone, lm, res["flag"]))
            if mi > 1:
                del r["dx"]
            settle(worst["map_iter" if mi > 1 else "map"], r, name, where)
            kept = dict(R=R_PIX, max_iter=mi, tol=0.0, landmark=remap, Sigma_L=Sig[ids])
            if partial and mref.rows(clone[used], remap, np.zeros(used.sum())) > ss.K["kLmkMaxRows"]:
                # regrouped past the cap (a landmark that lost a clone forms a set of its own): the plain call on the kept
                # matches is refused, the consensus call over the input's groups is not
                before = snapshot(b.e)
                with pytest.raises(RuntimeError, match="rc=-3"):
                    b.e.landmark_update(clone[used], z[used], p_L[used], **kept)
                assert b"rows" in capi.lib().msckf_b200_last_error()
                assert_unchanged(snapshot(b.e), before)
                continue
            plain = b.e.landmark_update(clone[used], z[used], p_L[used], **kept)
            for k in ("dof", "used", "applied", "status", "iterations", "converged"):
                assert res[k] == plain[k], (where, k)
            assert np.array_equal(res["flag"][used], plain["flag"])
            if not partial:  # the same groups less whole landmarks: bit for bit
                same_call(res, plain, used)
                same_state(a, b)
            else:  # regrouped (a landmark that lost some of its clones): held to the ceilings
                xa, xb = a.snapshot(), b.snapshot()
                settle(worst["regroup"], {"P": rel(xa[2], xb[2]), "state": max(rel(xa[0], xb[0]), rel(xa[1], xb[1])),
                                          "nis": abs(res["nis"] - plain["nis"]) / plain["nis"]}, name, where)
    for group, w in worst.items():
        assert_measured(group, name, w)


# ---- (f) consensus-excluded rows across k_lmk_gain's panel edges ----------------------------------------------------------
def excluded_rows_cases():
    """(right, wrong) clone -> observations: LMK_GATE's middle clone all wrong, and cons_sweep at every LMK_SWEEP_ROWS"""
    out = []
    for counts in ss.CONS_GATE:
        clones = sorted(counts)
        mid = clones[len(clones) // 2]
        out.append(({k: a for k, a in counts.items() if k != mid}, {mid: counts[mid]}))
    return out + [ss.cons_sweep(192, rows) for rows in ss.CONS_SWEEP_ROWS]


@pytest.mark.parametrize("dtype", DTYPES)
def test_excluded_rows_below_the_planned_stride(dtype):
    rng = np.random.default_rng(108)
    name = np.dtype(dtype).name
    worst = {}
    for right, wrong_counts in excluded_rows_cases():
        a, b = fresh(dtype, 192), fresh(dtype, 192)
        imu, poses = state_of(a.e)
        P = a.e.covariance().astype(np.float64)
        clone, z, p_L, wrong = pushed(rng, poses, right, wrong_counts)
        used_rows = ss.lmk_rows(right)
        planned = ss.lmk_rows({k: int(np.sum(clone == k)) for k in np.unique(clone)})
        assert planned > used_rows
        res = a.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(64, seed=planned))
        assert np.array_equal(res["flag"] == 3, wrong) and res["rows"] == used_rows, (used_rows, res["rows"])
        H, r, Rb, gam, flag = dense(P, poses, clone[~wrong], z[~wrong], p_L[~wrong], R_PIX)
        gam_all = dense(P, poses, clone, z, p_L, R_PIX)[3]
        rel_ = lmk_checked(res, a.e, numpy_update(P, imu, poses, H, r, Rb), gam_all, np.where(wrong, 3, 0), imu, used_rows)
        settle(worst, rel_, name, used_rows)
        same_call(res, b.e.landmark_update(clone[~wrong], z[~wrong], p_L[~wrong], R=R_PIX), ~wrong)
        same_state(a, b)
    assert_measured("lmk", name, worst)


# ---- (g) one device batch of 40 members -----------------------------------------------------------------------------------
BATCH_H = (1, 7, 8, 9, 64, 256, 1023, 1024)


def batch_member(rng, i, poses, M):
    """member i's spec: exact or uncertain map, consensus or none, single or iterated, H from BATCH_H; member 17 has no
    observations"""
    if i == 17:
        return None
    spec = {"R": R_PIX, "max_iter": 8 if i % 4 == 3 else 0, "tol": 0.0,
            "consensus": None if i % 5 == 0 else cons(BATCH_H[i % 8], seed=i, min_inliers=2 + i % 3)}
    if i % 3 == 1:  # uncertain map: one-clone landmarks, a 2-clone and a 3-clone set, one landmark swapped, one match pushed
        sets = {(1,): 4, (M - 1,): 3, (0, M - 1): 3, (1, 2, M - 2): 2}
        clone, z, p_L, lm, Sig, _ = ref.planted_map(rng, poses, sets, correction(0.3), swap=[2], push=[(7, 0)], noise=QUIET)
        spec.update(landmark=lm, Sigma_L=Sig)
    else:
        counts = {int(k): int(rng.integers(2, 12)) for k in rng.choice(M, size=min(M, 1 + i % 5), replace=False)}
        clone, z, p_L, _ = ref.planted(rng, poses, counts, correction(0.3), 0.3)
    spec.update(clone=clone, z=z, p_L=p_L)
    return spec


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_of_40_equals_single_calls(dtype):
    rng = np.random.default_rng(109)
    assert ss.chunks(ss.CONS_BATCH, ss.K["kBatchMembers"]) == 2
    Ms = [(5, 12, 40, 91)[i % 4] for i in range(ss.CONS_BATCH)]
    mem = [fresh(dtype, M) for M in Ms]
    twins = [fresh(dtype, M) for M in Ms]
    specs = [batch_member(rng, i, state_of(m.e)[1], M) for i, (m, M) in enumerate(zip(mem, Ms))]
    hs = [s["consensus"]["hypotheses"] for s in specs if s is not None and s["consensus"] is not None]
    assert min(hs) == 1 and max(hs) == 1024
    single = [None if s is None else t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], max_iter=s["max_iter"], tol=s["tol"],
                                                         landmark=s.get("landmark"), Sigma_L=s.get("Sigma_L"),
                                                         consensus=s["consensus"] or cons(0))
              for t, s in zip(twins, specs)]
    before = snapshot(mem[17].e)
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    assert got[17] is None
    assert_unchanged(snapshot(mem[17].e), before)
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            continue
        for key in KEYS:
            assert got[i][key] == single[i][key] or (np.isnan(got[i][key]) and np.isnan(single[i][key])), (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"], equal_nan=True) and np.array_equal(got[i]["flag"], single[i]["flag"])
        cg, cs = got[i]["consensus"], single[i]["consensus"]
        for key in ("status", "inliers", "best", "valid", "refit", "yaw"):
            assert cg[key] == cs[key], (i, key)
        assert np.array_equal(cg["t"], cs["t"]) and np.array_equal(cg["pivot"], cs["pivot"])
        assert (cg["scores"] is None) == (cs["scores"] is None)
        if cg["scores"] is not None:
            assert np.array_equal(cg["scores"], cs["scores"]), i
        same_state(m, t)
