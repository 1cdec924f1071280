"""The consensus on mapped-landmark matches on the device (msckf_b200_landmark_update_consensus / _batch_...) against the numpy
reference of tests/landmark_consensus_reference.py: each hypothesis's validity and inlier count, the chosen hypothesis and the
final flags at windows of 1-90 clones, 2-4096 observations (256 on one clone), 1-1024 hypotheses and drifts of 0.05 / 0.3 / 1 m.
A count or flag may differ from the reference only through observations whose e_i lies within 1e-9 relative of thresh.
Then: with an exact map the call is bit for bit the plain call without the excluded observations (single and iterated); with
Sigma_L it agrees to 1e-12; a failed consensus writes nothing; a batch of 33 mixed members equals single calls bit for bit; and
hypotheses = 0 is the plain call bit for bit."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import landmark_consensus_reference as ref
from tests.test_aid_gpu import assert_unchanged, snapshot
from tests.test_batch_stream_gpu import Member
from tests.test_landmark_gpu import state_of

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
R_PIX = np.array([[4.0e-6, 5.0e-7], [5.0e-7, 3.0e-6]])
THRESH = 13.8
KEYS = ("nis", "dx_norm", "dof", "rows", "used", "applied", "status", "iterations", "converged", "step")
# (clones, {clone: observations}, hypotheses)
SHAPES = [(1, {0: 2}, 1), (3, {0: 6, 2: 5}, 16), (12, {4: 256}, 64), (40, {0: 30, 13: 30, 27: 30, 39: 30}, 256),
          (90, {k: 256 for k in range(0, 90, 6)} | {89: 256}, 1024)]
DRIFTS = (0.05, 0.3, 1.0)


def correction(drift):
    return np.array([drift / 20, 0.8 * drift, -0.5 * drift, 0.3 * drift])


def near(e, thresh=THRESH):
    """observations whose e_i is within 1e-9 relative of thresh (their side of it may differ by rounding)"""
    return np.isfinite(e) & (np.abs(e - thresh) <= 1e-9 * thresh)


def cons(h, seed=7, min_inliers=2, thresh=THRESH):
    return {"hypotheses": h, "thresh": thresh, "min_inliers": min_inliers, "seed": seed}


def check_against_reference(res, rf, flag_plain):
    """res: the consensus call; rf: the reference's consensus; flag_plain: the flags of the plain call on the same input and
    filter (its 2 / 1 / 0).  The device's final flags must be final_flags(rf["pre"], flag_plain) outside the near-threshold set."""
    c = res["consensus"]
    H = len(rf["scores"])
    dev = c["scores"]
    for h in range(H):
        if dev[h] == rf["scores"][h]:
            continue
        amb = int(near(rf["e"][h]).sum())
        assert amb > 0 and (dev[h] < 0) == (rf["scores"][h] < 0) and abs(int(dev[h]) - int(rf["scores"][h])) <= amb, \
            (h, dev[h], rf["scores"][h], amb)
    assert c["valid"] == int(rf["valid"].sum())
    if c["best"] != rf["best"]:  # only a near-threshold observation can move the arg-max
        assert any(near(rf["e"][h]).any() for h in (c["best"], rf["best"])), (c["best"], rf["best"])
        return
    if rf["best"] < 0:
        assert c["status"] == 1 and np.all(res["flag"][res["flag"] != 2] == 3)
        return
    amb = near(rf["e_best"]) | near(rf["e_refit"])
    assert c["refit"] == rf["refit"] or amb.any()
    assert c["status"] == rf["status"]
    assert abs(c["inliers"] - int(rf["inliers"].sum())) <= int(amb.sum()), (c["inliers"], int(rf["inliers"].sum()))
    if not amb.any():
        assert c["inliers"] == int(rf["inliers"].sum())
    expect = ref.final_flags(rf["pre"], flag_plain)
    assert np.array_equal(res["flag"][~amb], expect[~amb]), np.flatnonzero(res["flag"] != expect)
    # kept (0) exactly where the reference keeps a match the plain call uses, excluded (3) where it excludes one not behind
    assert np.all(res["flag"][~amb & (rf["pre"] == 0) & (flag_plain == 0)] == 0)
    assert np.all(res["flag"][~amb & (rf["pre"] == 3) & (flag_plain != 2)] == 3)
    assert np.allclose(c["pivot"], rf["pivot"], rtol=1e-12, atol=1e-12)
    if c["refit"] == rf["refit"]:
        assert np.allclose([c["yaw"], *c["t"]], rf["th_final"], rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_the_reference(dtype):
    rng = np.random.default_rng(21)
    for si, (M, counts, H) in enumerate(SHAPES):
        base = Member(dtype, M, seed=50 + si, max_clones=M + 2)
        for drift in (DRIFTS if H < 1024 else (0.3,)):
            mem, twin = base.twin(dtype, max_clones=M + 2), base.twin(dtype, max_clones=M + 2)
            _, poses = state_of(mem.e)
            n = sum(counts.values())
            clone, z, p_L, wrong = ref.planted(rng, poses, counts, correction(drift), 0.3 if n > 2 else 0.0)
            min_inl = max(2, n // 2)  # above the wrong matches' share: a consensus that keeps too few fails
            res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, consensus=cons(H, seed=si + 100, min_inliers=min_inl))
            plain = twin.e.landmark_update(clone, z, p_L, R=R_PIX)
            rf = ref.consensus(poses, clone, z, p_L, R_PIX, H, THRESH, min_inl, seed=si + 100)
            check_against_reference(res, rf, plain["flag"])
            if res["consensus"]["status"] == 0 and n >= 20:
                assert not np.any((res["flag"] == 0) & wrong), (M, drift)


def _drop(clone, z, p_L, keep):
    return clone[keep], z[keep], p_L[keep]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("max_iter", [0, 8])
def test_exact_map_is_the_plain_call_without_the_excluded(dtype, max_iter):
    rng = np.random.default_rng(31 + max_iter)
    for M in (3, 30, 90):
        base = Member(dtype, M, seed=M, max_clones=M + 2)
        _, poses = state_of(base.e)
        counts = {0: 12, M // 2: 12, M - 1: 12}
        clone, z, p_L, wrong = ref.planted(rng, poses, counts, correction(0.3), 0.3)
        a, b = base.twin(dtype, max_clones=M + 2), base.twin(dtype, max_clones=M + 2)
        n0 = a.e.launch_count()
        got = a.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=40.0, max_iter=max_iter, tol=1e-10, consensus=cons(128))
        assert a.e.launch_count() == n0
        assert got["consensus"]["status"] == 0
        keep = got["flag"] != 3
        rf = ref.consensus(poses, clone, z, p_L, R_PIX, 128, THRESH, 2, seed=7)
        amb = near(rf["e_best"]) | near(rf["e_refit"])
        assert np.array_equal(keep[~amb], (rf["pre"] == 0)[~amb])  # the reference's kept set, not the device's own
        assert not np.any(keep & wrong) and keep.sum() < len(clone) and keep[~wrong].mean() > 0.9
        plain = b.e.landmark_update(*_drop(clone, z, p_L, keep), R=R_PIX, chi2_obs=40.0, max_iter=max_iter, tol=1e-10)
        for k in KEYS:
            assert got[k] == plain[k], (M, k, got[k], plain[k])
        assert got["applied"] == 1
        assert np.array_equal(got["gamma"][keep], plain["gamma"]) and np.array_equal(got["flag"][keep], plain["flag"])
        for x, y in zip(a.snapshot(), b.snapshot()):
            assert np.array_equal(x, y), M


@pytest.mark.parametrize("max_iter", [0, 8])
def test_uncertain_map_agrees_with_the_plain_call_without_the_excluded(max_iter):
    rng = np.random.default_rng(41 + max_iter)
    M = 20
    base = Member(np.float64, M, seed=4, max_clones=M + 2)
    _, poses = state_of(base.e)
    clone, z, p_L, wrong = ref.planted(rng, poses, {2: 15, 9: 15, 19: 15}, correction(0.3), 0.3)
    n = len(clone)
    Sig = np.tile(np.diag([4e-4, 4e-4, 9e-4]), (n, 1, 1))
    a, b = base.twin(np.float64, max_clones=M + 2), base.twin(np.float64, max_clones=M + 2)
    got = a.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=max_iter, tol=1e-10, landmark=np.arange(n), Sigma_L=Sig,
                              consensus=cons(128))
    keep = got["flag"] != 3
    assert got["consensus"]["status"] == 0 and not np.any(keep & wrong)
    plain = b.e.landmark_update(*_drop(clone, z, p_L, keep), R=R_PIX, max_iter=max_iter, tol=1e-10,
                                landmark=np.arange(keep.sum()), Sigma_L=Sig[keep])
    for k in ("dof", "rows", "used", "applied", "status", "iterations"):
        assert got[k] == plain[k], k
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.abs(x - y).max() <= 1e-12 * max(np.abs(y).max(), 1.0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_failed_consensus_writes_nothing(dtype):
    rng = np.random.default_rng(51)
    m = Member(dtype, 10, seed=3, max_clones=12)
    _, poses = state_of(m.e)
    clone, z, p_L, _ = ref.planted(rng, poses, {1: 10, 8: 10}, correction(0.3), 0.3)
    before, n0 = snapshot(m.e), m.e.launch_count()
    for c in (cons(64, min_inliers=len(clone) + 1), cons(64, thresh=1e-30, min_inliers=3)):
        r = m.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=4, consensus=c)
        assert r["consensus"]["status"] == 1 and r["applied"] == 0 and r["used"] == 0
        assert np.all(r["flag"] == 3)
        assert_unchanged(snapshot(m.e), before)
        assert m.e.launch_count() == n0
    r = m.e.landmark_update(clone[:1], z[:1], p_L[:1], R=R_PIX, consensus=cons(8))  # one observation: no pair
    assert r["consensus"]["status"] == 1 and r["consensus"]["valid"] == 0 and r["consensus"]["best"] == -1
    assert np.all(r["consensus"]["scores"] == -1) and r["applied"] == 0
    assert_unchanged(snapshot(m.e), before)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(61)
    mem = [Member(dtype, Ms[i % 4], seed=200 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    specs = []
    for i, m in enumerate(mem):
        M = m.e.num_clones()
        if M == 0 or i % 7 == 3:
            specs.append(None)
            continue
        _, poses = state_of(m.e)
        counts = {int(k): int(rng.integers(2, 12)) for k in rng.choice(M, size=min(M, 1 + i % 5), replace=False)}
        clone, z, p_L, _ = ref.planted(rng, poses, counts, correction(0.3), 0.3)
        specs.append({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX if i % 2 else None, "chi2_obs": 0.0 if i % 3 else 50.0,
                      "max_iter": 0 if i % 4 else 5, "tol": 1e-10,
                      "consensus": None if i % 5 == 0 else cons((0, 1, 37, 256)[i % 4], seed=i, min_inliers=2 + i % 3)})
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], chi2_obs=s["chi2_obs"],
                                                         max_iter=s["max_iter"], tol=s["tol"], consensus=s["consensus"] or cons(0))
              for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs, consensus=cons(0))
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        for key in KEYS:
            assert got[i][key] == single[i][key] or (np.isnan(got[i][key]) and np.isnan(single[i][key])), (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"], equal_nan=True)
        assert np.array_equal(got[i]["flag"], single[i]["flag"])
        cg, cs = got[i]["consensus"], single[i]["consensus"]
        for key in ("status", "inliers", "best", "valid", "refit", "yaw"):
            assert cg[key] == cs[key], (i, key)
        assert np.array_equal(cg["t"], cs["t"]) and np.array_equal(cg["pivot"], cs["pivot"])
        assert (cg["scores"] is None) == (cs["scores"] is None)
        if cg["scores"] is not None:
            assert np.array_equal(cg["scores"], cs["scores"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


@pytest.mark.parametrize("dtype", DTYPES)
def test_no_hypotheses_is_the_plain_call(dtype):
    rng = np.random.default_rng(71)
    base = Member(dtype, 12, seed=9, max_clones=14)
    _, poses = state_of(base.e)
    clone, z, p_L, _ = ref.planted(rng, poses, {0: 8, 11: 8}, correction(0.3), 0.3)
    for mi in (0, 6):
        a, b = base.twin(dtype, max_clones=14), base.twin(dtype, max_clones=14)
        r1 = a.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=20.0, max_iter=mi, tol=1e-10, consensus=cons(0))
        r2 = b.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=20.0, max_iter=mi, tol=1e-10)
        for k in KEYS:
            assert r1[k] == r2[k], k
        assert np.array_equal(r1["flag"], r2["flag"]) and np.array_equal(r1["gamma"], r2["gamma"])
        assert r1["consensus"]["best"] == -1 and r1["consensus"]["status"] == 0
        for x, y in zip(a.snapshot(), b.snapshot()):
            assert np.array_equal(x, y)


def test_arguments_refused_before_any_launch():
    rng = np.random.default_rng(81)
    m = Member(np.float64, 4, seed=1)
    _, poses = state_of(m.e)
    clone, z, p_L, _ = ref.planted(rng, poses, {0: 4, 3: 4}, correction(0.3), 0.0)
    before = snapshot(m.e)
    for c in ({"hypotheses": 1025, "thresh": 9.0, "min_inliers": 2}, {"hypotheses": -1, "thresh": 9.0, "min_inliers": 2},
              {"hypotheses": 8, "thresh": 0.0, "min_inliers": 2}, {"hypotheses": 8, "thresh": float("nan"), "min_inliers": 2},
              {"hypotheses": 8, "thresh": float("inf"), "min_inliers": 2}, {"hypotheses": 8, "thresh": 9.0, "min_inliers": 1}):
        a, keep = capi.landmark_struct({"clone": clone, "z": z, "p_L": p_L})
        s = capi.LandmarkConsensus(c["hypotheses"], c["thresh"], c["min_inliers"], 0, None)
        out, cout = capi.LandmarkResult(), capi.LandmarkConsensusResult()
        rc = capi.lib().msckf_b200_landmark_update_consensus(m.e.h, C.byref(a), None, C.byref(s), C.byref(out), C.byref(cout))
        assert rc == -3, c
    assert_unchanged(snapshot(m.e), before)


def test_batch_edge_cases_match_the_single_call():
    """a consensus member without observations gets scores -1 and status 1 as the single call gives, and cons NULL leaves every
    cons_out at best = -1 and zeros, as the single call does"""
    rng = np.random.default_rng(91)
    mem = [Member(np.float64, 6, seed=60 + i, max_clones=8) for i in range(2)]
    _, poses = state_of(mem[1].e)
    clone, z, p_L, _ = ref.planted(rng, poses, {0: 6, 5: 6}, correction(0.3), 0.0)
    a0, _ = capi.landmark_struct(None)
    a1, keep = capi.landmark_struct({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX})
    lm = (capi.Landmarks * 2)(a0, a1)
    scores = np.full(4, 7, dtype=np.int32)
    cs = (capi.LandmarkConsensus * 2)(capi.LandmarkConsensus(4, THRESH, 2, 1, scores.ctypes.data), capi.LandmarkConsensus(0, 0.0, 0, 0, None))
    out, cout = (capi.LandmarkResult * 2)(), (capi.LandmarkConsensusResult * 2)()
    for c in cout:
        c.best, c.status = 5, 5
    b = capi.Batch([m.e for m in mem])
    try:
        assert capi.lib().msckf_b200_batch_landmark_update_consensus(b.h, lm, None, cs, out, cout) == 0
        assert np.all(scores == -1) and (cout[0].status, cout[0].best, cout[0].valid) == (1, -1, 0)
        assert (cout[1].status, cout[1].best, cout[1].inliers) == (0, -1, 0)
        for c in cout:
            c.best, c.status = 5, 5
        assert capi.lib().msckf_b200_batch_landmark_update_consensus(b.h, lm, None, None, out, cout) == 0
        assert [(c.status, c.best, c.inliers, c.yaw) for c in cout] == [(0, -1, 0, 0.0)] * 2
    finally:
        b.close()
    single = capi.LandmarkConsensusResult()
    s1 = np.full(4, 7, dtype=np.int32)
    c1 = capi.LandmarkConsensus(4, THRESH, 2, 1, s1.ctypes.data)
    e0, _ = capi.landmark_struct(None)
    o1 = capi.LandmarkResult()
    assert capi.lib().msckf_b200_landmark_update_consensus(mem[0].e.h, C.byref(e0), None, C.byref(c1), C.byref(o1), C.byref(single)) == 0
    assert np.all(s1 == -1) and (single.status, single.best, single.valid) == (1, -1, 0)
