"""The consensus on mapped-landmark matches without a GPU: the numpy reference of tests/landmark_consensus_reference.py on its
own (a planted correction recovered with 0 / 30 / 60 % wrong matches, a minimal fit that reproduces its two observations, the
sampler's golden pairs), the argument checks of the Python surface, and the runner's outlier draw.  Then the designed cases
of tests/test_landmark_consensus_shapes_gpu.py on the reference: the multi-clone map builder passes the host's map checks
and its wrong matches are exactly what the consensus excludes, each tie layout puts the first valid hypothesis at its index,
and the degenerate pair, rejected refit and min_inliers cases take their branches."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import landmark_consensus_reference as ref, landmark_map_reference as mref, side_shapes as ss
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)

R_PIX = np.array([[4.0e-6, 5.0e-7], [5.0e-7, 3.0e-6]])
THRESH = 13.8  # chi-square, 2 dof, 0.999


def window(rng, M):
    """[M, 7] clone poses p_C_G, q_CG along a 1 m-per-clone path with random attitudes"""
    poses = np.zeros((M, 7))
    poses[:, 0:3] = np.cumsum(rng.normal(size=(M, 3)) * [1.0, 1.0, 0.1], axis=0)
    q = rng.normal(size=(M, 4))
    poses[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return poses


def test_golden_pairs():
    # splitmix64 of (seed + 2h, seed + 2h + 1), mapped to i != j; fixed values keep the generator (and DESIGN.md 4.17) honest
    assert ref.splitmix64(0) == 0xE220A8397B1DCDAF
    assert ref.splitmix64(1) == 0x910A2DEC89025CC1
    pairs = ref.sample_pairs(12345, 6, 100)
    assert pairs.tolist() == GOLDEN_12345_100, pairs.tolist()
    assert ref.sample_pairs(7, 3, 2).tolist() == [[i, 1 - i] for i, _ in ref.sample_pairs(7, 3, 2).tolist()]
    assert ref.sample_pairs(1, 4, 1) is None
    big = ref.sample_pairs(2 ** 64 - 3, 1024, 4096)  # seed + 2h wraps mod 2^64
    assert np.all(big[:, 0] != big[:, 1]) and big.min() >= 0 and big.max() < 4096


GOLDEN_12345_100 = [[44, 40], [53, 28], [19, 80], [85, 20], [76, 60], [76, 62]]  # seed 12345, 100 observations


@pytest.mark.parametrize("rate", [0.0, 0.3, 0.6])
def test_recovers_a_planted_correction(rate):
    rng = np.random.default_rng(int(rate * 10) + 3)
    poses = window(rng, 12)
    th = np.array([0.04, 0.9, -0.6, 0.2])
    clone, z, p_L, wrong = ref.planted(rng, poses, {0: 40, 5: 40, 11: 40}, th, rate)
    out = ref.consensus(poses, clone, z, p_L, R_PIX, 256, THRESH, 8, seed=99)
    assert out["status"] == 0 and out["best"] >= 0
    assert np.abs(out["th_final"] - th).max() < 2e-2, out["th_final"]
    # every wrong match is excluded, nearly every right one kept
    assert not np.any(out["inliers"] & wrong)
    assert out["inliers"][~wrong].mean() > 0.97
    assert np.array_equal(out["pre"], np.where(out["inliers"], 0, 3))
    assert out["valid"].sum() >= 1 and out["scores"][out["best"]] == out["scores"].max()


def test_minimal_fit_reproduces_its_pair():
    rng = np.random.default_rng(5)
    poses = window(rng, 6)
    clone, z, p_L, _ = ref.planted(rng, poses, {1: 3, 4: 3}, [-0.1, 0.5, 0.3, -0.2], 0.0, noise=0.003)
    W = ref.weight(R_PIX)
    c = ref.pivot(poses, clone)
    for i, j in [(0, 1), (2, 5), (3, 4)]:
        sel = [i, j]
        th, ok = ref.gauss_newton(np.zeros(4), c, poses, clone[sel], z[sel], p_L[sel], W)
        assert ok
        front, r, e = ref.model(th, c, poses, clone[sel], z[sel], p_L[sel], W)
        assert front.all() and np.abs(r).max() < 1e-10, r


def test_a_degenerate_pair_is_not_valid():
    rng = np.random.default_rng(8)
    poses = window(rng, 3)
    clone, z, p_L, _ = ref.planted(rng, poses, {0: 2}, [0.0, 0.0, 0.0, 0.0], 0.0)
    p_L[1], z[1] = p_L[0], z[0]  # one point twice: rank 2 of 4
    out = ref.consensus(poses, clone, z, p_L, R_PIX, 4, THRESH, 2, seed=1)
    assert not out["valid"].any() and out["best"] == -1 and out["status"] == 1 and np.all(out["pre"] == 3)


def test_final_flags_precedence():
    assert ref.final_flags([3, 3, 0, 0, 3], [2, 1, 1, 0, 0]).tolist() == [2, 3, 1, 0, 3]


def test_consensus_struct():
    s, keep = capi.consensus_struct({"hypotheses": 64, "thresh": 9.0, "min_inliers": 5, "seed": 2 ** 64 - 1})
    assert (s.hypotheses, s.thresh, s.min_inliers, s.seed) == (64, 9.0, 5, 2 ** 64 - 1)
    assert len(keep[0]) == 64
    s, keep = capi.consensus_struct(None)
    assert s.hypotheses == 0 and keep == ()


# ---- the class and the C view over a fake C-ABI (tests/stub/stub_landmark_consensus.cpp) -------------------------------------


def _calls(f):
    import ctypes as C
    out = (C.c_longlong * 3)()
    f.lib.msckf_b200_stub_consensus_calls(C.c_void_p(f.engineHandle()), out)
    return list(out)


def _last(f):
    import ctypes as C
    cl, c3 = (C.c_int * 64)(), (C.c_ulonglong * 3)()
    n = f.lib.msckf_b200_stub_consensus_last(C.c_void_p(f.engineHandle()), cl, 64, c3)
    return list(cl[:n]), list(c3)


BAD = [{"hypotheses": 1025, "thresh": 9.0, "min_inliers": 2}, {"hypotheses": 8, "thresh": 0.0, "min_inliers": 2},
       {"hypotheses": 8, "thresh": float("nan"), "min_inliers": 2}, {"hypotheses": 8, "thresh": float("inf"), "min_inliers": 2},
       {"hypotheses": 8, "thresh": 9.0, "min_inliers": 1}]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_class_maps_ids_and_forwards_the_consensus(stub_view, dtype):
    from tests.test_landmark_cpu import _filters
    (f,), wl = _filters(stub_view, 1, dtype, frames=4)
    z, p = np.tile([0.01, -0.02], (4, 1)), np.tile([1.0, 2.0, 5.0], (4, 1))
    ids = [wl["frames"][k]["state_id"] for k in (2, 0, 2, 1)]
    cb = _calls(f)
    r = f.landmark_update(ids, z, p, consensus={"hypotheses": 64, "thresh": 9.0, "min_inliers": 3, "seed": 2 ** 63 + 5})
    assert list(r["flag"]) == [0, 3, 0, 3] and r["used"] == 2
    c = r["consensus"]
    assert c["best"] == 0 and c["inliers"] == 2 and c["valid"] == 64 and np.all(c["scores"] == 2)
    c0 = _calls(f)
    assert c0[0] - cb[0] == 1 and c0[1] == cb[1]
    assert _last(f) == ([2, 0, 2, 1], [64, 3, 2 ** 63 + 5])
    for (w, a, dT) in wl["frames"][3]["imu"][:3]:  # queued IMU readings are handed over first
        f.propagate(w, a, dT)
    f.landmark_update(ids[:1], z[:1], p[:1], consensus={"hypotheses": 1, "thresh": 9.0, "min_inliers": 2})
    c1 = _calls(f)
    assert c1[0] - c0[0] == 1 and c1[2] - c0[2] == 3
    for bad in BAD:  # refused before any C-ABI call
        with pytest.raises(RuntimeError, match="hypotheses|thresh|min_inliers"):
            f.landmark_update(ids, z, p, consensus=bad)
    with pytest.raises(RuntimeError, match="not in the window"):
        f.landmark_update([999], z[:1], p[:1], consensus={"hypotheses": 4, "thresh": 9.0, "min_inliers": 2})
    assert _calls(f) == c1
    f.close()


def test_batch_makes_one_call(stub_view):
    from msckf_mono_b200.cview import FilterBatch
    from tests.test_landmark_cpu import _filters
    fs, wl = _filters(stub_view, 3, np.float64, frames=4)
    fb = FilterBatch(fs)
    z, p = np.tile([0.01, -0.02], (3, 1)), np.tile([1.0, 2.0, 5.0], (3, 1))
    sid = [fr["state_id"] for fr in wl["frames"][:3]]
    cb = [_calls(f)[:2] for f in fs]
    cons = [{"hypotheses": 16, "thresh": 9.0, "min_inliers": 2, "seed": 1}, None, {"hypotheses": 0}]
    res = fb.landmark_update([([sid[1], sid[0], sid[2]], z, p), None, ([sid[2]], z[:1], p[:1])], consensus=cons)
    assert res[1] is None and list(res[0]["flag"]) == [0, 3, 0] and list(res[2]["flag"]) == [0]
    assert res[0]["consensus"]["best"] == 0 and res[2]["consensus"]["best"] == -1
    assert [[a - b for a, b in zip(_calls(f)[:2], c)] for f, c in zip(fs, cb)] == [[0, 1], [0, 0], [0, 1]]
    assert _last(fs[0]) == ([1, 0, 2], [16, 2, 1])
    for bad in BAD:
        with pytest.raises(RuntimeError, match="hypotheses|thresh|min_inliers"):
            fb.landmark_update([([sid[0]], z[:1], p[:1]), None, None], consensus=[bad, None, None])
    assert [[a - b for a, b in zip(_calls(f)[:2], c)] for f, c in zip(fs, cb)] == [[0, 1], [0, 0], [0, 1]]
    fb.close()
    for f in fs:
        f.close()


def test_runner_draws_nothing_new_without_wrong_matches():
    """with map_outlier_rate = 0 the runner makes no draw from the wrong-match stream [seed, k, 12], so every trial input is the
    one make_trial gives; map rows carry the wrong / kept counts only when wrong matches or a consensus are on"""
    import inspect
    from msckf_mono_b200 import montecarlo as mc
    sig = inspect.signature(mc.run).parameters
    assert sig["map_outlier_rate"].default == 0.0 and sig["map_consensus"].default == 0 and sig["map_chi2"].default == 0.0
    src = inspect.getsource(mc.run)
    assert "[seed, tr[\"k\"], 12]) if map_outlier_rate > 0 else None" in src
    nees = [{"orientation": 3.0, "position": 3.0, "pose": 6.0, "imu": 15.0, "full": 15.0, "dim_full": 15, "first_bad_pivot": -1}] * 2
    plain = [dict(nis=2.0, dof=4, used=2, applied=1, n=2)]
    assert set(mc.trial_record(nees, [0.01] * 2, map_rows=plain)["map"]) == {"nis", "dof", "used", "applied", "n"}
    cons = [dict(plain[0], wrong=1, wrong_excluded=1, right=3, right_kept=2, cons_status=0)]
    rec = mc.trial_record(nees, [0.01] * 2, map_rows=cons)["map"]
    assert rec["wrong_excluded"] == [1] and rec["right_kept"] == [2] and rec["cons_status"] == [0]


# ---- the designed cases of tests/test_landmark_consensus_shapes_gpu.py on the reference -------------------------------------
def test_pairs_fast_is_the_sampler():
    for seed, H, n in ((12345, 6, 100), (2 ** 64 - 3, 1024, 4096), (7, 64, 2), (99, 1024, 128)):
        assert np.array_equal(ref.pairs_fast(seed, H, n), ref.sample_pairs(seed, H, n))


@pytest.mark.parametrize("shape", sorted(ss.CONS_MAP))
def test_planted_map_passes_the_host_checks_and_excludes_as_designed(shape):
    """every exclusion pattern of a CONS_MAP shape: ids, one p_L per landmark, one observation per clone, <= 8 clones, <= 256
    clone sets and the planned rows within kLmkMaxRows; the reference's consensus excludes exactly the wrong matches"""
    rng = np.random.default_rng(11)
    poses = spread_window(rng, ss.LMK_WINDOW)
    sets = ss.CONS_MAP[shape]
    for pattern in ss.CONS_MAP_PATTERNS:
        swap, move, push = ref.map_exclusions(sets, pattern)
        if swap is None:
            assert shape == "full_set" and pattern == "clone_set"
            continue
        clone, z, p_L, lm, Sig, wrong = ref.planted_map(rng, poses, ref.set_counts(sets), [0.015, 0.24, -0.15, 0.09], swap=swap,
                                                        move=move, push=push, noise=0.0005)
        ref.map_checks(clone, p_L, lm, len(Sig))
        groups = {tuple(sorted(clone[lm == l])) for l in np.unique(lm)}
        assert len([g for g in groups if len(g) > 1]) <= ss.K["kLmkMaxSets"]
        assert mref.rows(clone, lm, np.zeros(len(clone))) <= ss.K["kLmkMaxRows"]
        assert wrong.any() and (bool(move) == (shape == "sets" and pattern == "one_observation"))
        out = ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, 2, seed=len(clone))
        assert out["status"] == 0 and np.array_equal(out["pre"] == 3, wrong), (shape, pattern)


def test_planted_map_outliers_of_both_kinds():
    rng = np.random.default_rng(12)
    poses = spread_window(rng, 12)
    sets = {(0, 5): 3, (2, 7, 11): 2, (4,): 2}
    clone, z, p_L, lm, Sig, wrong = ref.planted_map(rng, poses, sets, [0.0] * 4, swap=[1], move=[(3, 2)])
    ref.map_checks(clone, p_L, lm, 7)
    assert np.all(wrong[lm == 1]) and wrong.sum() == 3  # landmark 1 (2 observations) and the moved one
    moved = np.flatnonzero(wrong & (lm != 1))[0]
    assert clone[moved] == 2 and lm[moved] != 3 and 2 not in clone[(lm == 3)]
    assert np.array_equal(p_L[moved], p_L[lm == lm[moved]][0])
    clone, z, p_L, lm, Sig, wrong = ref.planted_map(rng, poses, sets, [0.0] * 4, outlier_rate=1.0)
    assert wrong.all()
    ref.map_checks(clone, p_L, lm, 7)


@pytest.mark.parametrize("first", ss.CONS_FIRST)
def test_tie_layout_puts_the_first_valid_hypothesis_at_its_index(first):
    """the seed and degenerate set of each (c) case: the sampler's first pair free of degenerate observations is `first`,
    the reference finds exactly that, every valid hypothesis counts the same inliers, and (but for the last index) ties sit
    in other warps of k_lmk_cons"""
    H, n = ss.K["kLmkMaxHyp"], ss.CONS_TIE_OBS
    seed, deg = ref.first_valid_layout(first, H, n, min_later=0 if first == H - 1 else 8)
    pr = ref.sample_pairs(seed, H, n)
    free = ~deg[pr[:, 0]] & ~deg[pr[:, 1]]
    assert np.flatnonzero(free)[0] == first
    rng = np.random.default_rng(first)
    poses = spread_window(rng, 12)
    clone, z, p_L = ref.tied(rng, poses, {0: 32, 4: 32, 8: 32, 11: 32}, [0.015, 0.24, -0.15, 0.09], deg)
    out = ref.consensus(poses, clone, z, p_L, R_PIX, H, ref.TIE_THRESH, 2, seed=seed)
    valid = np.flatnonzero(out["valid"])
    # (a pair free of them may still fail its fit, e.g. a Gauss-Newton that leaves the front: rare)
    assert np.all(free[valid]) and (free & ~out["valid"]).sum() <= 0.01 * free.sum()
    assert out["valid"][first] and out["best"] == first and out["refit"] == 1
    assert np.all(out["scores"][valid] == (~deg).sum())
    if first < H - 1:
        assert len({(h % ss.K["kLmkThreads"]) // 32 for h in valid}) > 1


def test_refit_rejected_search_reaches_the_branch():
    rng = np.random.default_rng(13)
    poses = spread_window(rng, 12)
    clone, z, p_L, seed, rf = ref.refit_rejected(rng, poses, R_PIX, 6.0)
    assert rf["refit"] == 0 and rf["best"] >= 0 and np.isfinite(rf["e_refit"]).any()
    assert (rf["e_refit"] <= 6.0).sum() < (rf["e_best"] <= 6.0).sum() and rf["inliers"].sum() == (rf["e_best"] <= 6.0).sum()
    assert np.array_equal(rf["th_final"], rf["th"][rf["best"]])


def test_identical_pair_fails_the_cholesky_and_min_inliers_edges():
    rng = np.random.default_rng(14)
    poses = spread_window(rng, 12)
    clone, z, p_L, _ = ref.planted(rng, poses, {2: 10, 9: 10}, [0.015, 0.24, -0.15, 0.09], 0.0)
    clone[1], z[1], p_L[1] = clone[0], z[0], p_L[0]
    out = ref.consensus(poses, clone, z, p_L, R_PIX, 1024, THRESH, 2, seed=11)
    hs = [h for h, p in enumerate(out["pairs"].tolist()) if sorted(p) == [0, 1]]
    assert hs and not out["valid"][hs].any() and out["valid"].sum() > 900
    W, c = ref.weight(R_PIX), ref.pivot(poses, clone)
    assert ref.model(np.zeros(4), c, poses, clone[:2], z[:2], p_L[:2], W)[0].all()  # in front: the Cholesky fails the fit
    assert not ref.gauss_newton(np.zeros(4), c, poses, clone[:2], z[:2], p_L[:2], W)[1]
    for copies in (2, 5):
        o = ref.consensus(poses, np.repeat(clone[:1], copies), np.repeat(z[:1], copies, 0), np.repeat(p_L[:1], copies, 0), R_PIX, 16,
                          THRESH, 2, seed=7)
        assert not o["valid"].any() and o["status"] == 1 and np.all(o["pre"] == 3)
    clone, z, p_L, wrong = ref.planted(rng, poses, {0: 15, 6: 15, 11: 15}, [0.015, 0.24, -0.15, 0.09], 0.3, noise=0.0005)
    k = int(ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, 2, seed=3)["inliers"].sum())
    assert k == (~wrong).sum()
    assert ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, k, seed=3)["status"] == 0
    assert ref.consensus(poses, clone, z, p_L, R_PIX, 64, THRESH, k + 1, seed=3)["status"] == 1


def test_excluded_rows_cases_cross_the_planned_stride():
    K = ss.K
    for rows in ss.CONS_SWEEP_ROWS:
        right, wrong = ss.cons_sweep(ss.LMK_WINDOW, rows)
        allc = {k: right.get(k, 0) + wrong.get(k, 0) for k in set(right) | set(wrong)}
        used, planned = ss.lmk_rows(right), ss.lmk_rows(allc)
        assert planned <= K["kLmkMaxRows"] and sum(allc.values()) <= K["kLmkMaxObs"]
        assert (used, planned) == ((rows, rows + 2) if rows < K["kLmkMaxRows"] else (rows - 2, rows))
    for counts in ss.CONS_GATE:
        mid = sorted(counts)[len(counts) // 2]
        used = ss.lmk_rows({k: a for k, a in counts.items() if k != mid})
        assert ss.chunks(ss.lmk_rows(counts)) > ss.chunks(used)


def spread_window(rng, M):
    """window() with the clones' attitudes near one another, as a filter's window is: every landmark of a clone set is seen
    from each of its clones"""
    poses = window(rng, M)
    q0 = poses[0, 3:7]
    q = q0 + 0.05 * rng.normal(size=(M, 4))
    poses[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return poses
