"""The numpy FDE over a stack's items (tests/aid_fde_reference.py), without a device: the block w-test against the NIS
difference, and the outcomes the rounds of msckf_b200_aid_stack_update_fde reach on range stacks with and without NLOS faults;
capi.fde_thresholds / fde_struct; and what the class and C view forms send to the C-ABI, through the recording fake of
tests/fake_engine.py."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests import aid_fde_reference as ref
from tests.fake_engine import recorded, stub_view  # noqa: F401 (stub_view: the fixture)
from tests.test_shim_bookkeeping_cpu import shim_filter

CHI2 = capi.fde_thresholds(0.01)


def _state(rng, M=3):
    imu = np.zeros(19)
    imu[0:3] = [1.0, 2.0, 1.5]
    imu[3:6] = [0.5, -0.2, 0.1]
    q = rng.normal(size=4)
    imu[15:19] = q / np.linalg.norm(q)
    poses = np.zeros((M, 7))
    for k in range(M):
        poses[k, 0:3] = imu[0:3] + 0.1 * rng.normal(size=3)
        qk = rng.normal(size=4)
        poses[k, 3:7] = qk / np.linalg.norm(qk)
    n = 15 + 6 * M
    G = rng.normal(size=(n, n)) * 0.02
    P = np.diag(np.full(n, 0.01)) + G @ G.T
    return imu, poses, P


def test_thresholds_are_upper_quantiles():
    from scipy.stats import chi2
    assert len(CHI2) == 32 and all(np.isfinite(CHI2))
    assert abs(CHI2[0] - 6.6348966) < 1e-6 and abs(CHI2[3] - 13.2767041) < 1e-6
    assert np.allclose([chi2.sf(c, d) for d, c in enumerate(CHI2, 1)], 0.01, rtol=1e-9, atol=0)
    f = capi.fde_struct({"chi2": CHI2, "max_exclude": 2})
    assert list(f.chi2) == CHI2 and f.max_exclude == 2


def test_exclusion_statistic_is_the_nis_difference():
    rng = np.random.default_rng(5)
    imu, poses, P = _state(rng)
    worst = 0.0
    for trial in range(20):
        items = ref.range_scene(rng, imu, poses, faults=(trial % 4,), gnss=True, jump=float(trial % 3), odometry=trial % 2 == 0,
                                clone=trial % 3)
        lin = ref.linearise(items, imu, poses, P.shape[0])
        from scipy.linalg import block_diag
        H = np.vstack([h for h, _ in lin])
        r = np.concatenate([v for _, v in lin])
        S = H @ P @ H.T + block_diag(*[it["R"] for it in items])
        first = np.cumsum([0] + [len(v) for _, v in lin])
        blocks = [np.arange(first[i], first[i + 1]) for i in range(len(items))]
        t = ref.exclusion_tests(S, r, blocks)
        full = ref.set_nis(S, r, np.arange(first[-1]))
        for j, tj in enumerate(t):
            rest = np.concatenate([b for i, b in enumerate(blocks) if i != j])
            diff = full - ref.set_nis(S, r, rest)
            worst = max(worst, abs(tj - diff) / max(abs(diff), 1.0))
    assert worst <= 1e-10, worst


def test_outcomes():
    rng = np.random.default_rng(11)
    imu, poses, P = _state(rng)
    # no fault: passed at once
    for _ in range(10):
        got = ref.fde(ref.range_scene(rng, imu, poses), imu, poses, P, CHI2, 2)
        assert got["outcome"] == 0 and got["excluded"] == [] and np.all(np.isnan(got["tests"]))
    # one range 2 m long among four 0.1 m ranges: that range, and only it, is excluded in round 0
    for k in range(4):
        items = ref.range_scene(rng, imu, poses, faults=(k,))
        got = ref.fde(items, imu, poses, P, CHI2, 2)
        assert got["outcome"] == 1 and got["excluded"] == [(k, 0)] and got["kept"] == [i for i in range(4) if i != k]
        assert got["dof"] == 3 and got["nis"] <= CHI2[2]
        assert np.argmax(got["tests"]) == k and got["tests"][k] > CHI2[0]
    # two faults and max_exclude = 1: rejected at max_exclude; max_exclude = 0: the stack gate alone
    items = ref.range_scene(rng, imu, poses, n_ranges=6, faults=(1, 4))
    got = ref.fde(items, imu, poses, P, CHI2, 1)
    assert got["outcome"] == 2 and len(got["excluded"]) == 1
    assert ref.fde(items, imu, poses, P, CHI2, 0)["outcome"] == 2
    assert ref.fde(items, imu, poses, P, CHI2, 2)["outcome"] == 1
    # a failing one-item stack is not identifiable
    got = ref.fde(ref.range_scene(rng, imu, poses, n_ranges=1, faults=(0,)), imu, poses, P, CHI2, 2)
    assert got["outcome"] == 3 and got["excluded"] == []
    # a degenerate item is dropped and does not count
    items = ref.range_scene(rng, imu, poses, faults=(2,))
    got = ref.fde(items + items[:1], imu, poses, P, CHI2, 1, dropped=(4,))
    assert got["outcome"] == 1 and got["excluded"] == [(2, 0)] and np.isnan(got["item_nis"][4])


def test_scene_is_consistent_at_the_state():
    rng = np.random.default_rng(2)
    imu, poses, _ = _state(rng)
    items = ref.range_scene(rng, imu, poses, sigma=0.0, gnss=True, odometry=True, clone=1)
    items[4]["z"][0:3] = mc.antenna_position(imu[0:3], imu[15:19], items[4]["z"][3:6])
    items[5]["z"] = mc.body_velocity(imu)
    for it in items:
        assert np.abs(mc.odometry_residual(it, imu, poses)).max() <= 1e-12


# ---- the class and C view forms over the recording fake of the C-ABI --------------------------------------------------------
def _filters(lib, n, dtype, frames=4):
    wl = synth.make_stream_workload(n_frames=frames + 1, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:frames]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_views_pass_fde_and_items_through_unchanged(stub_view, dtype):
    """MSCKF::aidedUpdate(items, fde) and MSCKFBatch::aidedUpdate(items, fde) through the C view hand the thresholds, max_exclude
    and every item to the C-ABI exactly as given and leave unnamed members alone; a thresholds table or max_exclude the C-ABI
    would refuse throws std::invalid_argument in the class before any call"""
    fs = _filters(stub_view, 3, dtype)
    rng = np.random.default_rng(8)
    stack = [{"model": capi.AID_RANGE, "z": rng.normal(size=7), "R": np.array([[0.01]])},
             {"model": capi.AID_CLONE_PLANE_RANGE, "a": 2, "z": rng.normal(size=8), "R": np.array([[0.03]])},
             {"model": capi.AID_BODY_VELOCITY, "a": 0b110, "z": rng.normal(size=3), "R": np.eye(2)},
             {"model": capi.AID_ANTENNA_POSITION, "a": 7, "z": rng.normal(size=6), "R": np.diag([0.1, 0.2, 0.3])},
             {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": 3, "b": 7, "z": rng.normal(size=6), "R": 0.01 * np.eye(3)}]
    fde = {"chi2": [float(x) for x in 1.0 + rng.random(32)], "max_exclude": 3}

    def check(f, items, fde):
        _, _, (chi2, K), got = recorded(f)
        assert chi2 == fde["chi2"] and K == fde["max_exclude"]
        assert len(got) == len(items)
        for g, it in zip(got, items):
            assert g["model"] == it["model"] and g["a"] == it.get("a", 0) and g["b"] == it.get("b", 0)
            assert np.array_equal(g["z"], np.asarray(it["z"], dtype=np.float64))
            assert np.array_equal(g["R"], np.asarray(it["R"], dtype=np.float64).ravel())

    base = [recorded(f)[0] for f in fs]
    r = fs[0].aid_stack_update(stack, fde=fde)
    assert r["dof"] == 1 + 1 + 2 + 3 + 3 and r["outcome"] == 0 and [it["state"] for it in r["items"]] == [0] * 5
    assert recorded(fs[0])[0] == [base[0][0] + 1, base[0][1]]
    check(fs[0], stack, fde)
    fb = FilterBatch(fs)
    fde2 = dict(fde, max_exclude=0)
    res = fb.aid_stack_update([stack[3:], None, stack[:2]], fde=fde2)
    assert res[1] is None and res[0]["dof"] == 6 and res[2]["dof"] == 2 and len(res[0]["items"]) == 2
    assert [[c[0] - b[0], c[1] - b[1]] for c, b in zip([recorded(f)[0] for f in fs], base)] == [[1, 1], [0, 0], [0, 1]]
    check(fs[0], stack[3:], fde2)
    check(fs[2], stack[:2], fde2)
    # refused in the class: nothing reaches the C-ABI
    err = fs[0].lib.msckf_mono_last_error
    err.restype = C.c_char_p
    n_calls = [recorded(f)[0] for f in fs]
    bad = [dict(fde, max_exclude=8), dict(fde, max_exclude=-1), dict(fde, chi2=[np.nan] + fde["chi2"][1:]),
           dict(fde, chi2=fde["chi2"][:31] + [0.0]), dict(fde, chi2=fde["chi2"][:5] + [np.inf] + fde["chi2"][6:])]
    for b in bad:
        with pytest.raises(RuntimeError):
            fs[0].aid_stack_update(stack, fde=b)
        assert "fde" in err().decode()
        with pytest.raises(RuntimeError):
            fb.aid_stack_update([stack, stack[:1], None], fde=b)
        assert "fde" in err().decode()
    assert [recorded(f)[0] for f in fs] == n_calls
    fb.close()
    for f in fs:
        f.close()


# ---- the Monte-Carlo runner ----------------------------------------------------------------------------------------------------
def test_runner_fault_counts_and_summary():
    """what _fault_counts makes of FDE, gated and ungated stack results, and the counts in the summary under "range" / "gnss";
    with the outlier flags off the runner draws nothing from the fault streams, so every trial input is the one make_trial gives"""
    import inspect
    it = lambda st: {"nis": np.nan, "test": np.nan, "state": st, "round": -1}  # noqa: E731
    fde_rows = [dict(nis=3.0, dof=4, applied=1, status=0, outcome=1, faults=[1], items=[it(0), it(1), it(0), it(0)]),
                dict(nis=9.0, dof=4, applied=0, status=0, outcome=2, faults=[0, 2], items=[it(1), it(3), it(3), it(3)]),
                dict(nis=2.0, dof=4, applied=1, status=0, outcome=1, faults=[], items=[it(0), it(0), it(1), it(0)]),
                dict(nis=2.0, dof=4, applied=1, status=0, outcome=0, faults=[3], items=[it(0), it(0), it(0), it(0)])]
    assert mc._fault_counts(fde_rows) == {"injected": 4, "faults_excluded": 2, "clean_excluded": 1, "faults_missed": 1,
                                          "stacks_rejected": 1}
    plain = [dict(nis=30.0, dof=4, applied=1, status=0, faults=[2]), dict(nis=30.0, dof=4, applied=0, status=0, faults=[0, 1]),
             dict(nis=0.0, dof=0, applied=0, status=0)]
    assert mc._fault_counts(plain) == {"injected": 3, "faults_excluded": 0, "clean_excluded": 0, "faults_missed": 1,
                                       "stacks_rejected": 1}
    nees = [{"orientation": 3.0, "position": 3.0, "pose": 6.0, "imu": 15.0, "full": 15.0, "dim_full": 15, "first_bad_pivot": -1}] * 4
    recs = {k: mc.trial_record(nees, [0.01] * 4, range_rows=fde_rows, gnss_rows=plain + [plain[0]]) for k in range(2)}
    s = mc.summarize(recs)
    for key, want in (("range", (8, 4, 2, 2, 2)), ("gnss", (8, 0, 0, 4, 2))):
        assert tuple(s[key][c] for c in ("injected", "faults_excluded", "clean_excluded", "faults_missed", "stacks_rejected")) == want
    # the ANIS is over the stacks applied: the rejected FDE stack's NIS (9 over 4 dof) is left out
    assert s["range"]["mean_anis"] == (3.0 + 2.0 + 2.0) / 3
    sig = inspect.signature(mc.run).parameters
    assert sig["range_outlier_rate"].default == 0.0 and sig["gnss_outlier_rate"].default == 0.0 and sig["fde_alpha"].default == 0.0
    src = inspect.getsource(mc.run)
    assert "if range_outlier_rate > 0" in src and "if gnss_outlier_rate > 0" in src  # (no draws with the flags off)
