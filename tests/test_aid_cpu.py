"""Host side of the aided measurement updates without a GPU: the class's bookkeeping around MSCKF::aidedUpdate and
MSCKFBatch::aidedUpdate (one C-ABI call per class call, queued IMU readings handed over first, the host mirror refreshed
afterwards), and the Monte-Carlo runner's position fixes (the trials' other inputs do not change).

The C view is linked against the recording fake of the C-ABI (tests/fake_engine.py), whose aided calls
(tests/stub/stub_aid.cpp) copy z of a VELOCITY / POSITION "update" into the fake's IMU state."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)
from tests.test_shim_bookkeeping_cpu import shim_filter


def _calls(f, base=(0, 0)):
    """[single calls, batched calls naming f] since `base`, and the readings handed over before the last one"""
    out = (C.c_longlong * 3)()
    f.lib.msckf_b200_stub_aid_calls(C.c_void_p(f.engineHandle()), out)
    return [out[0] - base[0], out[1] - base[1], out[2]]


def _filters(lib, n, dtype):
    wl = synth.make_stream_workload(n_frames=3, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:2]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs, wl


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_single_filter_calls_the_engine_once_and_refreshes_its_mirror(stub_view, dtype):
    (f,), wl = _filters(stub_view, 1, dtype)
    p0 = f.getImuState()["p_I_G"].copy()
    c0 = _calls(f)  # (the fake's records are per engine address: a freed engine's address may come back)
    for (w, a, dT) in wl["frames"][2]["imu"][:5]:
        f.propagate(w, a, dT)
    z = p0 + np.array([1.0, -2.0, 0.5])
    r = f.aid_update(capi.AID_POSITION, z, 0.01 * np.eye(3))
    assert r["applied"] == 1 and r["dof"] == 3 and r["status"] == 0
    assert _calls(f, c0) == [1, 0, 5]  # one C-ABI call, after the 5 queued readings were handed over
    assert np.array_equal(f.getImuState()["p_I_G"], z.astype(dtype))  # the mirror was marked stale and refreshed
    v = np.array([0.1, 0.2, 0.3])
    f.aid_update(capi.AID_VELOCITY, v, np.eye(3))
    assert _calls(f, c0)[0] == 2 and np.array_equal(f.getImuState()["v_I_G"], v.astype(dtype))
    f.aid_update(capi.AID_CLONE_POSE, np.r_[z, 0, 0, 0, 1], np.eye(6), clone=1)
    n = 15 + 6 * f.getNumCamStates()
    f.aid_update(capi.AID_LINEAR, [0.5], np.eye(1), H=np.eye(1, n, 13))
    assert _calls(f, c0)[0] == 4
    with pytest.raises(RuntimeError):  # an out-of-window clone: refused by the engine, the mirror is not touched
        f.aid_update(capi.AID_CLONE_POSE, np.r_[z, 0, 0, 0, 1], np.eye(6), clone=2)
    assert _calls(f, c0)[0] == 4 and np.array_equal(f.getImuState()["p_I_G"], z.astype(dtype))
    f.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_batch_makes_one_call_and_leaves_unnamed_members_alone(stub_view, dtype):
    fs, wl = _filters(stub_view, 3, dtype)
    fb = FilterBatch(fs)
    p0 = [f.getImuState()["p_I_G"].copy() for f in fs]
    c0 = [_calls(f) for f in fs]
    for (w, a, dT) in wl["frames"][2]["imu"][:3]:
        fb.propagate(1, w, a, dT)
    zs = [p + 10.0 * (i + 1) for i, p in enumerate(p0)]
    res = fb.aid_update([{"model": capi.AID_POSITION, "z": zs[0], "R": np.eye(3)}, None,
                         {"model": capi.AID_POSITION, "z": zs[2], "R": np.eye(3), "chi2_max": 100.0}])
    assert res[1] is None and res[0]["applied"] == 1 and res[2]["applied"] == 1
    assert fs[0].lib.msckf_b200_stub_batch_aid_calls(C.c_void_p(fb.handle())) == 1
    assert [_calls(f, c)[:2] for f, c in zip(fs, c0)] == [[0, 1], [0, 0], [0, 1]]
    assert np.array_equal(fs[0].getImuState()["p_I_G"], zs[0].astype(dtype))
    assert np.array_equal(fs[1].getImuState()["p_I_G"], p0[1])
    assert np.array_equal(fs[2].getImuState()["p_I_G"], zs[2].astype(dtype))
    # the readings queued on member 1 were handed over before the batched call, although member 1 was not updated
    fb.aid_update([None, {"model": capi.AID_VELOCITY, "z": np.zeros(3), "R": np.eye(3)}, None])
    assert _calls(fs[1], c0[1]) == [0, 1, 3]
    fb.close()
    for f in fs:
        f.close()


def test_position_fixes_leave_the_trial_inputs_unchanged():
    truth = mc.make_truth(n_frames=40, seq=8)
    for k in (0, 3):
        a = mc.make_trial(truth, k)
        b = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2)
        assert "fixes" not in a and len(b["fixes"]) == 40
        assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
        for key in a["injected"]:
            assert np.array_equal(a["injected"][key], b["injected"][key]), key
        for fa, fb_ in zip(a["frames"], b["frames"]):
            for key in ("update", "add"):
                assert np.array_equal(fa[key][0], fb_[key][0]) and np.array_equal(fa[key][1], fb_[key][1])
            for ra, rb in zip(fa["imu"], fb_["imu"]):
                assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
        fixes = [(f, z) for f, z in enumerate(b["fixes"]) if z is not None]
        assert [f for f, _ in fixes] == [4, 9, 14, 19, 24, 29, 34, 39]
        err = np.array([z - truth["truth_imu"][f][0:3] for f, z in fixes]).ravel() / 0.2
        assert stats.chi2.ppf(0.0005, err.size) <= float(err @ err) <= stats.chi2.ppf(0.9995, err.size)
    # another trial draws other fix noise; the same trial the same noise
    c = mc.make_trial(truth, 1, fix_every=5, fix_sigma=0.2)["fixes"][4]
    assert not np.array_equal(c, mc.make_trial(truth, 0, fix_every=5, fix_sigma=0.2)["fixes"][4])
    assert np.array_equal(c, mc.make_trial(truth, 1, fix_every=5, fix_sigma=0.2)["fixes"][4])


def test_summary_reports_the_anis_of_the_fixes():
    rng = np.random.default_rng(3)
    recs = {}
    for k in range(20):
        rows = [{c: 1.0 for c in mc.COMPONENTS} | {"dim_full": 21, "first_bad_pivot": -1} for _ in range(6)]
        recs[k] = mc.trial_record(rows, [0.0] * 6, rng.chisquare(3, size=4))
    s = mc.summarize(recs)
    lo, hi = stats.chi2.ppf(0.025, 60) / 20, stats.chi2.ppf(0.975, 60) / 20
    f = s["fixes"]
    assert f["dof"] == 3 and len(f["anis"]) == 4 and abs(f["lower"] - lo) < 1e-12 and abs(f["upper"] - hi) < 1e-12
    assert 0.0 <= f["fixes_inside"] <= 1.0 and abs(f["mean_anis"] - np.mean(f["anis"])) < 1e-12
    assert "fixes" not in mc.summarize({0: mc.trial_record(rows, [0.0] * 6)})  # (no fixes: no ANIS)
