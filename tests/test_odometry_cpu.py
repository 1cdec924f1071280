"""Host side of the stacked aided updates (odometry) without a GPU: the class's bookkeeping around MSCKF::aidedUpdate(items),
bodyVelocityUpdate, relativePoseUpdate and MSCKFBatch::aidedUpdate(items) (one C-ABI call per class call, queued IMU readings
handed over first, the host mirror refreshed afterwards, state ids mapped to window positions), and the Monte-Carlo runner's
odometry (the trials' other inputs do not change; the truth odometry agrees with the truth trajectory).

The C view is linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp)
plus tests/stub/stub_aid_stack.cpp, whose VELOCITY / POSITION items copy z into the fake's IMU state."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.test_shim_bookkeeping_cpu import shim_filter


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_odometry_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / n for n in ("stub_engine.cpp", "stub_batch_state.cpp", "stub_aid.cpp", "stub_aid_stack.cpp")]
    src += [csrc / n for n in ("filter_capi.cpp", "batch_capi.cpp", "aid_capi.cpp", "aid_stack_capi.cpp")]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", *map(str, src), "-o", str(so)])
    return so


def _calls(f, base=(0, 0)):
    """[single calls, batched calls naming f] since `base`, the readings handed over before the last one, and that call's
    items as (model, a, b) triples"""
    out = (C.c_longlong * 3)()
    items = (C.c_int * 24)()
    n = f.lib.msckf_b200_stub_aid_stack_calls(C.c_void_p(f.engineHandle()), out, items, 8)
    return [out[0] - base[0], out[1] - base[1], out[2]], [tuple(items[3 * k:3 * k + 3]) for k in range(n)]


def _filters(lib, n, dtype, frames=3):
    wl = synth.make_stream_workload(n_frames=frames + 1, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:frames]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs, wl


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_single_filter_calls_the_engine_once_and_refreshes_its_mirror(stub_view, dtype):
    (f,), wl = _filters(stub_view, 1, dtype)
    ids = list(f.getCamStates()["state_id"])
    assert len(ids) == 3
    p0 = f.getImuState()["p_I_G"].copy()
    c0 = _calls(f)[0]
    for (w, a, dT) in wl["frames"][3]["imu"][:5]:
        f.propagate(w, a, dT)
    z = p0 + np.array([1.0, -2.0, 0.5])
    q = np.array([0.0, 0.0, 0.0, 1.0])
    items = [{"model": capi.AID_BODY_VELOCITY, "a": 0b110, "z": np.zeros(3), "R": np.eye(2)},
             {"model": capi.AID_RELATIVE_POSE, "a": 0, "b": 2, "z": np.r_[0.1, 0.0, 0.0, q], "R": np.eye(6)},
             {"model": capi.AID_POSITION, "z": z, "R": 0.01 * np.eye(3)}]
    r = f.aid_stack_update(items)
    assert r["applied"] == 1 and r["dof"] == 11 and r["status"] == 0
    calls, got = _calls(f, c0)
    assert calls == [1, 0, 5]  # one C-ABI call, after the 5 queued readings were handed over
    assert got == [(capi.AID_BODY_VELOCITY, 0b110, 0), (capi.AID_RELATIVE_POSE, 0, 2), (capi.AID_POSITION, 0, 0)]
    assert np.array_equal(f.getImuState()["p_I_G"], z.astype(dtype))  # the mirror was marked stale and refreshed
    # the single-item forms: one call each; state ids become window positions
    f.body_velocity_update([1.0, 0.0, 0.0], np.eye(1), mask=0b001)
    calls, got = _calls(f, c0)
    assert calls[0] == 2 and got == [(capi.AID_BODY_VELOCITY, 0b001, 0)]
    f.relative_pose_update(ids[2], ids[1], [0.1, 0.2, 0.3], q, np.eye(6))
    calls, got = _calls(f, c0)
    assert calls[0] == 3 and got == [(capi.AID_RELATIVE_POSE, 2, 1)]
    # a state id that is not in the window, or a mask that selects nothing: refused before any device call
    with pytest.raises(RuntimeError, match="not in the window"):
        f.relative_pose_update(ids[0], max(ids) + 1, [0.1, 0.2, 0.3], q, np.eye(6))
    with pytest.raises(RuntimeError):
        f.body_velocity_update([1.0, 0.0, 0.0], np.eye(1), mask=0)
    # an item the engine refuses (a == b) leaves the mirror alone
    with pytest.raises(RuntimeError):
        f.aid_stack_update([{"model": capi.AID_RELATIVE_POSE, "a": 1, "b": 1, "z": np.r_[0.1, 0.0, 0.0, q], "R": np.eye(6)}])
    assert _calls(f, c0)[0][0] == 3 and np.array_equal(f.getImuState()["p_I_G"], z.astype(dtype))
    f.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_batch_makes_one_call_and_leaves_unnamed_members_alone(stub_view, dtype):
    fs, wl = _filters(stub_view, 3, dtype)
    fb = FilterBatch(fs)
    p0 = [f.getImuState()["p_I_G"].copy() for f in fs]
    c0 = [_calls(f)[0] for f in fs]
    for (w, a, dT) in wl["frames"][3]["imu"][:3]:
        fb.propagate(1, w, a, dT)
    zs = [p + 10.0 * (i + 1) for i, p in enumerate(p0)]
    bv = {"model": capi.AID_BODY_VELOCITY, "a": 0b111, "z": np.zeros(3), "R": np.eye(3)}
    res = fb.aid_stack_update([[bv, {"model": capi.AID_POSITION, "z": zs[0], "R": np.eye(3)}], None,
                               [{"model": capi.AID_POSITION, "z": zs[2], "R": np.eye(3)}]])
    assert res[1] is None and res[0]["dof"] == 6 and res[2]["dof"] == 3
    assert fs[0].lib.msckf_b200_stub_batch_aid_stack_calls(C.c_void_p(fb.handle())) == 1
    assert [_calls(f, c)[0][:2] for f, c in zip(fs, c0)] == [[0, 1], [0, 0], [0, 1]]
    assert np.array_equal(fs[0].getImuState()["p_I_G"], zs[0].astype(dtype))
    assert np.array_equal(fs[1].getImuState()["p_I_G"], p0[1])
    assert np.array_equal(fs[2].getImuState()["p_I_G"], zs[2].astype(dtype))
    # the readings queued on member 1 were handed over before the batched call, although member 1 was not updated
    fb.aid_stack_update([[], [bv], None])
    assert _calls(fs[1], c0[1])[0] == [0, 1, 3]
    fb.close()
    for f in fs:
        f.close()


def test_odometry_leaves_the_trial_inputs_unchanged():
    truth = mc.make_truth(n_frames=40, seq=8)
    for k in (0, 3):
        a = mc.make_trial(truth, k)
        b = mc.make_trial(truth, k, odo_every=4)
        assert "odometry" not in a and len(b["odometry"]) == 40
        assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
        for key in a["injected"]:
            assert np.array_equal(a["injected"][key], b["injected"][key]), key
        for fa, fb_ in zip(a["frames"], b["frames"]):
            for key in ("update", "add"):
                assert np.array_equal(fa[key][0], fb_[key][0]) and np.array_equal(fa[key][1], fb_[key][1])
            for ra, rb in zip(fa["imu"], fb_["imu"]):
                assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
        assert [f for f, n in enumerate(b["odometry"]) if n is not None] == list(range(3, 40, 4))
        # fixes and the map draw from their own streams: the same with odometry on or off
        c = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2, odo_every=1)
        d = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2)
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(c["fixes"], d["fixes"]))
    # another trial draws other odometry noise; the same trial the same noise
    n1 = mc.make_trial(truth, 1, odo_every=2)["odometry"][3]
    assert not np.array_equal(n1, mc.make_trial(truth, 0, odo_every=2)["odometry"][3])
    assert np.array_equal(n1, mc.make_trial(truth, 1, odo_every=2)["odometry"][3])


@pytest.mark.parametrize("nhc", [False, True])
def test_truth_odometry_has_zero_residual_against_the_truth(nhc):
    """noise-free odometry items from truth_imu / truth_pose against the trajectory itself (rotation matrices of synth, not
    montecarlo's quaternion products)"""
    truth = mc.make_truth(n_frames=30, seq=8)
    traj, cam = truth["traj"], truth["camera"]
    for f in (1, 7, 29):
        a, b = f - 1, f
        t, ta = truth["frames"][b]["time"], truth["frames"][a]["time"]
        items = mc.odometry_items(truth["truth_imu"][f], truth["truth_pose"][a], truth["truth_pose"][b], np.zeros(9), 0.1, 0.1, nhc)
        bv, rel = items
        v_I = traj.R_GI(t).T @ traj.vel(t)
        assert bv["a"] == (0b110 if nhc else 0b111) and bv["R"].shape == ((2, 2) if nhc else (3, 3))
        assert np.abs(bv["z"] - v_I).max() <= 1e-12 * max(1.0, np.abs(v_I).max())
        Ca, pa = synth.cam_pose(traj, ta, cam)
        Cb, pb = synth.cam_pose(traj, t, cam)
        p_rel, C_rel = Ca @ (pb - pa), Cb @ Ca.T
        assert np.abs(rel["z"][0:3] - p_rel).max() <= 1e-12
        assert np.abs(mc.quat_to_rot(rel["z"][3:7]) - C_rel).max() <= 1e-12
        assert abs(np.linalg.norm(rel["z"][3:7]) - 1.0) <= 1e-15
        # the residual of the models at the truth state is zero (dtheta of POSE's convention)
        q_hat = mc.quat_mul(truth["truth_pose"][b][3:7], mc.quat_inv(truth["truth_pose"][a][3:7]))
        assert np.abs(mc.quat_error(rel["z"][3:7], q_hat)).max() <= 1e-12


def test_summary_reports_the_anis_of_the_odometry():
    from scipy import stats
    rng = np.random.default_rng(3)
    recs = {}
    rows = [{c: 1.0 for c in mc.COMPONENTS} | {"dim_full": 21, "first_bad_pivot": -1} for _ in range(5)]
    for k in range(10):
        dof = [3, 9, 9, 9]
        recs[k] = mc.trial_record(rows, [0.0] * 5, odo_rows=[{"nis": rng.chisquare(d), "dof": d, "applied": 1} for d in dof])
    s = mc.summarize(recs)
    o = s["odometry"]
    assert o["dof"] == [30, 90, 90, 90] and len(o["anis"]) == 4
    assert abs(o["lower"][0] - stats.chi2.ppf(0.025, 30) / 10) < 1e-12 and abs(o["upper"][1] - stats.chi2.ppf(0.975, 90) / 10) < 1e-12
    assert abs(o["mean_dof"] - 7.5) < 1e-12 and o["applied"] == 1.0
    assert "odometry" not in mc.summarize({0: mc.trial_record(rows, [0.0] * 5)})
