"""Host side of the mapped-landmark updates without a GPU: the class's bookkeeping around MSCKF::landmarkUpdate and
MSCKFBatch::landmarkUpdate (one C-ABI call per class call, queued IMU readings handed over first, state ids mapped to window
positions, unknown ids refused before any call, marginalize() refusing tracks queued before an applied update), and the
Monte-Carlo runner's map observations (the trials' other inputs do not change).

The C view is linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp, stub_batch_state.cpp) plus
tests/stub/stub_landmark.cpp, which records the window positions it is given and applies nothing."""
import ctypes as C
import subprocess

import numpy as np
import pytest
from scipy import stats

from msckf_mono_b200 import montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.test_shim_bookkeeping_cpu import shim_filter


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_landmark_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / "stub_engine.cpp", ROOT / "tests" / "stub" / "stub_batch_state.cpp",
           ROOT / "tests" / "stub" / "stub_landmark.cpp", csrc / "filter_capi.cpp", csrc / "batch_capi.cpp", csrc / "landmark_capi.cpp"]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", *map(str, src), "-o", str(so)])
    return so


def _calls(f, base=(0, 0)):
    """[single calls, batched calls naming f] since `base`, and the readings handed over before the last one"""
    out = (C.c_longlong * 3)()
    f.lib.msckf_b200_stub_landmark_calls(C.c_void_p(f.engineHandle()), out)
    return [out[0] - base[0], out[1] - base[1], out[2]]


def _clones(f):
    out = (C.c_int * 256)()
    n = f.lib.msckf_b200_stub_landmark_clones(C.c_void_p(f.engineHandle()), out, 256)
    return list(out[:n])


def _filters(lib, n, dtype, frames=3):
    wl = synth.make_stream_workload(n_frames=frames, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:frames - 1]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs, wl


def _obs(n):
    return np.tile([0.01, -0.02], (n, 1)), np.tile([1.0, 2.0, 5.0], (n, 1))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_single_filter_calls_the_engine_once_after_the_queued_readings(stub_view, dtype):
    (f,), wl = _filters(stub_view, 1, dtype, frames=4)
    c0 = _calls(f)
    for (w, a, dT) in wl["frames"][3]["imu"][:4]:
        f.propagate(w, a, dT)
    z, p = _obs(3)
    r = f.landmark_update([2, 0, 2], z, p, R=[[1e-5, 0.0], [0.0, 1e-5]])
    assert r["applied"] == 1 and r["used"] == 3 and list(r["flag"]) == [0, 0, 0]
    assert _calls(f, c0) == [1, 0, 4] and _clones(f) == [2, 0, 2]
    # an image that is not in the window: refused before any C-ABI call
    with pytest.raises(RuntimeError, match="not in the window"):
        f.landmark_update([1, 7], *_obs(2))
    assert _calls(f, c0)[:2] == [1, 0]
    f.close()


def test_state_ids_map_to_window_positions_after_prunes(stub_view):
    wl = synth.make_stream_workload(n_frames=12, seq=2, max_features=10, max_cam_states=6)
    f = shim_filter(stub_view, np.float64)
    f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    for fr in wl["frames"][:12]:  # images without features: pruneEmptyStates trims the window to max_cam_states
        f.augmentState(fr["state_id"], fr["time"])
        f.pruneEmptyStates()
    ids = list(f.getCamStates()["state_id"])
    assert ids[0] > 0 and ids != list(range(len(ids)))  # the window was pruned
    pick = [ids[-1], ids[0], ids[len(ids) // 2], ids[-1]]
    f.landmark_update(pick, *_obs(4))
    assert _clones(f) == [len(ids) - 1, 0, len(ids) // 2, len(ids) - 1]
    with pytest.raises(RuntimeError, match="not in the window"):
        f.landmark_update([0], *_obs(1))  # pruned long ago
    f.close()


def test_applied_update_between_update_and_marginalize_is_refused(stub_view):
    wl = synth.make_stream_workload(n_frames=5, seq=2, max_features=10)
    f = shim_filter(stub_view, np.float64)
    f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    z2, ids = np.array([[0.01, 0.02], [-0.03, 0.01]]), np.array([1, 2], dtype=np.uint64)
    for k, fr in enumerate(wl["frames"][:5]):
        f.augmentState(fr["state_id"], fr["time"])
        if k == 0:
            f.addFeatures(z2, ids)
        elif k < 4:
            f.update(z2, ids)
        else:
            f.update(np.zeros((0, 2)), np.zeros(0, dtype=np.uint64))  # both tracks end: queued for marginalize()
    assert len(f.queuedTracks()[0]) == 2
    f.landmark_update([4], *_obs(1))
    with pytest.raises(RuntimeError, match="measurement update was applied"):
        f.marginalize()
    f.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_batch_makes_one_call_and_leaves_empty_lists_alone(stub_view, dtype):
    fs, wl = _filters(stub_view, 3, dtype, frames=4)
    fb = FilterBatch(fs)
    c0 = [_calls(f) for f in fs]
    for (w, a, dT) in wl["frames"][3]["imu"][:3]:
        fb.propagate(1, w, a, dT)
    z, p = _obs(3)
    res = fb.landmark_update([([0, 1], z[:2], p[:2]), None, ([2], z[:1], p[:1])])
    assert res[1] is None and res[0]["used"] == 2 and res[2]["used"] == 1 and len(res[0]["gamma"]) == 2
    assert fs[0].lib.msckf_b200_stub_batch_landmark_calls(C.c_void_p(fb.handle())) == 1
    assert [_calls(f, c)[:2] for f, c in zip(fs, c0)] == [[0, 1], [0, 0], [0, 1]]
    assert _clones(fs[0]) == [0, 1] and _clones(fs[2]) == [2]
    # the readings queued on member 1 were handed over before the batched call, although member 1 was not updated
    fb.landmark_update([None, ([1], z[:1], p[:1]), None])
    assert _calls(fs[1], c0[1]) == [0, 1, 3]
    with pytest.raises(RuntimeError, match="not in the window"):  # one unknown id: no call at all
        fb.landmark_update([([0], z[:1], p[:1]), ([9], z[:1], p[:1]), None])
    assert fs[0].lib.msckf_b200_stub_batch_landmark_calls(C.c_void_p(fb.handle())) == 2
    fb.close()
    for f in fs:
        f.close()


def test_map_leaves_the_trial_inputs_unchanged():
    truth = mc.make_truth(n_frames=30, seq=8)
    nz = truth["noise"]
    for k in (0, 3):
        a = mc.make_trial(truth, k)
        b = mc.make_trial(truth, k, map_every=1, map_stride=20)
        assert "maps" not in a and len(b["maps"]) == 30
        assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
        for key in a["injected"]:
            assert np.array_equal(a["injected"][key], b["injected"][key]), key
        for fa, fb_ in zip(a["frames"], b["frames"]):
            for key in ("update", "add"):
                assert np.array_equal(fa[key][0], fb_[key][0]) and np.array_equal(fa[key][1], fb_[key][1])
            for ra, rb in zip(fa["imu"], fb_["imu"]):
                assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
        # the map observations' noise against the truth projections lies inside chi^2 99.9 % bounds
        err = []
        for f, m in enumerate(b["maps"]):
            idx, p_L, z = m
            idx0, z0 = mc.map_observations(truth, f, 20)
            assert np.array_equal(idx, idx0) and np.array_equal(p_L, truth["landmarks"][::20][idx])
            err.append(((z - z0) / np.sqrt([nz["u_var_prime"], nz["v_var_prime"]])).ravel())
        err = np.concatenate(err)
        assert err.size > 100
        assert stats.chi2.ppf(0.0005, err.size) <= float(err @ err) <= stats.chi2.ppf(0.9995, err.size)


def test_visibility_helper_is_the_stream_rule():
    wl = synth.make_stream_workload(n_frames=5, seq=1, max_features=30)
    for fr in wl["frames"]:
        C_, p = synth.cam_pose(wl["traj"], fr["time"], wl["camera"])
        vis, xn, yn = synth.visible(C_, p, wl["landmarks"])
        assert vis.sum() > 30
