"""Host logic of the batched per-image step (msckf_mono::MSCKFBatch, include/msckf_mono/msckf.h) on a box WITHOUT a GPU.

The C view is linked against the recording fake of the C-ABI (no numerics, tests/fake_engine.py), like
test_shim_bookkeeping_cpu.py does; `tests/stub/stub_batch_state.cpp` holds the fake's batched state calls.  Filters driven through the batch and single filters driven alone on the same streams
must make the same integer decisions frame by frame, and the batch must reach the C-ABI through one batched call per
device operation and frame."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import synth
from msckf_mono_b200.cview import FilterBatch
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)
from tests.test_shim_bookkeeping_cpu import _ids, shim_filter

PROPAGATE, AUGMENT, PRUNE, GET_STATE = range(4)


def _calls(fb):
    out = (C.c_longlong * 4)()
    fb.lib.msckf_b200_stub_batch_calls(C.c_void_p(fb.handle()), out)
    return list(out)


def _workloads(prune_redundant):
    if prune_redundant:  # the setting of tests/parity_cases.py::prune_redundant_case: window 21, redundancy thresholds 0.2
        wls = [synth.make_stream_workload(n_frames=60, seq=9 + i, max_features=30 + 5 * i, max_track_length=30 + 5 * i, max_cam_states=21)
               for i in range(3)]
        for wl in wls:
            wl["params"]["redundancy_angle_thresh"] = 0.2
            wl["params"]["redundancy_distance_thresh"] = 0.2
        return wls
    return [synth.make_stream_workload(n_frames=60, seq=i, max_features=40 + 5 * i, max_track_length=(50, 12, 6)[i], max_cam_states=(30, 10, 20)[i])
            for i in range(3)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("prune_redundant", [False, True])
def test_batched_step_keeps_the_bookkeeping_of_single_filters(stub_view, dtype, prune_redundant):
    wls = _workloads(prune_redundant)
    solo = [shim_filter(stub_view, dtype) for _ in wls]
    grp = [shim_filter(stub_view, dtype) for _ in wls]
    for wl, a, b in zip(wls, solo, grp):
        a.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        b.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    fb = FilterBatch(grp)
    pruned_frames = 0
    for k in range(len(wls[0]["frames"])):
        c0 = _calls(fb)
        n0 = [a.getNumCamStates() for a in solo]
        frs = [wl["frames"][k] for wl in wls]
        queued = 0
        for i, fr in enumerate(frs):
            if i == 1 and k % 3 == 0:
                continue  # frames where a member has nothing queued
            queued += len(fr["imu"])
            for (w, acc, dT) in fr["imu"]:
                solo[i].propagate(w, acc, dT)
                fb.propagate(i, w, acc, dT)
        for a, fr in zip(solo, frs):
            a.augmentState(fr["state_id"], fr["time"])
        fb.augmentState([fr["state_id"] for fr in frs], [fr["time"] for fr in frs])
        for a, b, fr in zip(solo, grp, frs):
            for f in (a, b):
                f.update(*fr["update"])
                f.addFeatures(*fr["add"])
        for a in solo:
            a.marginalize()
        fb.marginalize()
        for a, b in zip(solo, grp):
            assert len(a.lastReport()["valid"]) == len(b.lastReport()["valid"]), k
        if prune_redundant:
            for a in solo:
                a.pruneRedundantStates()
            fb.pruneRedundantStates()
        for a in solo:
            a.pruneEmptyStates()
        fb.pruneEmptyStates()
        c1 = _calls(fb)
        for a, b in zip(solo, grp):
            assert _ids(a) == _ids(b), k
            assert np.array_equal(a.getPrunedStates()["state_id"], b.getPrunedStates()["state_id"]), k
        # one batched call per device operation: propagate (where readings are queued) and augment once a frame, prune at
        # most once per prune step
        assert c1[PROPAGATE] - c0[PROPAGATE] == (1 if queued else 0) and c1[AUGMENT] - c0[AUGMENT] == 1, k
        shrank = any(a.getNumCamStates() < n + 1 for a, n in zip(solo, n0))
        assert (c1[PRUNE] - c0[PRUNE] > 0) == shrank, k
        assert c1[PRUNE] - c0[PRUNE] <= (2 if prune_redundant else 1), k
        pruned_frames += shrank
    assert pruned_frames > 5
    assert all(len(a.getPrunedStates()["state_id"]) > 0 for a in solo)
    # finish(): every remaining track residualised through one batched update
    ok = []
    for a in solo:
        try:
            a.finish()
            ok.append(True)
        except RuntimeError as e:
            assert "stale residualisation queue" in str(e)
            ok.append(False)
    if all(ok):
        fb.finish()
        for a, b in zip(solo, grp):
            assert len(a.lastReport()["valid"]) == len(b.lastReport()["valid"])
            assert _ids(a) == _ids(b)
    fb.close()


def test_batched_propagate_rejects_a_bad_member_index(stub_view):
    wl = synth.make_stream_workload(n_frames=2, seq=1, max_features=10)
    fs = [shim_filter(stub_view, np.float64) for _ in range(2)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    fb = FilterBatch(fs)
    with pytest.raises(RuntimeError, match="member index"):
        fb.propagate(2, [0, 0, 0], [0, 0, 9.81], 0.005)
    fb.close()
