"""Host logic of the drop-in class shim (`include/msckf_mono/msckf.h`) on a box WITHOUT a GPU.

The shim keeps every integer decision of the reference on the host (update(): which tracks are residualised and with
which clones, addFeatures(), pruneEmptyStates(), finish(); msckf.h:215-332, :685-807) and forwards only numerics to the
C-ABI.  Here the C view of the shim is linked against the recording fake of the C-ABI built by `tests/fake_engine.py`
-- without any numerics (test infrastructure, not a fallback) -- and driven next to the oracle on the same streams.
Everything that does not depend on a computed number must be identical, frame by frame."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import synth
from msckf_mono_b200.cview import CFilter
from tests.common import make_oracle
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)


def shim_filter(lib, dtype, max_clones=0):
    f = CFilter(lib, "msckf_mono_", dtype)
    assert f.lib.msckf_mono_set_engine_options(f.h, C.c_int(0), C.c_int(max_clones), C.c_int(0), C.c_int(0)) == 0
    return f


def _step(f, fr):
    for (omega, a, dT) in fr["imu"]:
        f.propagate(omega, a, dT)
    f.augmentState(fr["state_id"], fr["time"])
    if fr["update"] is not None:
        f.update(fr["update"][0], fr["update"][1])
    if fr["add"] is not None:
        f.addFeatures(fr["add"][0], fr["add"][1])


def _ids(f):
    cs = f.getCamStates()
    per_clone = [tuple(int(x) for x in f.getCamTrackedIds(i)) for i in range(f.getNumCamStates())]
    return (tuple(int(x) for x in cs["state_id"]), tuple(int(x) for x in cs["last_correlated_id"]),
            tuple(int(x) for x in f.getTrackedFeatureIds()), per_clone)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("seq,max_track_length,max_cam_states", [(0, 50, 30), (3, 12, 10), (5, 6, 30)])
def test_stream_bookkeeping_matches_oracle(stub_view, oracle_lib, dtype, seq, max_track_length, max_cam_states):
    wl = synth.make_stream_workload(n_frames=70, seq=seq, max_features=50, max_track_length=max_track_length,
                                    max_cam_states=max_cam_states)
    s, o = shim_filter(stub_view, dtype), make_oracle(oracle_lib, dtype)
    for f in (s, o):
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    n_queued = 0
    for k, fr in enumerate(wl["frames"]):
        _step(s, fr); _step(o, fr)
        qs, qo = s.queuedTracks(), o.queuedTracks()  # what update() decided to residualise, with how many observations
        assert np.array_equal(qs[0], qo[0]) and np.array_equal(qs[1], qo[1]), k
        n_queued += len(qs[0])
        assert _ids(s) == _ids(o), k
        s.marginalize(); o.marginalize()
        assert len(s.lastReport()["valid"]) == len(o.lastReport()["valid"]) == len(qs[0])
        s.pruneEmptyStates(); o.pruneEmptyStates()
        assert _ids(s) == _ids(o), k
        assert np.array_equal(s.getPrunedStates()["state_id"], o.getPrunedStates()["state_id"]), k
    assert n_queued > 50  # the streams do residualise tracks
    # finish() residualises everything that is left (msckf.h:765-807).  The reference clears the residualisation queue in
    # update() only (:218), so when the last update() queued tracks, finish() would run them a second time with their old
    # positional clone indices -- past the end of the window once pruneEmptyStates() removed clones: undefined behaviour
    # there, a loud error in both the oracle and the shim.
    def finish(f):
        try:
            f.finish()
            return True
        except RuntimeError as e:
            assert "stale residualisation queue" in str(e)
            return False

    ok_s, ok_o = finish(s), finish(o)
    assert ok_s == ok_o
    if ok_s:
        assert len(s.lastReport()["valid"]) == len(o.lastReport()["valid"])
        assert _ids(s) == _ids(o)


def test_finish_after_a_quiet_frame(stub_view, oracle_lib):
    """finish() where it is well defined in the reference: the last update() queued nothing."""
    wl = synth.make_stream_workload(n_frames=69, seq=0, max_features=50, max_track_length=50, max_cam_states=30)
    s, o = shim_filter(stub_view, np.float64), make_oracle(oracle_lib, np.float64)
    for f in (s, o):
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"]:
            _step(f, fr)
            last_queue = len(f.queuedTracks()[0])
            f.marginalize()
            f.pruneEmptyStates()
        assert last_queue == 0
        f.finish()
    ns, no = len(s.lastReport()["valid"]), len(o.lastReport()["valid"])
    assert ns == no and ns > 20
    assert _ids(s) == _ids(o) and len(s.getTrackedFeatureIds()) > 0  # (finish() leaves the id lists alone, like the reference)


def test_packed_batch_is_what_the_reference_would_residualise(stub_view, oracle_lib):
    """the flat SoA batch handed to the C-ABI: offsets, observations in arrival order, POSITIONAL clone indices (msckf.h:1481)"""
    wl = synth.make_stream_workload(n_frames=40, seq=2, max_features=30, max_track_length=8)
    s = shim_filter(stub_view, np.float64)
    s.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    seen = {}
    checked = 0
    for fr in wl["frames"]:
        for key in ("update", "add"):
            for z, i in zip(np.asarray(fr[key][0]).reshape(-1, 2), fr[key][1]):
                seen.setdefault(int(i), []).append((fr["state_id"], z))
        _step(s, fr)
        ids, nobs = s.queuedTracks()
        if len(ids):
            off, obs, idx = s.packQueued()
            cam_ids = list(s.getCamStates()["state_id"])
            assert list(np.diff(off)) == list(nobs)
            for t, fid in enumerate(ids):
                hist = seen[int(fid)]
                assert nobs[t] == len(hist)
                for j, (sid, z) in enumerate(hist):
                    assert np.array_equal(obs[2 * (off[t] + j):2 * (off[t] + j) + 2], z)
                    assert cam_ids[idx[off[t] + j]] == sid  # positional index -> the clone that saw it
                checked += 1
        s.marginalize()
        s.pruneEmptyStates()
    assert checked > 20


def test_duplicate_feature_id_drops_the_rest_like_the_reference(stub_view, oracle_lib):
    """addFeatures() with an id that is already tracked prints and returns early, dropping the remaining new features
    (msckf.h:327-330) -- reproduced, not fixed."""
    wl = synth.make_stream_workload(n_frames=3, seq=1, max_features=10)
    s, o = shim_filter(stub_view, np.float64), make_oracle(oracle_lib, np.float64)
    for f in (s, o):
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        _step(f, wl["frames"][0])
        f.augmentState(1, 1.05)
        dup = np.array([9001, int(wl["frames"][0]["add"][1][0]), 9002], dtype=np.uint64)
        f.addFeatures(np.zeros((3, 2)), dup)
    assert np.array_equal(s.getTrackedFeatureIds(), o.getTrackedFeatureIds())
    assert 9001 in s.getTrackedFeatureIds() and 9002 not in s.getTrackedFeatureIds()
