"""Device batches of the whole per-image step: msckf_b200_batch_{propagate_n, augment, prune, get_state} and the full
msckf_mono::MSCKFBatch step must give every member exactly the bits of the same calls made filter by filter."""
import numpy as np
import pytest

from msckf_mono_b200 import capi, synth
from msckf_mono_b200.cview import FilterBatch
from tests.parity_cases import make_engine

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]


class Member:
    """an initialised engine (owned by a class filter, driven through the raw C-ABI) with M clones and a non-trivial P"""

    def __init__(self, dtype, M, seed, max_clones=None, twin_of=None):
        wl = synth.make_window_workload(n_features=4, n_clones=2, seq=3)
        self.f = make_engine(dtype, max_clones=max_clones or M + 8, max_tracks=16, max_obs=256)
        self.f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        self.e = capi.Engine(dtype, borrowed=self.f.engineHandle())
        if twin_of is not None:
            self.e.copy_state_from(twin_of.e)
            return
        rng = np.random.default_rng(seed)
        self.e.propagate_n(readings(rng, 3))
        for _ in range(M):
            self.e.propagate_n(readings(rng, 2))
            self.e.augment()
        n = 15 + 6 * M
        A = rng.normal(size=(n, n))
        self.e.set_covariance(A @ A.T / n + np.eye(n))

    def twin(self, dtype, max_clones=None):
        return Member(dtype, self.e.num_clones(), 0, max_clones=max_clones or self.e.num_clones() + 8, twin_of=self)

    def snapshot(self):
        imu, poses = self.e.state()
        return imu, poses, self.e.covariance()


def readings(rng, k):
    r = np.zeros((k, 7))
    r[:, 0:3] = rng.normal(0, 0.3, (k, 3))
    r[:, 3:6] = np.array([0, 0, 9.81]) + rng.normal(0, 0.5, (k, 3))
    r[:, 6] = 0.005
    return r


def assert_same(a, b):
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert x.shape == y.shape and np.array_equal(x, y)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batched_propagate_is_bit_identical(dtype):
    """windows 0, 5, 30 and 90 clones (90: past the 85 clones whose P_IC columns k_propagate keeps in registers), per-member
    reading counts 0, 1, 16, 17 and 40 (one, two and three steps of 16 readings); then a batch of one member, which takes the
    NM = 1 form of the kernels"""
    for Ms in ([0, 5, 30, 90], [30]):
        mem = [Member(dtype, M, seed=i) for i, M in enumerate(Ms)]
        twins = [m.twin(dtype) for m in mem]
        for a, b in zip(mem, twins):
            assert_same(a, b)
        batch = capi.Batch([m.e for m in mem])
        rng = np.random.default_rng(7)
        for ks in ([1, 16, 17, 40], [40, 0, 1, 16], [17, 40, 0, 1], [0, 0, 0, 0]):
            rs = [readings(rng, k) for k in ks[:len(Ms)]]
            batch.propagate_n(rs)
            for t, r in zip(twins, rs):
                if len(r):
                    t.e.propagate_n(r)
            for a, b in zip(mem, twins):
                assert_same(a, b)
        # the batched getter returns what the single-engine getter returns
        for (imu, poses), m in zip(batch.state(), mem):
            imu1, poses1 = m.e.state()
            assert np.array_equal(imu, imu1) and np.array_equal(poses, poses1)
        batch.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_batched_prune_and_augment_are_bit_identical(dtype):
    keeps = [list(range(6)), [], [0, 2, 4], [2, 3, 4, 5], None]  # keep all, keep none, every other, drop the first two, untouched
    mem = [Member(dtype, 6, seed=10 + i) for i in range(len(keeps))]
    mem.append(Member(dtype, 6, seed=20, max_clones=6))  # full: its augment has to grow the clone capacity
    twins = [m.twin(dtype, max_clones=6 if i == len(mem) - 1 else None) for i, m in enumerate(mem)]
    batch = capi.Batch([m.e for m in mem])
    batch.prune(keeps + [None])
    for t, k in zip(twins, keeps):
        if k is not None:
            t.e.prune(k)
    for a, b in zip(mem, twins):
        assert_same(a, b)
    assert [m.e.num_clones() for m in mem] == [6, 0, 3, 4, 6, 6]
    which = [1, 0, 1, 1, 1, 1]
    batch.augment(which)
    for t, w in zip(twins, which):
        if w:
            t.e.augment()
    assert [m.e.num_clones() for m in mem] == [7, 0, 4, 5, 7, 7]
    for a, b in zip(mem, twins):
        assert_same(a, b)
    batch.close()


def test_launch_counts():
    """one launch per device operation for up to 32 members; past that one launch per 32 members (and per step of 16 readings)"""
    mem = [Member(np.float32, 3, seed=i) for i in range(40)]
    rng = np.random.default_rng(1)
    b8 = capi.Batch([m.e for m in mem[:8]])
    for call, expect in ((lambda: b8.propagate_n([readings(rng, k) for k in (16, 3, 0, 1, 16, 7, 9, 2)]), 1),
                         (lambda: b8.propagate_n([readings(rng, k) for k in (17, 3, 0, 1, 16, 7, 9, 2)]), 2),
                         (lambda: b8.augment(), 1),
                         (lambda: b8.prune([[0, 2]] * 8), 1)):
        n0 = b8.launch_count()
        call()
        assert b8.launch_count() - n0 == expect
    b8.close()
    b40 = capi.Batch([m.e for m in mem])
    for call, expect in ((lambda: b40.propagate_n([readings(rng, 1)] * 40), 2),
                         (lambda: b40.propagate_n([readings(rng, 20)] * 33 + [readings(rng, 1)] * 7), 4),
                         (lambda: b40.augment(), 2),
                         (lambda: b40.prune([[0]] * 40), 2)):
        n0 = b40.launch_count()
        call()
        assert b40.launch_count() - n0 == expect
    b40.close()


def test_bad_arguments_change_no_member():
    mem = [Member(np.float64, 5, seed=30 + i) for i in range(4)]
    before = [m.snapshot() for m in mem]
    batch = capi.Batch([m.e for m in mem])
    rng = np.random.default_rng(2)
    with pytest.raises(RuntimeError, match="rc=-3"):  # MSCKF_B200_ERR_ARG
        batch.prune([[0, 1], [0, 2], [3, 1], None])  # member 2's list is not ascending
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.prune([[0, 1], [0, 7], None, None])  # position past the window
    import ctypes as C
    r = readings(rng, 2)
    ptrs = (C.c_void_p * 4)(*[r.ctypes.data] * 4)
    with pytest.raises(RuntimeError, match="rc=-3"):
        capi.check(capi.lib().msckf_b200_batch_propagate_n(batch.h, ptrs, (C.c_int * 4)(2, 2, -1, 2)), "batch_propagate_n")
    with pytest.raises(RuntimeError, match="rc=-3"):
        capi.check(capi.lib().msckf_b200_batch_propagate_n(batch.h, (C.c_void_p * 4)(ptrs[0], None, ptrs[0], ptrs[0]), (C.c_int * 4)(2, 2, 2, 2)), "batch_propagate_n")
    for m, b in zip(mem, before):
        for x, y in zip(m.snapshot(), b):
            assert np.array_equal(x, y)
    batch.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_class_stream_fully_batched_is_bit_identical(dtype):
    """four filters (different seeds, windows, track lengths; pruneRedundantStates really prunes: redundancy thresholds 0.2)
    streamed in lockstep through the fully batched MSCKFBatch step, against the same filters run alone"""
    cfg = [(9, 21, 40), (60, 24, 30), (61, 21, 20), (62, 28, 40)]
    wls = []
    for seq, window, track in cfg:
        wl = synth.make_stream_workload(n_frames=90, seq=seq, max_features=40, max_track_length=track, max_cam_states=window)
        wl["params"]["redundancy_angle_thresh"] = 0.2
        wl["params"]["redundancy_distance_thresh"] = 0.2
        wls.append(wl)
    solo, grp = [], []
    for wl in wls:
        a, b = make_engine(dtype), make_engine(dtype)
        for f in (a, b):
            f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        solo.append(a); grp.append(b)
    fb = FilterBatch(grp, threads=2)
    quiet = 0
    for k in range(90):
        frs = [wl["frames"][k] for wl in wls]
        for i, fr in enumerate(frs):
            if i == 2 and k % 7 == 3:
                continue  # a member with no IMU readings queued in this frame
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
        for i, (a, b) in enumerate(zip(solo, grp)):
            ra, rb = a.lastReport(), b.lastReport()
            quiet += len(ra["accepted"]) == 0
            assert np.array_equal(ra["accepted"], rb["accepted"]) and np.array_equal(ra["gamma"], rb["gamma"]), (k, i)
        for a in solo:
            a.pruneRedundantStates()
            a.pruneEmptyStates()
        fb.pruneRedundantStates()
        fb.pruneEmptyStates()
        fb.refreshState()
        for a, b in zip(solo, grp):
            assert a.getNumCamStates() == b.getNumCamStates(), k
    assert quiet > 0
    n_pruned = [len(a.getPrunedStates()["state_id"]) for a in solo]
    assert max(n_pruned) > 10

    def compare():
        for a, b in zip(solo, grp):
            assert a.counters() == b.counters()
            assert np.array_equal(a.getPrunedStates()["state_id"], b.getPrunedStates()["state_id"])
            assert np.array_equal(a.getMap(), b.getMap())
            assert np.array_equal(a.getCovariance(), b.getCovariance())
            sa, sb = a.getImuState(), b.getImuState()
            assert all(np.array_equal(sa[key], sb[key]) for key in sa)
            ca, cb = a.getCamStates(), b.getCamStates()
            assert all(np.array_equal(ca[key], cb[key]) for key in ca)

    compare()

    def finish(call):
        try:
            call()
            return True
        except RuntimeError as e:  # finish() after the last update's tracks lost clones: refused (test_shim_bookkeeping_cpu.py)
            assert "stale residualisation queue" in str(e)
            return False

    if all([finish(a.finish) for a in solo]):
        assert finish(fb.finish)
        compare()
    fb.close()
