"""NEES on the device (msckf_b200_nees / _batch_nees, MSCKF::nees, MSCKFBatch::nees) against numpy on the fetched covariance,
against the Monte-Carlo runner's sampled initial error, batch against single calls, and the call's read-only contract."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, engine_filter, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
KEYS = ("orientation", "position", "pose", "imu", "full")
# worst relative difference to numpy of test_known_perturbation_matches_numpy, measured on an H100 80GB HBM3 (fp64 NEES of
# fp64 inputs: the engine's float32 P widens exactly, so both dtypes compare fp64 arithmetic); bounds are 10 x these
MEASURED_REL = {"float32": 1.354e-15, "float64": 1.332e-15}


def est_of(e):
    imu, poses = e.state()
    return {"imu": np.concatenate([imu[0:15], imu[15:19]]).astype(np.float64), "poses": poses.astype(np.float64)}


def numpy_nees(P, err, full):
    out = {}
    for c, idx in mc.BLOCK.items():
        eb = err[idx]
        out[c] = float(eb @ np.linalg.solve(P[np.ix_(idx, idx)], eb))
    out["full"] = float(err @ np.linalg.solve(P, err)) if full else float("nan")
    return out


def as_row(r):
    return np.array([r[k] for k in KEYS] + [r["dim_full"], r["first_bad_pivot"]], dtype=np.float64)


@pytest.mark.parametrize("dtype", DTYPES)
def test_truth_equal_to_estimate_gives_zero(dtype):
    for M in (0, 4):
        m = Member(dtype, M, seed=3 + M)
        est = est_of(m.e)
        r = m.e.nees(est["imu"], est["poses"])
        assert r["dim_full"] == 15 + 6 * M and r["first_bad_pivot"] == -1
        for k in KEYS:
            assert 0.0 <= r[k] < 1e-20, (k, r[k])


@pytest.mark.parametrize("dtype", DTYPES)
def test_known_perturbation_matches_numpy(dtype):
    rng = np.random.default_rng(11)
    worst = 0.0
    for M, seed in ((0, 1), (3, 2), (12, 3), (40, 4)):
        m = Member(dtype, M, seed=seed)
        est = est_of(m.e)
        n = 15 + 6 * M
        truth = mc.perturb(est, 0.05 * rng.standard_normal(n))
        err = mc.error_state(truth, est)
        P = m.e.covariance().astype(np.float64)
        ref = numpy_nees(P, err, True)
        for poses in (truth["poses"], None):
            r = m.e.nees(truth["imu"], poses)
            assert r["first_bad_pivot"] == -1 and r["dim_full"] == (n if poses is not None else 0)
            for k in KEYS:
                if k == "full" and poses is None:
                    assert np.isnan(r[k])
                    continue
                rel = abs(r[k] - ref[k]) / ref[k]
                assert rel <= 1e-9, (M, k, r[k], ref[k])
                worst = max(worst, rel)
    print(f"nees rel vs numpy {np.dtype(dtype).name}: {worst:.3e}")
    assert worst <= 10 * MEASURED_REL[np.dtype(dtype).name]


@pytest.mark.parametrize("dtype", DTYPES)
def test_initial_nees_equals_the_runners_sampled_error(dtype):
    truth = mc.make_truth(n_frames=2, seq=8)
    P0 = np.asarray(truth["noise"]["initial_imu_covar"], dtype=np.float64)
    t0 = mc.imu_vector(truth["imu_state"])
    for k in (0, 5):
        tr = mc.make_trial(truth, k)
        f = engine_filter(dtype)
        f.initialize(truth["camera"], truth["noise"], truth["params"], tr["imu_state"])
        r = f.nees(t0)
        if dtype == np.float64:
            e0 = tr["e0"]
        else:  # the filter holds the float32-rounded initial estimate and covariance
            est = {"imu": np.asarray(mc.imu_vector(tr["imu_state"]), dtype=np.float32).astype(np.float64), "poses": None}
            e0 = mc.error_state({"imu": t0, "poses": None}, est)
            P0 = np.asarray(truth["noise"]["initial_imu_covar"], dtype=np.float32).astype(np.float64)
        want = float(e0 @ np.linalg.solve(P0, e0))
        assert abs(r["imu"] - want) <= 1e-9 * want, (k, r["imu"], want)
        assert np.isnan(r["full"]) and r["dim_full"] == 0
        f.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(4)
    mem = [Member(dtype, Ms[i % 4], seed=40 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    truths = []
    for i, m in enumerate(mem):
        est = est_of(m.e)
        t = mc.perturb(est, 0.02 * rng.standard_normal(15 + 6 * m.e.num_clones()))
        truths.append((t["imu"], None if i % 3 == 0 else t["poses"]))
    single = [as_row(m.e.nees(*t)) for m, t in zip(mem, truths)]
    batch = capi.Batch([m.e for m in mem])
    got = [as_row(r) for r in batch.nees([t[0] for t in truths], [t[1] for t in truths])]
    for i, (a, b) in enumerate(zip(single, got)):
        assert np.array_equal(a, b, equal_nan=True), (i, a, b)
        assert np.isnan(a[4]) == (i % 3 == 0)
    assert all(np.isfinite(a[:4]).all() for a in single)
    batch.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_indefinite_covariance_reports_the_first_bad_pivot(dtype):
    rng = np.random.default_rng(9)
    mem = [Member(dtype, 5, seed=60 + i) for i in range(3)]
    truths = []
    for m in mem:
        est = est_of(m.e)
        t = mc.perturb(est, 0.02 * rng.standard_normal(45))
        truths.append((t, est))
    before = [m.e.nees(t["imu"], t["poses"]) for m, (t, _) in zip(mem, truths)]
    P = mem[1].e.covariance()
    P[27, 27] = -1.0  # a clone's diagonal: permuted index 27
    mem[1].e.set_covariance(P)
    batch = capi.Batch([m.e for m in mem])
    res = batch.nees([t["imu"] for t, _ in truths], [t["poses"] for t, _ in truths])
    r = res[1]
    assert 15 <= r["first_bad_pivot"] <= 27 and np.isnan(r["full"])
    ref = numpy_nees(P.astype(np.float64), mc.error_state(*truths[1]), False)
    for k in ("orientation", "position", "pose", "imu"):
        assert np.isfinite(r[k]) and abs(r[k] - ref[k]) <= 1e-9 * ref[k], (k, r[k], ref[k])
    for i in (0, 2):
        assert np.array_equal(as_row(res[i]), as_row(before[i]), equal_nan=True)
        assert res[i]["first_bad_pivot"] == -1
    assert mem[1].e.nees(truths[1][0]["imu"], truths[1][0]["poses"])["first_bad_pivot"] == r["first_bad_pivot"]
    batch.close()


def _stream(dtype, with_nees):
    wls = [synth.make_stream_workload(n_frames=40, seq=s, max_features=40, max_track_length=20, max_cam_states=15) for s in (3, 4, 5, 6)]
    truth = mc.make_truth(n_frames=40, seq=3, max_features=40, max_track_length=20, max_cam_states=15)
    fs = [engine_filter(dtype) for _ in wls]
    for f, wl in zip(fs, wls):
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    fb = FilterBatch(fs)
    for k in range(40):
        frs = [wl["frames"][k] for wl in wls]
        for i, fr in enumerate(frs):
            for (w, a, dT) in fr["imu"]:
                fb.propagate(i, w, a, dT)
        fb.augmentState([fr["state_id"] for fr in frs], [fr["time"] for fr in frs])
        for f, fr in zip(fs, frs):
            f.update(*fr["update"])
            f.addFeatures(*fr["add"])
        fb.marginalize()
        fb.pruneEmptyStates()
        if with_nees:
            res = fb.nees([truth["truth_imu"][k]] * 4, [truth["truth_pose"][f.getCamStates()["state_id"]] for f in fs])
            assert all(np.isfinite(r["imu"]) for r in res)
            fs[0].nees(truth["truth_imu"][k])  # (single-filter form, through the C view)
    fb.close()
    launches = [capi.Engine(dtype, borrowed=f.engineHandle()).launch_count() for f in fs]
    out = [(f.getCovariance(), np.concatenate(list(f.getImuState().values())), np.hstack([f.getCamStates()["p_C_G"], f.getCamStates()["q_CG"]]))
           for f in fs]
    return out, launches


@pytest.mark.parametrize("dtype", DTYPES)
def test_nees_is_read_only(dtype):
    a, la = _stream(dtype, False)
    b, lb = _stream(dtype, True)
    assert la == lb
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert u.shape == v.shape and np.array_equal(u, v)


def test_argument_and_state_errors_write_nothing():
    mem = [Member(np.float64, 4, seed=80 + i) for i in range(3)]
    ests = [est_of(m.e) for m in mem]
    lib = capi.lib()
    sentinel = capi.NeesResult(7.0, 7.0, 7.0, 7.0, 7.0, 7, 7)

    def call_single(e, imu, poses):
        out = capi.NeesResult.from_buffer_copy(sentinel)
        rc = lib.msckf_b200_nees(e.h, None if imu is None else C.c_void_p(imu.ctypes.data),
                                 None if poses is None else C.c_void_p(poses.ctypes.data), C.byref(out))
        return rc, out.as_dict()

    good = ests[0]["imu"].copy()
    bad_nan = good.copy(); bad_nan[4] = np.nan
    bad_q = good.copy(); bad_q[15:19] = 0.0
    bad_pose = ests[0]["poses"].copy(); bad_pose[2, 3:7] = 0.0
    for imu, poses in ((None, None), (bad_nan, None), (bad_q, None), (good, bad_pose)):
        rc, out = call_single(mem[0].e, imu, poses)
        assert rc == -3 and out == sentinel.as_dict()
    rc = lib.msckf_b200_nees(mem[0].e.h, C.c_void_p(good.ctypes.data), None, None)
    assert rc == -3
    batch = capi.Batch([m.e for m in mem])
    outs = (capi.NeesResult * 3)(*[capi.NeesResult.from_buffer_copy(sentinel) for _ in range(3)])
    imus = (C.c_void_p * 3)(ests[0]["imu"].ctypes.data, None, ests[2]["imu"].ctypes.data)
    assert lib.msckf_b200_batch_nees(batch.h, imus, None, outs) == -3
    assert all(o.as_dict() == sentinel.as_dict() for o in outs)
    assert lib.msckf_b200_batch_nees(batch.h, None, None, outs) == -3
    # an un-fetched update (a triangulation of one track) on member 1
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    imus = (C.c_void_p * 3)(*[e["imu"].ctypes.data for e in ests])
    assert lib.msckf_b200_batch_nees(batch.h, imus, None, outs) == -5
    assert all(o.as_dict() == sentinel.as_dict() for o in outs)
    rc, out = call_single(mem[1].e, ests[1]["imu"], None)
    assert rc == -5 and out == sentinel.as_dict()
    mem[1].e.fetch(1)
    assert np.isfinite(batch.nees([e["imu"] for e in ests])[1]["imu"])
    batch.close()


def test_runner_smoke_and_trial_alone_is_bit_identical():
    truth = mc.make_truth(n_frames=60, seq=8)
    records, final = mc.run(range(8), truth, dtype=np.float64)
    for k, rec in records.items():
        for c in ("orientation", "position", "pose", "imu"):
            assert np.all(np.isfinite(rec["nees"][c])), (k, c)
        # the whole state right after a frame's update: the newest clone is still a copy of the IMU pose (no propagation since
        # its augmentation), so P is singular there and the factorisation stops inside that clone's block
        for v, d, bad in zip(rec["nees"]["full"], rec["dim"]["full"], rec["first_bad_pivot"]):
            assert np.isfinite(v) or d - 6 <= bad < d, (k, d, bad)
    s = mc.summarize(records)
    for c in KEYS:
        v = s["components"][c]
        assert len(v["anees"]) == 60 and len(v["lower"]) == 60 and 0.0 <= v["frames_inside"] <= 1.0
        print(f"ANEES {c}: {v['mean_anees']:.3f} (mean dof {v['mean_dof']:.1f}), frames inside 95 % bounds {v['frames_inside']:.2f}")
    assert len(s["pos_rmse"]) == 60 and np.isfinite(s["pos_rmse_run"])
    rec3, fin3 = mc.run([3], truth, dtype=np.float64)
    for c in KEYS:  # (NaN != NaN: compared as arrays)
        assert np.array_equal(rec3[3]["nees"][c], records[3]["nees"][c], equal_nan=True), c
    assert rec3[3]["pos_err2"] == records[3]["pos_err2"] and rec3[3]["first_bad_pivot"] == records[3]["first_bad_pivot"]
    for x, y in zip(fin3[3], final[3]):
        assert np.array_equal(x, y)
