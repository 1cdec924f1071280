"""The iterated mapped-landmark update on the device (msckf_b200_landmark_update / _batch_landmark_update with max_iter >= 2)
against the dense numpy IEKF of tests/landmark_iter_reference.py, at windows of 1-90 clones with truths drifted by 0.05, 0.3 and
1 m; max_iter 0 / 1 against the single linearisation bit for bit; the stationarity of the converged result; batch against
single calls bit for bit (mixed max_iter, early and late convergence, two chunks); calls that write nothing; the stop at an
iterate where a used landmark is behind the camera; no state hidden from copy_state; and the runner's relocalisation case."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from oracle.msckf_numpy import quat_mul, quat_to_rot
from tests.landmark_iter_reference import boxminus, boxplus, iekf, linearise, stationarity
from tests.test_aid_gpu import assert_unchanged, snapshot
from tests.test_batch_stream_gpu import Member
from tests.test_landmark_gpu import R_PIX, landmarks_in_front, project, state_of

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
WINDOWS = ((1, 1), (3, 2), (12, 3), (40, 4), (90, 5))
DRIFTS = (0.05, 0.3, 1.0)
# worst relative differences to the numpy IEKF of test_matches_numpy_iekf, measured on an H100 80GB HBM3 (700 W power limit);
# the bounds are 10 x these.  fp32: P and the state are rounded to float32 once.
MEASURED_REL = {"float32": {"P": 5.48e-8, "state": 3.75e-8, "nis": 3.22e-11},
                "float64": {"P": 1.01e-14, "state": 1.14e-12, "nis": 3.59e-11}}
MEASURED_STATIONARITY = 2.14e-8  # test_converged_result_is_stationary, same card
CONTRACT = {"float32": 1e-5, "float64": 1e-9}
KEYS = ("nis", "dx_norm", "dof", "rows", "used", "applied", "status", "iterations", "converged", "step")


def drifted_obs(rng, poses, clones, per, drift, noise=0.002):
    """observations of `per` landmarks from each clone in `clones`, made from truth poses that share a drift of `drift` m in
    position (and drift / 20 rad in yaw) against the estimate `poses`: clone [n], z [n, 2], p_L [n, 3]"""
    M = len(poses)
    e = np.zeros(15 + 6 * M)
    shared = np.concatenate([[0.0, 0.0, drift / 20], drift * np.array([0.8, -0.5, 0.3])])
    for k in range(M):
        e[15 + 6 * k:21 + 6 * k] = shared + rng.normal(size=6) * np.array([1e-3] * 3 + [1e-2] * 3)
    truth = boxplus(poses, e)
    clone, z, p_L = [], [], []
    for k in clones:
        pl = landmarks_in_front(rng, truth[k], per, depth=(3.0, 15.0))
        clone += [k] * per
        z.append(project(truth[k], pl)[1] + noise * rng.normal(size=(per, 2)))
        p_L.append(pl)
    return np.array(clone, np.int32), np.vstack(z), np.vstack(p_L)


def observed_clones(M):
    return sorted({0, M // 2, M - 1})


def full_state(imu, poses):
    return np.concatenate([imu[0:19], poses.ravel()])


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_linearisation_is_todays_call_bit_for_bit(dtype):
    rng = np.random.default_rng(41)
    for M, seed in WINDOWS:
        base = Member(dtype, M, seed=seed, max_clones=M + 2)
        _, poses = state_of(base.e)
        clone, z, p_L = drifted_obs(rng, poses, observed_clones(M), 6, 0.3)
        out = []
        for kw in ({}, {"max_iter": 0, "tol": 3.0}, {"max_iter": 1}, {"max_iter": 1, "tol": 1e-10}):
            t = base.twin(dtype, max_clones=M + 2)
            n0 = t.e.launch_count()
            r = t.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=0.0 if M < 12 else 40.0, **kw)
            assert t.e.launch_count() == n0
            out.append((r, t.snapshot()))
        r0, s0 = out[0]
        assert r0["applied"] == 1 and r0["iterations"] == 1 and r0["converged"] == 0 and r0["step"] == 0.0
        for r, s in out[1:]:
            for k in KEYS:
                assert r[k] == r0[k], (M, k)
            assert np.array_equal(r["gamma"], r0["gamma"]) and np.array_equal(r["flag"], r0["flag"])
            for x, y in zip(s, s0):
                assert np.array_equal(x, y), M


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_numpy_iekf(dtype):
    rng = np.random.default_rng(43)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0}
    for M, seed in WINDOWS:
        base = Member(dtype, M, seed=seed, max_clones=M + 2)
        for drift in DRIFTS:
            mem = base.twin(dtype, max_clones=M + 2)
            imu, poses = state_of(mem.e)
            P = mem.e.covariance().astype(np.float64)
            clone, z, p_L = drifted_obs(rng, poses, observed_clones(M), 8, drift)
            res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=10, tol=1e-10)
            ref = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=10, tol=1e-10)
            assert res["applied"] == 1 and res["status"] == 0 and res["used"] == ref["used"] and res["dof"] == ref["dof"]
            assert (res["iterations"], res["converged"]) == (ref["iterations"], ref["converged"]), (M, drift, res, ref["step"])
            assert np.array_equal(res["flag"], ref["flag"])
            if drift >= 0.3:
                assert ref["iterations"] >= 3, (M, drift)
            Pd = mem.e.covariance()
            assert np.array_equal(Pd, Pd.T)
            imud, posesd = state_of(mem.e)
            sd, sr = full_state(imud, posesd), full_state(ref["imu"], ref["poses"])
            rel = {"P": np.abs(Pd.astype(np.float64) - ref["P"]).max() / np.abs(ref["P"]).max(),
                   "state": np.abs(sd - sr).max() / np.abs(sr).max(),
                   "nis": abs(res["nis"] - ref["nis"]) / ref["nis"]}
            for k, v in rel.items():
                assert v <= CONTRACT[name], (M, drift, k, v)
                worst[k] = max(worst[k], v)
    print(f"landmark iekf rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 10 * MEASURED_REL[name][k], (k, v)


def _delta(imu0, poses0, imu1, poses1):
    """the applied error state: x1 = x0 [+] delta (IMU quaternion not renormalised, as the injection)"""
    n = 15 + 6 * len(poses0)
    d = np.zeros(n)
    q0 = imu0[15:19]
    qe = quat_mul(imu1[15:19], np.array([-q0[0], -q0[1], -q0[2], q0[3]]) / (q0 @ q0))
    d[0:3] = -2.0 * qe[0:3] * np.sign(qe[3])
    d[3:6] = imu1[6:9] - imu0[6:9]
    d[6:9] = imu1[3:6] - imu0[3:6]
    d[9:12] = imu1[9:12] - imu0[9:12]
    d[12:15] = imu1[0:3] - imu0[0:3]
    d[15:] = boxminus(poses1, poses0)
    return d


def test_converged_result_is_stationary():
    rng = np.random.default_rng(47)
    worst = 0.0
    for M, seed in WINDOWS[1:4]:
        mem = Member(np.float64, M, seed=seed, max_clones=M + 2)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance()
        clone, z, p_L = drifted_obs(rng, poses, observed_clones(M), 8, 1.0)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=16, tol=1e-12)
        assert res["converged"] == 1 and res["step"] <= 1e-12, res
        imud, posesd = state_of(mem.e)
        d = _delta(imu, poses, imud, posesd)
        H, r = linearise(P.shape[0], posesd, clone, z, p_L, res["flag"] == 0)
        s = stationarity(P, H, r, np.kron(np.eye(len(r) // 2), R_PIX), d)
        worst = max(worst, s)
    print(f"stationarity of the converged device result: {worst:.3e}")
    assert worst <= 10 * MEASURED_STATIONARITY


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [3, 12, 30, 90]
    rng = np.random.default_rng(53)
    mem = [Member(dtype, Ms[i % 4], seed=120 + i, max_clones=Ms[i % 4] + 2) for i in range(35)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    specs = []
    for i, m in enumerate(mem):
        if i % 11 == 5:
            specs.append(None)
            continue
        M = m.e.num_clones()
        _, poses = state_of(m.e)
        clone, z, p_L = drifted_obs(rng, poses, sorted({0, (i * 7) % M, M - 1}), 1 + i % 6, (0.05, 0.3, 1.0)[i % 3])
        specs.append({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX if i % 2 else None, "chi2_obs": 0.0,
                      "max_iter": (0, 1, 2, 4, 10, 16)[i % 6], "tol": (1e-10, 1e-6, 0.0)[i % 3]})
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], max_iter=s["max_iter"], tol=s["tol"])
              for t, s in zip(twins, specs)]
    its = {r["iterations"] for r in single if r is not None}
    assert min(its) == 1 and max(its) >= 4, its  # early and late convergence in one batch
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        for key in KEYS:
            assert got[i][key] == single[i][key], (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"]) and np.array_equal(got[i]["flag"], single[i]["flag"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


def test_calls_that_write_nothing():
    rng = np.random.default_rng(59)
    mem = [Member(np.float64, 4, seed=60 + i) for i in range(3)]
    lib = capi.lib()
    _, poses = state_of(mem[0].e)
    clone, z, p_L = drifted_obs(rng, poses, [0, 2], 3, 0.3)
    good = {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX, "max_iter": 8, "tol": 1e-10}
    before = [snapshot(m.e) for m in mem]
    sentinel = capi.LandmarkResult(7.0, 7.0, 7, 7, 7, 7, 7, 7, 7, 7.0)
    for spec in (dict(good, max_iter=-1), dict(good, max_iter=17), dict(good, tol=np.nan), dict(good, tol=-1e-3),
                 dict(good, tol=np.inf), {"clone": [], "max_iter": 17}):
        a, keep = capi.landmark_struct({"clone": [], "z": [], "p_L": []} if not len(spec["clone"]) else spec)
        if not len(spec["clone"]):
            a.max_iter = spec["max_iter"]
        out = capi.LandmarkResult.from_buffer_copy(sentinel)
        assert lib.msckf_b200_landmark_update(mem[0].e.h, C.byref(a), C.byref(out)) == -3, spec
        assert out.as_dict() == sentinel.as_dict()
    assert_unchanged(snapshot(mem[0].e), before[0])
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.landmark_update([good, dict(good, max_iter=17), good])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.landmark_update([good, None, dict(good, tol=np.nan)])
    # an un-fetched update (a triangulation of one track) on member 1
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.landmark_update([good, good, good])
    a, keep = capi.landmark_struct(good)
    out = capi.LandmarkResult.from_buffer_copy(sentinel)
    assert lib.msckf_b200_landmark_update(mem[1].e.h, C.byref(a), C.byref(out)) == -5 and out.as_dict() == sentinel.as_dict()
    mem[1].e.fetch(1)
    batch.close()
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stop_when_a_used_landmark_goes_behind_the_camera(dtype):
    """clone j is seen from a truth 1 m ahead along its optical axis, so the first step moves it about 1 m forward; one more
    landmark on its axis 0.4 m ahead (zero residual, used at linearisation 0) is behind the camera at that iterate"""
    M, j = 6, 3
    base = Member(dtype, M, seed=7, max_clones=M + 2)
    imu, poses = state_of(base.e)
    rng = np.random.default_rng(61)
    Cj = quat_to_rot(poses[j, 3:7])
    tpose = poses[j].copy()
    tpose[0:3] += Cj.T @ np.array([0.0, 0.0, 1.0])
    pl = landmarks_in_front(rng, tpose, 12, depth=(3.0, 15.0))
    z = project(tpose, pl)[1] + 0.001 * rng.normal(size=(12, 2))
    p_near = poses[j, 0:3] + Cj.T @ np.array([0.0, 0.0, 0.4])
    clone = np.full(13, j, np.int32)
    z = np.vstack([z, [[0.0, 0.0]]])
    p_L = np.vstack([pl, p_near])
    P = base.e.covariance().astype(np.float64)
    ref = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=8)
    assert ref["iterations"] == 1 and ref["converged"] == 0 and np.all(ref["flag"] == 0)
    assert project(boxplus(poses, ref["dx"])[j], p_near)[0][0, 2] < 0  # behind at the first iterate
    one, it = base.twin(dtype), base.twin(dtype)
    r1 = one.e.landmark_update(clone, z, p_L, R=R_PIX)
    r8 = it.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=8)
    assert r8["iterations"] == 1 and r8["converged"] == 0 and r8["applied"] == 1 and r8["step"] > 0.5
    for k in ("nis", "dx_norm", "dof", "rows", "used", "applied", "status"):
        assert r8[k] == r1[k], k
    for x, y in zip(it.snapshot(), one.snapshot()):  # the first linearisation, applied: today's update bit for bit
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dtype", DTYPES)
def test_no_hidden_iterate_state(dtype):
    rng = np.random.default_rng(67)
    base = Member(dtype, 8, seed=9, max_clones=10)
    a = base.twin(dtype, max_clones=10)
    _, poses = state_of(a.e)
    clone, z, p_L = drifted_obs(rng, poses, [1, 7], 6, 1.0)
    assert a.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=10)["iterations"] > 2
    b = Member(dtype, 0, seed=0, max_clones=10, twin_of=a)
    c = Member(dtype, 0, seed=0, max_clones=10, twin_of=a)
    _, poses = state_of(b.e)
    clone, z, p_L = drifted_obs(rng, poses, [0, 3, 7], 5, 0.3)
    ra = a.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=6, tol=1e-8)
    rb = b.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=6, tol=1e-8)
    batch = capi.Batch([c.e])
    rc = batch.landmark_update([{"clone": clone, "z": z, "p_L": p_L, "R": R_PIX, "max_iter": 6, "tol": 1e-8}])[0]
    batch.close()
    for r in (rb, rc):
        for k in KEYS:
            assert r[k] == ra[k], k
    for m in (b, c):
        for x, y in zip(m.snapshot(), a.snapshot()):
            assert np.array_equal(x, y)


def test_runner_relocalisation():
    truth = mc.make_truth(n_frames=50, seq=8)
    out = {}
    for it in (1, 8):
        rec, _ = mc.run(range(8), truth, dtype=np.float64, map_every=1, map_start=40, map_iterations=it)
        s = mc.summarize(rec)
        f = s["map_first"]
        assert f["frame"] == 40 and len(s["map"]["anis"]) == 10 and np.isfinite(f["imu_anees"])
        assert f["iterations"] >= (1 if it == 1 else 2) and f["pos_rmse_after"] < f["pos_rmse_before"]
        out[it] = f
    print("runner relocalisation at frame 40: " + "; ".join(
        f"max_iter {k}: position RMSE {v['pos_rmse_before']:.3f} -> {v['pos_rmse_after']:.3f} m, ANIS {v['anis']:.1f} for "
        f"{v['mean_dof']:.1f} dof, IMU ANEES {v['imu_anees']:.2f}, {v['iterations']:.2f} linearisations" for k, v in out.items()))
