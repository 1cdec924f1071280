"""Aided measurement updates on the device (msckf_b200_aid_update / _batch_aid_update, MSCKF::aidedUpdate,
MSCKFBatch::aidedUpdate) against numpy fp64 on the fetched covariance and state: the Joseph-form covariance, the state
injection of oracle/msckf_numpy.py and the NIS.  Also: a caller-linearised selection against the built-in models, batch
against single calls bit for bit, updates that must write nothing, no state hidden from copy_state, and the runner's fixes."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from oracle.msckf_numpy import MSCKF as NumpyMSCKF, quat_mul, quat_normalized
from tests.parity_cases import make_engine
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
MODELS = (capi.AID_VELOCITY, capi.AID_POSITION, capi.AID_POSE, capi.AID_CLONE_POSE, capi.AID_LINEAR)
# worst relative differences to numpy of test_models_match_numpy, measured on an H100 80GB HBM3 (700 W power limit); the
# bounds are 10 x these.  fp32: P and the state are rounded to float32 once; the NIS is fp64 arithmetic on the widened P.
MEASURED_REL = {"float32": {"P": 5.44e-8, "state": 2.14e-8, "nis": 2.65e-15},
                "float64": {"P": 1.26e-14, "state": 1.80e-16, "nis": 5.29e-15}}
CONTRACT = {"float32": 1e-5, "float64": 1e-9}  # outright bounds: fp64 arithmetic, rounded to the filter's type once


def state_of(e):
    """(imu [29] fp64, poses [M, 7] fp64) of an engine"""
    imu, poses = e.state()
    return imu.astype(np.float64), poses.astype(np.float64)


def rows_of(model, clone=0):
    if model == capi.AID_VELOCITY:
        return [6, 7, 8]
    if model == capi.AID_POSITION:
        return [12, 13, 14]
    if model == capi.AID_POSE:
        return [0, 1, 2, 12, 13, 14]
    return list(range(15 + 6 * clone, 21 + 6 * clone))


def spd(rng, m, scale):
    B = rng.normal(size=(m, m))
    return scale * (B @ B.T / m + 0.5 * np.eye(m))


def make_spec(rng, model, imu, poses, n, clone=0, m=5):
    """a measurement near the current estimate: its dict for aid_struct, and (H, r) of the same measurement in numpy"""
    if model == capi.AID_LINEAR:
        H = rng.normal(size=(m, n)) / np.sqrt(n)
        r = 0.1 * rng.normal(size=m)
        return {"model": model, "z": r, "R": spd(rng, m, 0.05), "H": H}, H, r
    if model in (capi.AID_VELOCITY, capi.AID_POSITION):
        est = imu[3:6] if model == capi.AID_VELOCITY else imu[0:3]
        z = est + 0.1 * rng.normal(size=3)
        r = z - est
    else:
        p_est, q_est = (imu[0:3], imu[15:19]) if model == capi.AID_POSE else (poses[clone, 0:3], poses[clone, 3:7])
        q = quat_mul(mc.quat_of_error(0.05 * rng.normal(size=3)), q_est)
        z = np.concatenate([p_est + 0.1 * rng.normal(size=3), q / np.linalg.norm(q)])
        r = np.concatenate([mc.quat_error(z[3:7], q_est), z[0:3] - p_est])
    rows = rows_of(model, clone)
    H = np.zeros((len(r), n))
    H[np.arange(len(r)), rows] = 1.0
    return {"model": model, "z": z, "R": spd(rng, len(r), 0.02), "clone": clone}, H, r


def numpy_update(P, imu, poses, H, r, R):
    """Joseph form, injection of oracle/msckf_numpy.py (msckf.h:1373-1391), NIS; all fp64"""
    S = H @ P @ H.T + R
    K = np.linalg.solve(S, H @ P).T
    dx = K @ r
    A = np.eye(P.shape[0]) - K @ H
    Pn = A @ P @ A.T + K @ R @ K.T
    buq = lambda d: NumpyMSCKF._build_update_quat(SimpleNamespace(S=np.float64, dt=np.float64), d)  # noqa: E731
    imu, poses = imu.copy(), poses.copy()
    imu[15:19] = quat_mul(buq(dx[0:3]), imu[15:19])  # not renormalised
    imu[6:9] += dx[3:6]; imu[3:6] += dx[6:9]; imu[9:12] += dx[9:12]; imu[0:3] += dx[12:15]
    for k in range(len(poses)):
        poses[k, 3:7] = quat_normalized(quat_mul(buq(dx[15 + 6 * k:18 + 6 * k]), poses[k, 3:7]))
        poses[k, 0:3] += dx[18 + 6 * k:21 + 6 * k]
    return Pn, imu, poses, float(r @ np.linalg.solve(S, r)), float(np.linalg.norm(dx))


def call(e, spec):
    return e.aid_update(spec["model"], spec["z"], spec["R"], H=spec.get("H"), clone=spec.get("clone", 0), chi2_max=spec.get("chi2_max", 0.0))


def snapshot(e):
    imu, poses = e.state()
    return imu, poses, e.covariance(), e.launch_count()


def assert_unchanged(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dtype", DTYPES)
def test_models_match_numpy(dtype):
    rng = np.random.default_rng(21)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0}
    for M, seed in ((0, 1), (3, 2), (12, 3), (40, 4)):
        base = Member(dtype, M, seed=seed)
        n = 15 + 6 * M
        cases = [(m, 0, 5) for m in MODELS if m != capi.AID_CLONE_POSE] + [(capi.AID_LINEAR, 0, 32)]
        if M > 0:
            cases += [(capi.AID_CLONE_POSE, 0, 0), (capi.AID_CLONE_POSE, M - 1, 0)]
        for model, clone, m in cases:
            mem = base.twin(dtype)
            imu, poses = state_of(mem.e)
            P = mem.e.covariance().astype(np.float64)
            spec, H, r = make_spec(rng, model, imu, poses, n, clone, m)
            res = call(mem.e, spec)
            Pr, imur, posesr, nisr, dxr = numpy_update(P, imu, poses, H, r, spec["R"])
            Pd = mem.e.covariance()
            assert np.array_equal(Pd, Pd.T)  # both halves written from one value
            imud, posesd = state_of(mem.e)
            assert np.array_equal(imud[19:29], imu[19:29])  # the observability copies are not touched
            assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == len(r)
            sd = np.concatenate([imud[0:19], posesd.ravel()])
            sr = np.concatenate([imur[0:19], posesr.ravel()])
            rel = {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(),
                   "state": np.abs(sd - sr).max() / np.abs(sr).max(),
                   "nis": abs(res["nis"] - nisr) / nisr}
            assert abs(res["dx_norm"] - dxr) <= 1e-9 * dxr, (M, model)
            for k, v in rel.items():
                assert v <= CONTRACT[name], (M, model, clone, m, k, v)
                worst[k] = max(worst[k], v)
    print(f"aid rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 10 * MEASURED_REL[name][k], (k, v)


@pytest.mark.parametrize("dtype", DTYPES)
def test_linear_selection_equals_the_built_in_models(dtype):
    rng = np.random.default_rng(5)
    M = 12
    base = Member(dtype, M, seed=7)
    n = 15 + 6 * M
    for model, clone in ((capi.AID_VELOCITY, 0), (capi.AID_POSITION, 0), (capi.AID_POSE, 0), (capi.AID_CLONE_POSE, 4)):
        a, b = base.twin(dtype), base.twin(dtype)
        imu, poses = state_of(a.e)
        spec, H, r = make_spec(rng, model, imu, poses, n, clone)
        ra = call(a.e, spec)
        rb = call(b.e, {"model": capi.AID_LINEAR, "z": r, "R": spec["R"], "H": H})
        # P does not depend on r: bit for bit for every model
        assert np.array_equal(a.e.covariance(), b.e.covariance()), model
        sa, sb = a.e.state(), b.e.state()
        if model in (capi.AID_VELOCITY, capi.AID_POSITION):  # z - x in fp64 on both sides: the same residual bits
            assert ra == rb and all(np.array_equal(x, y) for x, y in zip(sa, sb)), model
        else:  # the host's dtheta may differ from the device's in the last bits
            assert abs(ra["nis"] - rb["nis"]) <= 1e-9 * ra["nis"]
            for x, y in zip(sa, sb):
                assert np.abs(x.astype(np.float64) - y).max() <= (1e-6 if dtype == np.float32 else 1e-12) * max(1.0, np.abs(x).max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(8)
    mem = [Member(dtype, Ms[i % 4], seed=90 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    specs = []
    for i, m in enumerate(mem):
        M = m.e.num_clones()
        model = [capi.AID_POSITION, capi.AID_POSE, capi.AID_CLONE_POSE, capi.AID_LINEAR, capi.AID_VELOCITY, -1][i % 6]
        if model == capi.AID_CLONE_POSE and M == 0:
            model = capi.AID_POSITION
        if model < 0:
            specs.append(None)
            continue
        imu, poses = state_of(m.e)
        specs.append(make_spec(rng, model, imu, poses, 15 + 6 * M, clone=M // 2, m=1 + i % 32)[0])
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else call(t.e, s) for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.aid_update(specs)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        assert got[i] == single[i] and got[i]["applied"] == 1, i
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


def test_updates_that_write_nothing():
    rng = np.random.default_rng(13)
    mem = [Member(np.float64, 4, seed=30 + i) for i in range(3)]
    lib = capi.lib()
    n = 15 + 6 * 4
    imu, poses = state_of(mem[0].e)
    good = make_spec(rng, capi.AID_POSE, imu, poses, n)[0]
    before = [snapshot(m.e) for m in mem]
    # gated out: NIS reported, nothing applied
    r = call(mem[0].e, dict(good, chi2_max=1e-12))
    assert r["applied"] == 0 and r["status"] == 0 and r["nis"] > 1e-12 and r["dx_norm"] == 0.0
    # S not positive definite
    r = call(mem[0].e, dict(good, R=-1e6 * np.eye(6)))
    assert r["status"] == 1 and r["applied"] == 0 and np.isnan(r["nis"])
    assert_unchanged(snapshot(mem[0].e), before[0])
    sentinel = capi.AidResult(7.0, 7.0, 7, 7, 7)

    def raw(e, a):
        out = capi.AidResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_aid_update(e.h, C.byref(a), C.byref(out)), out

    q0 = np.r_[imu[0:3], 0.0, 0.0, 0.0, 0.0]
    nan3 = np.array([0.0, np.nan, 0.0])
    R_upper_nan = np.eye(6); R_upper_nan[0, 5] = np.nan  # (only the lower triangle is read: valid)
    R_lower_nan = np.eye(6); R_lower_nan[5, 0] = np.nan
    H = np.ones((2, n))
    bad = [dict(model=9, z=imu[0:3], R=np.eye(3)), dict(model=capi.AID_CLONE_POSE, clone=4, z=good["z"], R=np.eye(6)),
           dict(model=capi.AID_POSITION, z=nan3, R=np.eye(3)), dict(model=capi.AID_POSE, z=q0, R=np.eye(6)),
           dict(model=capi.AID_POSE, z=good["z"], R=R_lower_nan), dict(model=capi.AID_LINEAR, z=[0.1, 0.2], R=np.eye(2), H=H[:, :-6]),
           dict(model=capi.AID_LINEAR, z=np.zeros(33), R=np.eye(33), H=np.zeros((33, n)))]
    keep = []
    for spec in bad:
        a, k = capi.aid_struct(spec)
        keep.append(k)
        rc, out = raw(mem[0].e, a)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), spec
    a, k = capi.aid_struct(dict(model=capi.AID_POSITION, z=imu[0:3], R=np.eye(3)))
    a.m = 6  # m of a built-in model: 0 or its own
    assert raw(mem[0].e, a)[0] == -3
    a.m, a.R = 3, None
    assert raw(mem[0].e, a)[0] == -3
    assert call(mem[0].e, dict(good, R=R_upper_nan))["applied"] == 1  # (the upper triangle is not read)
    before[0] = snapshot(mem[0].e)
    # a batch with one bad member changes no member
    batch = capi.Batch([m.e for m in mem])
    specs = [good, dict(model=capi.AID_POSITION, z=nan3, R=np.eye(3)), good]
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_update(specs)
    # an un-fetched update (a triangulation of one track) on member 1
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    launched = mem[1].e.launch_count()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.aid_update([good, None, good])
    a, k = capi.aid_struct(good)
    rc, out = raw(mem[1].e, a)
    assert rc == -5 and out.as_dict() == sentinel.as_dict()
    assert mem[1].e.launch_count() == launched
    mem[1].e.fetch(1)  # (a triangulation writes neither P nor the state)
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)
    batch.close()


def test_non_finite_covariance_is_reported_and_applied():
    mem = Member(np.float64, 4, seed=3)
    P = mem.e.covariance()
    P[30, 30] = np.inf  # outside the rows a position fix reads: only the downdate meets it
    mem.e.set_covariance(P)
    imu, _ = state_of(mem.e)
    with pytest.raises(RuntimeError, match="rc=-6"):
        mem.e.aid_update(capi.AID_POSITION, imu[0:3] + 0.1, 0.01 * np.eye(3))
    assert not np.array_equal(state_of(mem.e)[0], imu)  # applied, like the vision update's ERR_NUMERIC


def _stream(dtype, n_frames, aid_at):
    """two class filters on one stream; at frame aid_at filter A takes a pose fix, and B gets A's device state by copy_state"""
    wl = synth.make_stream_workload(n_frames=n_frames, seq=5, max_features=40, max_track_length=20, max_cam_states=15)
    fs = [make_engine(dtype) for _ in range(2)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    for k, fr in enumerate(wl["frames"]):
        for f in fs:
            for (w, a, dT) in fr["imu"]:
                f.propagate(w, a, dT)
            f.augmentState(fr["state_id"], fr["time"])
            f.update(*fr["update"])
            f.addFeatures(*fr["add"])
            f.marginalize()
            f.pruneEmptyStates()
        if k == aid_at:
            s = fs[0].getImuState()
            fs[0].aid_update(capi.AID_POSE, np.r_[s["p_I_G"] + 0.05, s["q_IG"]], 0.01 * np.eye(6))
            ea, eb = (capi.Engine(dtype, borrowed=f.engineHandle()) for f in fs)
            eb.copy_state_from(ea)
            assert np.array_equal(ea.covariance(), eb.covariance())
    out = [(f.getCovariance(), np.concatenate(list(f.getImuState().values())),
            np.hstack([f.getCamStates()["p_C_G"], f.getCamStates()["q_CG"]])) for f in fs]
    for f in fs:
        f.close()
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_no_hidden_state(dtype):
    a, b = _stream(dtype, 12, aid_at=6)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y)


def test_runner_with_position_fixes():
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, fix_every=10, fix_sigma=0.1)
    s = mc.summarize(rec)
    f = s["fixes"]
    assert len(f["anis"]) == 6 and all(np.isfinite(f["anis"]))
    for c in ("orientation", "position", "pose", "imu"):
        assert np.isfinite(s["components"][c]["mean_anees"]), c
    print(f"fixes: ANIS {f['mean_anis']:.3f} (3 dof, 95 % bounds [{f['lower']:.3f}, {f['upper']:.3f}]), fixes inside "
          f"{f['fixes_inside']:.2f}; ANEES imu {s['components']['imu']['mean_anees']:.3f}, position "
          f"{s['components']['position']['mean_anees']:.3f}; position RMSE {s['pos_rmse_run']:.4f} m")
    # until the first fix (after frame 9's prune) the trials are those of a run without fixes
    rec0, _ = mc.run(range(2), truth, dtype=np.float64)
    for k in range(2):
        for c in ("orientation", "position", "imu"):
            assert np.array_equal(rec0[k]["nees"][c][:9], rec[k]["nees"][c][:9]), (k, c)
        assert rec0[k]["nees"]["imu"][9] != rec[k]["nees"]["imu"][9]
