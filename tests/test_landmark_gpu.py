"""Mapped-landmark updates on the device (msckf_b200_landmark_update / _batch_landmark_update, MSCKF::landmarkUpdate,
MSCKFBatch::landmarkUpdate) against the dense, uncompressed stacked EKF in numpy fp64 on the fetched covariance and state
(Joseph form, the state injection of oracle/msckf_numpy.py, the NIS), against a central-difference Jacobian taken through that
injection, and against the caller-linearised aided update.  Also: batch against single calls bit for bit, calls that must write
nothing, ERR_NUMERIC, no state hidden from copy_state, and the runner's map updates."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from oracle.msckf_numpy import quat_to_rot
from tests.test_aid_gpu import numpy_update, snapshot, assert_unchanged
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
# worst relative differences to the dense numpy update of test_matches_dense_numpy, measured on an H100 80GB HBM3 (700 W power
# limit); the bounds are 10 x these.  fp32: P and the state are rounded to float32 once.
MEASURED_REL = {"float32": {"P": 5.54e-8, "state": 3.55e-8, "nis": 3.27e-11, "gamma": 5.48e-16},
                "float64": {"P": 1.46e-15, "state": 8.11e-13, "nis": 5.91e-11, "gamma": 4.85e-13}}
MEASURED_LINEAR = 1.33e-11  # fp64: landmark update against aid_update(LINEAR) (P, state, NIS), same card
CONTRACT = {"float32": 1e-5, "float64": 1e-9}


def state_of(e):
    imu, poses = e.state()
    return imu.astype(np.float64), poses.astype(np.float64)


def project(pose, p_L):
    """p_C and z^ of landmarks p_L [n, 3] from a clone pose (p_C_G, q_CG xyzw)"""
    C = quat_to_rot(pose[3:7])
    pc = (C @ (np.atleast_2d(p_L) - pose[0:3]).T).T
    return pc, pc[:, 0:2] / pc[:, 2:3]


def landmarks_in_front(rng, pose, n, depth=(2.0, 8.0)):
    """n landmark positions in G that clone `pose` sees at the given depth range"""
    d = rng.uniform(*depth, n)
    pc = np.stack([rng.uniform(-0.4, 0.4, n) * d, rng.uniform(-0.3, 0.3, n) * d, d], axis=1)
    C = quat_to_rot(pose[3:7])
    return (C.T @ pc.T).T + pose[0:3]


def jacobian(pose, p_L):
    """analytic 2 x 6 block [J [p_C]x, -J C] over the clone's [dtheta, dp] (msckf.h:929-936, no observability projection)"""
    C = quat_to_rot(pose[3:7])
    pc = C @ (p_L - pose[0:3])
    X, Y, Z = pc
    J = np.array([[1, 0, -X / Z], [0, 1, -Y / Z]]) / Z
    sk = np.array([[0, -Z, Y], [Z, 0, -X], [-Y, X, 0]])
    return np.hstack([J @ sk, -J @ C])


def dense(P, poses, clone, z, p_L, R, chi2=0.0, jac=None):
    """the uncompressed stacked system: (H, r, Rbig) of the used observations, gamma, flags"""
    n = P.shape[0]
    Hs, rs, gam, flag = [], [], [], []
    for k, zi, pl in zip(clone, z, p_L):
        pc, zh = project(poses[k], pl)
        if not (pc[0, 2] > 0 and np.all(np.isfinite(zh))):
            gam.append(np.nan); flag.append(2)
            continue
        r = zi - zh[0]
        H = np.zeros((2, n))
        H[:, 15 + 6 * k:21 + 6 * k] = jacobian(poses[k], pl) if jac is None else jac(k, pl)
        Pk = P[15 + 6 * k:21 + 6 * k, 15 + 6 * k:21 + 6 * k]
        A = H[:, 15 + 6 * k:21 + 6 * k]
        g = float(r @ np.linalg.solve(A @ Pk @ A.T + R, r))
        gam.append(g)
        f = 1 if (chi2 > 0 and g > chi2) else 0
        flag.append(f)
        if f == 0:
            Hs.append(H); rs.append(r)
    m = 2 * len(Hs)
    Hb = np.vstack(Hs) if Hs else np.zeros((0, n))
    rb = np.concatenate(rs) if rs else np.zeros(0)
    return Hb, rb, np.kron(np.eye(m // 2), R), np.array(gam), np.array(flag)


def rows_of(clone, flag):
    """rows of the compressed system: sum over clones of min(2 a_k, 6)"""
    used = np.bincount(np.asarray(clone)[np.asarray(flag) == 0], minlength=1)
    return int(np.minimum(2 * used, 6).sum())


def make_obs(rng, poses, counts, noise=0.003):
    """observations of clones (clone -> count), in shuffled input order: clone [n], z [n, 2], p_L [n, 3]"""
    clone = np.concatenate([np.full(c, k) for k, c in counts.items()]).astype(np.int32)
    rng.shuffle(clone)
    p_L = np.array([landmarks_in_front(rng, poses[k], 1)[0] for k in clone])
    z = np.array([project(poses[k], pl)[1][0] for k, pl in zip(clone, p_L)]) + noise * rng.normal(size=(len(clone), 2))
    return clone, z, p_L


R_PIX = np.array([[2.0e-5, 3.0e-6], [3.0e-6, 1.5e-5]])


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_dense_numpy(dtype):
    rng = np.random.default_rng(31)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0, "gamma": 0.0}
    for M, seed in ((1, 1), (3, 2), (12, 3), (40, 4), (90, 5)):
        base = Member(dtype, M, seed=seed, max_clones=M + 2)
        mem = base.twin(dtype, max_clones=M + 2)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        counts = {0: 1}
        if M >= 3:
            counts.update({1: 2, M - 1: 3})
        if M >= 12:
            counts.update({5: 256, 7: 1})
        clone, z, p_L = make_obs(rng, poses, counts)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX)
        H, r, Rb, gam, flag = dense(P, poses, clone, z, p_L, R_PIX)
        Pr, imur, posesr, nisr, dxr = numpy_update(P, imu, poses, H, r, Rb)
        Pd = mem.e.covariance()
        assert np.array_equal(Pd, Pd.T)
        imud, posesd = state_of(mem.e)
        assert np.array_equal(imud[19:29], imu[19:29])
        assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == len(r) and res["used"] == len(clone)
        assert res["rows"] == rows_of(clone, flag) and np.array_equal(res["flag"], flag)
        sd = np.concatenate([imud[0:19], posesd.ravel()])
        sr = np.concatenate([imur[0:19], posesr.ravel()])
        rel = {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(),
               "state": np.abs(sd - sr).max() / np.abs(sr).max(),
               "nis": abs(res["nis"] - nisr) / nisr,
               "gamma": np.max(np.abs(res["gamma"] - gam) / gam)}
        assert abs(res["dx_norm"] - dxr) <= 1e-9 * dxr, M
        for k, v in rel.items():
            assert v <= CONTRACT[name], (M, k, v)
            worst[k] = max(worst[k], v)
    print(f"landmark rel vs dense numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 10 * MEASURED_REL[name][k], (k, v)


def test_jacobian_by_finite_differences():
    """the engine's update against the dense update built from a central-difference Jacobian through the injection"""
    from types import SimpleNamespace
    from oracle.msckf_numpy import MSCKF as NumpyMSCKF, quat_mul, quat_normalized
    buq = lambda d: NumpyMSCKF._build_update_quat(SimpleNamespace(S=np.float64, dt=np.float64), d)  # noqa: E731
    rng = np.random.default_rng(4)
    M = 6
    base = Member(np.float64, M, seed=11)
    mem = base.twin(np.float64)
    imu, poses = state_of(mem.e)
    P = mem.e.covariance().astype(np.float64)
    clone, z, p_L = make_obs(rng, poses, {0: 2, 3: 4, 5: 1})
    eps = 1e-6

    def fd(k, pl):
        J = np.zeros((2, 6))
        for j in range(6):
            zz = []
            for s in (+1, -1):
                pk = poses[k].copy()
                d = np.zeros(6); d[j] = s * eps
                pk[3:7] = quat_normalized(quat_mul(buq(d[0:3]), pk[3:7]))
                pk[0:3] += d[3:6]
                zz.append(project(pk, pl)[1][0])
            J[:, j] = (zz[0] - zz[1]) / (2 * eps)
        return J

    H, r, Rb, _, _ = dense(P, poses, clone, z, p_L, R_PIX, jac=fd)
    Pr, imur, posesr, nisr, dxr = numpy_update(P, imu, poses, H, r, Rb)
    res = mem.e.landmark_update(clone, z, p_L, R=R_PIX)
    imud, posesd = state_of(mem.e)
    Pd = mem.e.covariance()
    dxd = np.concatenate([imud[0:19], posesd.ravel()]) - np.concatenate([imu[0:19], poses.ravel()])
    dxn = np.concatenate([imur[0:19], posesr.ravel()]) - np.concatenate([imu[0:19], poses.ravel()])
    assert np.abs(dxd - dxn).max() <= 1e-6 * np.abs(dxn).max()
    assert np.abs(Pd - Pr).max() <= 1e-6 * np.abs(Pr).max()
    assert abs(res["nis"] - nisr) <= 1e-6 * nisr


def test_against_caller_linearised_update():
    rng = np.random.default_rng(9)
    M = 10
    base = Member(np.float64, M, seed=12)
    worst = 0.0
    for k, cnt in ((0, 1), (4, 5), (9, 16)):
        a, b = base.twin(np.float64), base.twin(np.float64)
        imu, poses = state_of(a.e)
        P = a.e.covariance()
        clone, z, p_L = make_obs(rng, poses, {k: cnt})
        H, r, Rb, _, _ = dense(P, poses, clone, z, p_L, R_PIX)
        ra = a.e.landmark_update(clone, z, p_L, R=R_PIX)
        rb = b.e.aid_update(capi.AID_LINEAR, r, Rb, H=H)
        sa, sb = a.e.state(), b.e.state()
        rel = max(np.abs(a.e.covariance() - b.e.covariance()).max() / np.abs(b.e.covariance()).max(),
                  max(np.abs(x - y).max() / np.abs(y).max() for x, y in zip(sa, sb)),
                  abs(ra["nis"] - rb["nis"]) / rb["nis"])
        assert rel <= 1e-9, (k, cnt, rel)
        worst = max(worst, rel)
    print(f"landmark vs LINEAR fp64: {worst:.3e}")
    assert worst <= 10 * MEASURED_LINEAR


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(8)
    mem = [Member(dtype, Ms[i % 4], seed=90 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    specs = []
    for i, m in enumerate(mem):
        M = m.e.num_clones()
        if M == 0 or i % 7 == 3:
            specs.append(None)
            continue
        _, poses = state_of(m.e)
        counts = {int(k): int(rng.integers(1, 6)) for k in rng.choice(M, size=min(M, 1 + i % 9), replace=False)}
        clone, z, p_L = make_obs(rng, poses, counts)
        specs.append({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX if i % 2 else None, "chi2_obs": 0.0 if i % 3 else 50.0})
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], chi2_obs=s["chi2_obs"])
              for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        for key in ("nis", "dx_norm", "dof", "rows", "used", "applied", "status"):
            assert got[i][key] == single[i][key] or (np.isnan(got[i][key]) and np.isnan(single[i][key])), (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"]) and np.array_equal(got[i]["flag"], single[i]["flag"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


def test_calls_that_write_nothing():
    rng = np.random.default_rng(13)
    mem = [Member(np.float64, 4, seed=30 + i) for i in range(3)]
    lib = capi.lib()
    _, poses = state_of(mem[0].e)
    clone, z, p_L = make_obs(rng, poses, {0: 3, 2: 2})
    before = [snapshot(m.e) for m in mem]
    # every observation gated out
    r = mem[0].e.landmark_update(clone, z + 0.05, p_L, R=R_PIX, chi2_obs=1e-9)
    assert r["applied"] == 0 and r["status"] == 0 and r["used"] == 0 and r["dof"] == 0 and np.all(r["flag"] == 1)
    assert np.all(r["gamma"] > 1e-9)
    # every landmark behind the camera
    behind = np.array([2 * poses[k, 0:3] - pl for k, pl in zip(clone, p_L)])
    r = mem[0].e.landmark_update(clone, z, behind, R=R_PIX)
    assert r["applied"] == 0 and np.all(r["flag"] == 2) and np.all(np.isnan(r["gamma"]))
    assert_unchanged(snapshot(mem[0].e), before[0])
    sentinel = capi.LandmarkResult(7.0, 7.0, 7, 7, 7, 7, 7)

    def raw(e, spec):
        a, keep = capi.landmark_struct(spec)
        out = capi.LandmarkResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_landmark_update(e.h, C.byref(a), C.byref(out)), out, keep

    good = {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX}
    nan_z = z.copy(); nan_z[1, 0] = np.nan
    inf_p = p_L.copy(); inf_p[0, 2] = np.inf
    bad = [dict(good, clone=np.where(clone == 2, 4, clone)), dict(good, clone=np.where(clone == 2, -1, clone)),
           dict(good, z=nan_z), dict(good, p_L=inf_p), dict(good, R=np.array([[1e-5, 2e-5], [2e-5, 1e-5]])),
           dict(good, R=np.array([[np.nan, 0], [0, 1e-5]])), dict(good, R=-np.eye(2)), dict(good, chi2_obs=np.nan),
           {"clone": np.zeros(257, np.int32), "z": np.zeros((257, 2)), "p_L": np.ones((257, 3))}]
    for spec in bad:
        rc, out, _ = raw(mem[0].e, spec)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), spec
    a, keep = capi.landmark_struct(good)
    a.z = None
    assert lib.msckf_b200_landmark_update(mem[0].e.h, C.byref(a), C.byref(capi.LandmarkResult())) == -3
    a, keep = capi.landmark_struct(good)
    a.n_obs = 4097
    assert lib.msckf_b200_landmark_update(mem[0].e.h, C.byref(a), C.byref(capi.LandmarkResult())) == -3
    assert_unchanged(snapshot(mem[0].e), before[0])
    # a batch with one bad member changes no member
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.landmark_update([good, dict(good, z=nan_z), good])
    # an un-fetched update (a triangulation of one track) on member 1
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    launched = mem[1].e.launch_count()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.landmark_update([good, None, good])
    rc, out, _ = raw(mem[1].e, good)
    assert rc == -5 and out.as_dict() == sentinel.as_dict()
    assert mem[1].e.launch_count() == launched
    mem[1].e.fetch(1)
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)
    batch.close()
    # an applied update leaves the launch count alone too
    n0 = mem[2].e.launch_count()
    assert mem[2].e.landmark_update(clone, z, p_L, R=R_PIX)["applied"] == 1 and mem[2].e.launch_count() == n0


def test_non_finite_covariance_is_reported_and_applied():
    rng = np.random.default_rng(3)
    mem = Member(np.float64, 4, seed=3)
    P = mem.e.covariance()
    P[3, 3] = np.inf  # a gyro-bias variance: no clone row of P is read, only the downdate meets it
    mem.e.set_covariance(P)
    imu, poses = state_of(mem.e)
    clone, z, p_L = make_obs(rng, poses, {1: 2})
    with pytest.raises(RuntimeError, match="rc=-6"):
        mem.e.landmark_update(clone, z, p_L, R=R_PIX)
    assert not np.array_equal(state_of(mem.e)[1], poses)  # applied


def _stream(dtype, n_frames, at):
    """two class filters on one stream; at frame `at` filter A observes mapped landmarks from its two newest images, and B gets
    A's device state by copy_state"""
    from msckf_mono_b200 import synth
    from tests.parity_cases import make_engine
    rng = np.random.default_rng(6)
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
        if k == at:
            cs = fs[0].getCamStates()
            poses = np.hstack([cs["p_C_G"], cs["q_CG"]])
            ids, zs, ps = [], [], []
            for j in (-1, -2):
                pl = landmarks_in_front(rng, poses[j], 5)
                ids += [cs["state_id"][j]] * 5
                zs.append(project(poses[j], pl)[1] + 0.002 * rng.normal(size=(5, 2)))
                ps.append(pl)
            r = fs[0].landmark_update(ids, np.vstack(zs), np.vstack(ps))
            assert r["applied"] == 1 and r["used"] == 10
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
    a, b = _stream(dtype, 12, at=6)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y)


def test_runner_with_a_map():
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, map_every=1)
    s = mc.summarize(rec)
    m = s["map"]
    assert len(m["anis"]) == 60 and all(np.isfinite(m["anis"])) and m["applied"] == 1.0
    for c in ("orientation", "position", "pose", "imu"):
        assert np.all(np.isfinite(s["components"][c]["anees"][1:])), c
    rec0, _ = mc.run(range(8), truth, dtype=np.float64)
    s0 = mc.summarize(rec0)
    print(f"map: ANIS {m['mean_anis']:.3f} for {m['mean_dof']:.1f} dof per update (run bounds {m['run_bounds']}), updates inside "
          f"{m['updates_inside']:.2f}, gated {m['gated']:.3f}; position RMSE {s['pos_rmse_run']:.4f} m with the map, "
          f"{s0['pos_rmse_run']:.4f} m without; ANEES imu {s['components']['imu']['mean_anees']:.3f} / "
          f"{s0['components']['imu']['mean_anees']:.3f}")
    assert s["pos_rmse_run"] < s0["pos_rmse_run"]
