"""Mapped-landmark updates with map uncertainty on the device (msckf_b200_map_landmark_update / _batch_map_landmark_update:
msckf_b200_landmark_map's landmark ids and Sigma_L) against the dense marginal EKF in numpy fp64
(tests/landmark_map_reference.py: Joseph form, the oracle's injection), the exact-map call Sigma_L = NULL must be, the
inflated-R call a one-observation landmark equals, batches against single calls bit for bit, the iterated form, the calls
that must write nothing, and the runner with a noisy map."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import landmark_map_reference as ref
from tests.test_aid_gpu import numpy_update, snapshot, assert_unchanged
from tests.test_batch_stream_gpu import Member
from tests.test_landmark_gpu import R_PIX, state_of

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
CONTRACT = {"float32": 1e-5, "float64": 1e-9}
# worst relative differences to the dense marginal update of test_matches_dense_numpy, measured on an H100 80GB HBM3 (700 W
# power limit); the bounds are 10 x these.  fp32: P and the state are rounded to float32 once.
MEASURED_REL = {"float32": {"P": 5.67e-8, "state": 2.37e-8, "nis": 2.73e-11, "gamma": 4.76e-16},
                "float64": {"P": 2.35e-12, "state": 6.68e-13, "nis": 3.15e-11, "gamma": 2.18e-13}}
MEASURED_ONE_OBS = 4.14e-16  # test_one_observation_is_the_inflated_noise_call, same card
CHI2 = 1e-3  # gamma of an observation 0.5 off is ~0.1 at these P; of one at the pixel noise, ~1e-5


def scene(rng, poses, sets, sigma=0.05, noise=0.002, bad=()):
    """one landmark per clone set in `sets`, a dense random Sigma each; observations whose (landmark, clone) is in `bad` are
    pushed 0.5 off (the gate CHI2 rejects them).  clone, z, p_L, landmark, Sigma [L, 6] in shuffled order"""
    clone, z, p_L, lm, Sig = [], [], [], [], []
    for l, cs in enumerate(sets):
        pl = ref.landmarks_seen_from(rng, poses, cs)
        B = rng.normal(size=(3, 3)) * sigma
        Sig.append(ref.tri(B @ B.T + sigma ** 2 * np.eye(3)))
        for k in cs:
            zz = ref.project(poses[k], pl)[1][0] + noise * rng.normal(size=2)
            clone.append(k); lm.append(l); p_L.append(pl); z.append(zz + (0.5 if (l, k) in bad else 0.0))
    o = rng.permutation(len(clone))
    return np.array(clone, np.int32)[o], np.array(z)[o], np.array(p_L)[o], np.array(lm, np.int32)[o], np.array(Sig)


def sets_for(rng, M):
    """clone sets of 1, 2, 5 and 8 consecutive clones (as many as the window allows), some repeated, and the (landmark, clone)
    pairs to push off"""
    sets = [[k] for k in rng.choice(M, size=min(M, 4), replace=False)] + [[0]] * 2
    for c in (2, 5, 8):
        if M >= c:
            for _ in range(3):
                k0 = int(rng.integers(0, M - c + 1))
                sets.append(list(range(k0, k0 + c)))
    if M >= 2:
        sets.append(sets[-1])  # a second landmark of the same clone set
    bad = {(len(sets) - 1, sets[-1][0]), (0, sets[0][0])}
    return sets, bad


def compare(res, e, P, imu, poses, clone, z, p_L, lm, Sig, chi2, name):
    H, r, Rb, F, lmu, gam, flag = ref.dense(P, poses, clone, z, p_L, lm, Sig, R_PIX, chi2)
    Pr, imur, posesr, nisr, dxr = numpy_update(P, imu, poses, H, r, Rb)
    assert np.array_equal(res["flag"], flag)
    assert res["used"] == int(np.sum(flag == 0)) and res["dof"] == len(r) and res["applied"] == 1 and res["status"] == 0
    assert res["rows"] == ref.rows(clone, lm, flag)
    Pd = e.covariance()
    assert np.array_equal(Pd, Pd.T)
    imud, posesd = state_of(e)
    sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([imur[0:19], posesr.ravel()])
    ok = np.isfinite(gam)
    return {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(),
            "state": np.abs(sd - sr).max() / np.abs(sr).max(),
            "nis": abs(res["nis"] - nisr) / nisr,
            "gamma": np.max(np.abs(res["gamma"][ok] - gam[ok]) / gam[ok])}


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_dense_numpy(dtype):
    rng = np.random.default_rng(41)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0, "gamma": 0.0}
    for M, seed in ((1, 1), (3, 2), (12, 3), (40, 4), (90, 5)):
        mem = Member(dtype, M, seed=seed, max_clones=M + 2).twin(dtype, max_clones=M + 2)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        sets, bad = sets_for(rng, M)
        clone, z, p_L, lm, Sig = scene(rng, poses, sets, bad=bad)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=CHI2, landmark=lm, Sigma_L=Sig)
        assert res["used"] < len(clone)  # some observations are gated out
        rel = compare(res, mem.e, P, imu, poses, clone, z, p_L, lm, Sig, CHI2, name)
        for k, v in rel.items():
            assert v <= CONTRACT[name], (M, k, v)
            worst[k] = max(worst[k], v)
    print(f"map landmark rel vs dense numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 10 * MEASURED_REL[name][k], (k, v)


def test_null_sigma_is_the_exact_map_call():
    rng = np.random.default_rng(5)
    base = Member(np.float64, 12, seed=7, max_clones=14)
    a, b = base.twin(np.float64, max_clones=14), base.twin(np.float64, max_clones=14)
    _, poses = state_of(a.e)
    sets, _ = sets_for(rng, 12)
    clone, z, p_L, lm, _ = scene(rng, poses, sets)
    spec = {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX}
    la, keep = capi.landmark_struct(spec)
    lmk = np.ascontiguousarray(lm, dtype=np.int32)
    m = capi.LandmarkMap(lmk.ctypes.data, None, 3)
    out = capi.LandmarkResult()
    capi.check(capi.lib().msckf_b200_map_landmark_update(a.e.h, C.byref(la), C.byref(m), C.byref(out)), "map_landmark_update")
    ra = dict(out.as_dict(), gamma=keep[4], flag=keep[5])
    rb = b.e.landmark_update(clone, z, p_L, R=R_PIX)
    for k in ra:
        assert np.array_equal(ra[k], rb[k]), k
    for x, y in zip(snapshot(a.e), snapshot(b.e)):
        assert np.array_equal(x, y)


def test_one_observation_is_the_inflated_noise_call():
    rng = np.random.default_rng(6)
    base = Member(np.float64, 6, seed=8)
    a, b = base.twin(np.float64), base.twin(np.float64)
    imu, poses = state_of(a.e)
    clone, z, p_L, lm, Sig = scene(rng, poses, [[3]], sigma=0.1)
    _, _, _, F, _, _, _ = ref.dense(np.zeros((51, 51)), poses, clone, z, p_L, lm, Sig, R_PIX)
    Ri = R_PIX + F @ ref.sym(Sig[0]) @ F.T
    ra = a.e.landmark_update(clone, z, p_L, R=R_PIX, landmark=lm, Sigma_L=Sig)
    rb = b.e.landmark_update(clone, z, p_L, R=Ri)
    rel = max(np.abs(a.e.covariance() - b.e.covariance()).max() / np.abs(b.e.covariance()).max(),
              max(np.abs(x - y).max() / np.abs(y).max() for x, y in zip(a.e.state(), b.e.state())),
              abs(ra["nis"] - rb["nis"]) / rb["nis"], abs(ra["gamma"][0] - rb["gamma"][0]) / rb["gamma"][0])
    print(f"one-observation landmark vs inflated R: {rel:.3e}")
    assert rel <= 10 * MEASURED_ONE_OBS and ra["rows"] == rb["rows"] == 2


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [5, 30, 90, 0]  # member 32, alone in the second chunk of 32, has 5 clones and Sigma
    rng = np.random.default_rng(18)
    mem = [Member(dtype, Ms[i % 4], seed=190 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    specs = []
    for i, m in enumerate(mem):
        M = m.e.num_clones()
        if M == 0 or i % 7 == 3:
            specs.append(None)
            continue
        _, poses = state_of(m.e)
        sets, bad = sets_for(rng, M)
        clone, z, p_L, lm, Sig = scene(rng, poses, sets, bad=bad)
        s = {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX if i % 2 else None, "chi2_obs": 0.0 if i % 3 else CHI2,
             "max_iter": [0, 1, 4, 8][i % 4], "tol": 1e-12}
        if i % 5 != 1:
            s.update(landmark=lm, Sigma_L=Sig)
        specs.append(s)
    assert specs[32] is not None and "Sigma_L" in specs[32]
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], chi2_obs=s["chi2_obs"],
                                                         max_iter=s["max_iter"], tol=s["tol"], landmark=s.get("landmark"),
                                                         Sigma_L=s.get("Sigma_L"))
              for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, specs)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        for key in ("nis", "dx_norm", "dof", "rows", "used", "applied", "status", "iterations", "converged", "step"):
            assert got[i][key] == single[i][key] or (np.isnan(got[i][key]) and np.isnan(single[i][key])), (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"]) and np.array_equal(got[i]["flag"], single[i]["flag"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


def test_iterated_matches_numpy():
    rng = np.random.default_rng(9)
    for M, seed, max_iter in ((3, 21, 8), (12, 22, 8), (40, 23, 3)):
        mem = Member(np.float64, M, seed=seed, max_clones=M + 2).twin(np.float64, max_clones=M + 2)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        sets, _ = sets_for(rng, M)
        clone, z, p_L, lm, Sig = scene(rng, poses, sets)
        z = z + 0.01  # far enough from the linearisation point that iterating changes the answer
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, landmark=lm, Sigma_L=Sig, max_iter=max_iter, tol=1e-9)
        out = ref.iekf(P, imu, poses, clone, z, p_L, lm, Sig, R_PIX, max_iter=max_iter, tol=1e-9)
        assert res["iterations"] == out["iterations"] and res["converged"] == out["converged"], (M, res, out["iterations"])
        assert res["iterations"] >= 2
        assert np.abs(mem.e.covariance() - out["P"]).max() <= 1e-9 * np.abs(out["P"]).max()
        imud, posesd = state_of(mem.e)
        sd = np.concatenate([imud[0:19], posesd.ravel()])
        sr = np.concatenate([out["imu"][0:19], out["poses"].ravel()])
        assert np.abs(sd - sr).max() <= 1e-9 * np.abs(sr).max()
        assert abs(res["nis"] - out["nis"]) <= 1e-9 * out["nis"]


def test_calls_that_write_nothing():
    rng = np.random.default_rng(13)
    mem = [Member(np.float64, 10, seed=30 + i) for i in range(3)]
    lib = capi.lib()
    _, poses = state_of(mem[0].e)
    clone, z, p_L, lm, Sig = scene(rng, poses, [[0, 1, 2], [3], [4, 5]])
    before = [snapshot(m.e) for m in mem]
    sentinel = capi.LandmarkResult(7.0, 7.0, 7, 7, 7, 7, 7)
    # (snapshot includes the launch count, which landmark calls never change: P, the state and the poses are what is checked)
    good = {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX, "landmark": lm, "Sigma_L": Sig}

    def raw(e, spec, **fields):
        a, keep = capi.landmark_struct(spec)
        m, mkeep = capi.landmark_map_struct(spec)
        for k, v in fields.items():
            setattr(m, k, v)
        out = capi.LandmarkResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_map_landmark_update(e.h, C.byref(a), C.byref(m), C.byref(out)), out, (keep, mkeep)

    nan_S = Sig.copy(); nan_S[1, 2] = np.nan
    neg_S = Sig.copy(); neg_S[2] = [1e-2, 0, -1e-2, 0, 0, 1e-2]
    moved = p_L.copy(); moved[np.flatnonzero(lm == 0)[0], 0] += 1e-9
    twice = clone.copy(); i0 = np.flatnonzero(lm == 0); twice[i0[1]] = twice[i0[0]]
    nine = list(range(9))
    pl9 = ref.landmarks_seen_from(rng, poses, nine)
    big = {"clone": np.array(nine, np.int32), "z": np.zeros((9, 2)), "p_L": np.tile(pl9, (9, 1)), "landmark": np.zeros(9, np.int32),
           "Sigma_L": Sig[:1]}
    # 43 landmarks of the clone set {0, 1, 2, 3, 4, 5}: 258 observations in one group
    crowd = {"clone": np.tile(np.arange(6, dtype=np.int32), 43), "z": np.zeros((258, 2)), "p_L": np.ones((258, 3)),
             "landmark": np.repeat(np.arange(43, dtype=np.int32), 6), "Sigma_L": np.tile(Sig[:1], (43, 1))}
    cases = [dict(good, landmark=np.where(lm == 2, 3, lm)), dict(good, landmark=np.where(lm == 2, -1, lm)), dict(good, Sigma_L=nan_S),
             dict(good, Sigma_L=neg_S), dict(good, p_L=moved), dict(good, clone=twice), big, crowd]
    for spec in cases:
        rc, out, _ = raw(mem[0].e, spec)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), spec
    rc, out, _ = raw(mem[0].e, good, landmark=None)
    assert rc == -3 and out.as_dict() == sentinel.as_dict()
    assert_unchanged(snapshot(mem[0].e), before[0])
    # caps that need a wider window: 25 sets of 8 clones with 3 landmarks each may compress to 25 x 48 = 1200 > 1152 rows;
    # 257 clone sets of 2 clones exceed the 256 sets of a member
    wide = Member(np.float64, 40, seed=34)
    wb = snapshot(wide.e)
    sets = [list(range(k0, k0 + 8)) for k0 in range(25) for _ in range(3)]
    pairs = [[a, b] for a in range(40) for b in range(a + 1, 40)][:257]
    for ss in (sets, pairs):
        spec = {"clone": np.array([k for cs in ss for k in cs], np.int32), "z": np.zeros((sum(map(len, ss)), 2)),
                "p_L": np.repeat(np.arange(len(ss), dtype=float)[:, None] + np.ones(3), [len(cs) for cs in ss], axis=0),
                "landmark": np.repeat(np.arange(len(ss), dtype=np.int32), [len(cs) for cs in ss]), "Sigma_L": np.tile(Sig[:1], (len(ss), 1))}
        rc, out, _ = raw(wide.e, spec)
        assert rc == -3 and out.as_dict() == sentinel.as_dict()
        assert b"rows" in lib.msckf_b200_last_error() if ss is sets else b"clone sets" in lib.msckf_b200_last_error()
    assert_unchanged(snapshot(wide.e), wb)
    # a Sigma too small to invert in fp64 is refused, not launched
    rc, out, _ = raw(mem[0].e, dict(good, Sigma_L=np.tile([1e-300, 0, 1e-300, 0, 0, 1e-300], (3, 1))))
    assert rc == -3 and out.as_dict() == sentinel.as_dict()
    assert_unchanged(snapshot(mem[0].e), before[0])
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.landmark_update([good, dict(good, Sigma_L=neg_S), good])
    batch.close()
    for m, b in zip(mem, before):
        assert_unchanged(snapshot(m.e), b)


def test_runner_with_an_uncertain_map():
    from msckf_mono_b200 import montecarlo as mc
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, map_every=5, map_sigma=0.1, map_uncertain=True, map_clones=5)
    s = mc.summarize(rec)
    m = s["map"]
    assert len(m["anis"]) == 12 and all(np.isfinite(m["anis"])) and m["applied"] == 1.0
    for c in ("orientation", "position", "pose", "imu"):
        assert np.all(np.isfinite(s["components"][c]["anees"][1:])), c
    rex, _ = mc.run(range(8), truth, dtype=np.float64, map_every=5, map_sigma=0.1, map_clones=5)
    sx = mc.summarize(rex)
    print(f"noisy map (0.1 m), 5 clones every 5 frames: ANIS {m['mean_anis']:.2f} for {m['mean_dof']:.1f} dof uncertain, "
          f"{sx['map']['mean_anis']:.2f} exact; IMU ANEES {s['components']['imu']['mean_anees']:.2f} / "
          f"{sx['components']['imu']['mean_anees']:.2f}")
    assert m["mean_anis"] < sx["map"]["mean_anis"]
