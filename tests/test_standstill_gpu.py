"""Standstill detection and the zero-motion update on the device (msckf_b200_standstill_update / _batch_standstill_update) and
the at-rest stack models GYRO_AT_REST and ACCEL_AT_REST, against tests/standstill_reference.py: readings at rest are applied
and P and the state match the dense update over every reading row; the call is msckf_b200_aid_stack_update on the three items
the reference forms, bit for bit; a moving window launches nothing; a biased mean fails the gate and writes nothing; a batch
is its single calls; the new models in plain and FDE stacks with other items match numpy; the iterated forms refuse them."""
import numpy as np
import pytest
from scipy.linalg import block_diag

from msckf_mono_b200 import capi, synth
from tests import standstill_reference as ref
from tests.test_aid_gpu import CONTRACT, assert_unchanged, snapshot, spd, state_of
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
# worst relative differences of an applied standstill to the dense fp64 update over all 6k + 3 rows (test_applied_matches_the
# dense_update), measured on an H100 80GB HBM3 (700 W power limit); the bounds are 10 x these (and never above the aided
# updates' CONTRACT).  fp32: P and the state are rounded to float32 once; the NIS is fp64 on the widened P in both.
MEASURED = {"float32": {"P": 5.55e-8, "state": 5.31e-8, "nis": 1.89e-14},
            "float64": {"P": 5.88e-16, "state": 1.18e-14, "nis": 1.48e-14}}
CFG = {"noise_scale": 1.0, "sigma_v": 0.01, "scatter_max": 4.0, "chi2_max": 1e6}


def Q_of(dtype):
    """the engine's Q_imu (Member's workload), as the engine holds it"""
    Q = synth.make_window_workload(n_features=4, n_clones=2, seq=3)["noise"]["Q_imu"]
    return np.asarray(Q, dtype=dtype).astype(np.float64)


def rest(rng, m, k, dtype, **kw):
    imu, _ = state_of(m.e)
    return ref.rest_readings(rng, imu, k, Q_of(dtype), **kw).astype(dtype).astype(np.float64)


def moving(rng, k, dtype):
    r = rest(rng, Member(dtype, 0, seed=1), k, dtype)
    t = np.cumsum(r[:, 6])
    r[:, 0:3] += 2.0 * np.sin(8.0 * t)[:, None]
    r[:, 3:6] += 5.0 * np.cos(5.0 * t)[:, None]
    return r.astype(dtype).astype(np.float64)


def cap(M):
    """the engine capacity of a window of M clones (at most the engine's hard limit of 192)"""
    return min(M + 8, 192)


def _stack(res):
    return {k: res[k] for k in ("nis", "dx_norm", "dof", "applied", "status")}


@pytest.mark.parametrize("dtype", DTYPES)
def test_applied_matches_the_dense_update(dtype):
    name = np.dtype(dtype).name
    rng = np.random.default_rng(41)
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0}
    for M, seed in ((0, 1), (30, 2), (192, 3)):
        base = Member(dtype, M, seed=seed, max_clones=cap(M))
        for k in (2, 10, 400):
            m = base.twin(dtype, max_clones=cap(M))
            imu, poses = state_of(m.e)
            P = m.e.covariance().astype(np.float64)
            r = rest(rng, m, k, dtype)
            res = m.e.standstill_update(r, CFG)
            assert res["outcome"] == 0 and res["applied"] == 1 and res["dof"] == 9 and res["status"] == 0, (M, k, res)
            st = ref.stats(r, Q_of(dtype), CFG["noise_scale"], CFG["sigma_v"])
            assert abs(res["scatter"] - st["scatter"]) <= 1e-12 * st["scatter"], (M, k)
            d = ref.dense_update(P, imu[0:19], poses, r, Q_of(dtype), CFG["noise_scale"], CFG["sigma_v"])
            Pd = m.e.covariance().astype(np.float64)
            imud, posesd = state_of(m.e)
            sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([d["imu"], d["poses"].ravel()])
            rel = {"P": np.abs(Pd - d["P"]).max() / np.abs(d["P"]).max(), "state": np.abs(sd - sr).max() / np.abs(sr).max(),
                   "nis": abs(res["nis"] + st["sigma"] - d["nis"]) / d["nis"]}
            for key, v in rel.items():
                assert v <= min(10 * MEASURED[name][key], CONTRACT[name]), (M, k, key, v)
                worst[key] = max(worst[key], v)
    print(f"standstill rel vs dense {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))


@pytest.mark.parametrize("dtype", DTYPES)
def test_equals_the_stack_of_its_three_items_bit_for_bit(dtype):
    rng = np.random.default_rng(43)
    for M, k in ((0, 2), (30, 10), (192, 400)):
        a = Member(dtype, M, seed=10 + M, max_clones=cap(M))
        b = a.twin(dtype, max_clones=cap(M))
        r = rest(rng, a, k, dtype)
        st = ref.stats(r, Q_of(dtype), CFG["noise_scale"], CFG["sigma_v"])
        got = a.e.standstill_update(r, CFG)
        want = b.e.aid_stack_update(ref.items(st), chi2_max=CFG["chi2_max"])
        assert _stack(got) == want and got["outcome"] == 0, (M, k)
        for x, y in zip(a.snapshot(), b.snapshot()):
            assert np.array_equal(x, y), (M, k)


@pytest.mark.parametrize("dtype", DTYPES)
def test_a_moving_window_launches_and_writes_nothing(dtype):
    rng = np.random.default_rng(47)
    m = Member(dtype, 30, seed=5)
    before = snapshot(m.e)
    res = m.e.standstill_update(moving(rng, 40, dtype), CFG)
    assert res["outcome"] == 1 and res["scatter"] > CFG["scatter_max"] and res["applied"] == 0 and np.isnan(res["nis"])
    assert_unchanged(snapshot(m.e), before)


@pytest.mark.parametrize("dtype", DTYPES)
def test_a_biased_mean_fails_the_gate_and_writes_nothing(dtype):
    rng = np.random.default_rng(53)
    m = Member(dtype, 12, seed=6)
    n = 15 + 6 * 12
    m.e.set_covariance(1e-6 * np.eye(n))
    before = snapshot(m.e)
    r = rest(rng, m, 50, dtype, bias=np.r_[0.0, 0.0, 0.0, 2.0, -2.0, 0.0])
    res = m.e.standstill_update(r, dict(CFG, chi2_max=30.0))
    assert res["outcome"] == 2 and res["applied"] == 0 and res["nis"] > 30.0 and res["scatter"] <= CFG["scatter_max"]
    assert_unchanged(snapshot(m.e), before)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    rng = np.random.default_rng(59)
    Ms = [0, 3, 30]
    mem = [Member(dtype, Ms[i % 3], seed=600 + i) for i in range(40)]
    twins = [m.twin(dtype) for m in mem]
    kinds = ["rest", "moving", "biased", "absent", "rest"]
    rs = []
    for i, m in enumerate(mem):
        kind = kinds[i % 5]
        if kind in ("biased",):
            P = 1e-6 * np.eye(15 + 6 * m.e.num_clones())
            m.e.set_covariance(P); twins[i].e.set_covariance(P)
        rs.append(None if kind == "absent" else moving(rng, 20, dtype) if kind == "moving" else
                  rest(rng, m, 400, dtype, bias=np.r_[0, 0, 0, 1.0, -1.0, 0]) if kind == "biased" else
                  rest(rng, m, [2, 10, 400][i % 3], dtype))
    cfg = dict(CFG, chi2_max=50.0)
    before = [snapshot(m.e) for m in mem]
    single = [None if r is None else t.e.standstill_update(r, cfg) for t, r in zip(twins, rs)]
    assert {s["outcome"] for s in single if s} == {0, 1, 2}
    batch = capi.Batch([m.e for m in mem])
    got = batch.standstill_update(rs, cfg)
    batch.close()
    for i, m in enumerate(mem):
        if rs[i] is None:
            assert got[i] is None
        else:
            assert got[i].keys() == single[i].keys()
            assert all(got[i][k] == single[i][k] or (np.isnan(got[i][k]) and np.isnan(single[i][k])) for k in got[i]), i
        if rs[i] is None or single[i]["outcome"] != 0:
            assert_unchanged(snapshot(m.e), before[i])
        for x, y in zip(m.snapshot(), twins[i].snapshot()):
            assert np.array_equal(x, y), i


def test_refusals_write_nothing():
    rng = np.random.default_rng(61)
    m = Member(np.float64, 3, seed=7)
    before = snapshot(m.e)
    r = rest(rng, m, 10, np.float64)
    bad_r = [r[:1], np.vstack([r[:4], np.r_[r[4, :6], 0.0]]), np.where(np.arange(70).reshape(10, 7) == 12, np.nan, r),
             np.tile(r, (410, 1))[:4097]]
    for x in bad_r:
        with pytest.raises(RuntimeError, match="rc=-3"):
            m.e.standstill_update(x, CFG)
    for cfg in (dict(CFG, noise_scale=0.5), dict(CFG, sigma_v=0.0), dict(CFG, scatter_max=np.inf), dict(CFG, chi2_max=np.nan)):
        with pytest.raises(RuntimeError, match="rc=-3"):
            m.e.standstill_update(r, cfg)
    other = Member(np.float64, 0, seed=8)
    batch = capi.Batch([m.e, other.e])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.standstill_update([r, r[:1]], CFG)
    assert batch.standstill_update([None, None], CFG) == [None, None]
    batch.close()
    assert_unchanged(snapshot(m.e), before)


def _rows(item, imu, n):
    """(H, r) of a VELOCITY / POSITION / at-rest item"""
    z = np.asarray(item["z"], dtype=np.float64)
    if item["model"] in (capi.AID_GYRO_AT_REST, capi.AID_ACCEL_AT_REST):
        Hr, h = ref.rest_jacobian(imu, n), ref.predicted(imu)
        s = slice(0, 3) if item["model"] == capi.AID_GYRO_AT_REST else slice(3, 6)
        return Hr[s], z - h[s]
    o, c = (3, 6) if item["model"] == capi.AID_VELOCITY else (0, 12)
    H = np.zeros((3, n))
    H[:, c:c + 3] = np.eye(3)
    return H, z - imu[o:o + 3]


@pytest.mark.parametrize("dtype", DTYPES)
def test_new_models_in_plain_and_fde_stacks_match_numpy(dtype):
    name = np.dtype(dtype).name
    rng = np.random.default_rng(67)
    fde = {"chi2": [1e9] * 32, "max_exclude": 0}
    for M in (0, 30):
        base = Member(dtype, M, seed=70 + M)
        imu, poses = state_of(base.e)
        n = 15 + 6 * M
        h = ref.predicted(imu[0:19])
        items = [{"model": capi.AID_POSITION, "z": imu[0:3] + 0.05 * rng.normal(size=3), "R": spd(rng, 3, 0.01)},
                 {"model": capi.AID_ACCEL_AT_REST, "z": h[3:6] + 0.02 * rng.normal(size=3), "R": spd(rng, 3, 1e-3)},
                 {"model": capi.AID_GYRO_AT_REST, "z": h[0:3] + 1e-3 * rng.normal(size=3), "R": spd(rng, 3, 1e-5)},
                 {"model": capi.AID_VELOCITY, "z": np.zeros(3), "R": spd(rng, 3, 1e-4)}]
        P = base.e.covariance().astype(np.float64)
        Hs, rs = zip(*[_rows(it, imu, n) for it in items])
        d = ref.joseph(P, imu[0:19], poses, np.vstack(Hs), np.concatenate(rs), block_diag(*[it["R"] for it in items]))
        for use_fde in (False, True):
            m = base.twin(dtype)
            res = m.e.aid_stack_update(items, fde=fde if use_fde else None)
            assert res["applied"] == 1 and res["dof"] == 12 and (not use_fde or res["outcome"] == 0)
            Pd = m.e.covariance().astype(np.float64)
            imud, posesd = state_of(m.e)
            assert np.abs(Pd - d["P"]).max() / np.abs(d["P"]).max() <= CONTRACT[name]
            sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([d["imu"], d["poses"].ravel()])
            assert np.abs(sd - sr).max() / np.abs(sr).max() <= CONTRACT[name]
            assert abs(res["nis"] - d["nis"]) <= 1e-9 * d["nis"]
        # the iterated forms refuse the at-rest models and write nothing
        m = base.twin(dtype)
        before = snapshot(m.e)
        for kw in ({}, {"fde": fde}):
            with pytest.raises(RuntimeError, match="rc=-3"):
                m.e.aid_stack_update(items, max_iter=4, tol=1e-12, **kw)
        # ... and a at-rest item with a non-zero a or b is refused
        with pytest.raises(RuntimeError, match="rc=-3"):
            m.e.aid_stack_update([dict(items[2], a=1)])
        assert_unchanged(snapshot(m.e), before)


def test_runner_detects_a_stop_and_holds_the_position():
    """8 trials over one stop of 15 frames: at least 90 % of the stationary frames are found at rest and no cruising frame,
    and the position error grows less over the stop than without the standstill update"""
    from msckf_mono_b200 import montecarlo as mc
    truth = mc.make_truth(n_frames=66, seq=8, stop={"every": 60, "frames": 15, "ramp": 5})
    cfg = {"noise_scale": 1.0, "sigma_v": 0.01, "scatter_max": 2.0, "chi2_max": 27.9}
    on = mc.summarize(mc.run(range(8), truth, standstill=cfg)[0])["stops"]
    off = mc.summarize(mc.run(range(8), truth)[0])["stops"]
    print(f"standstill runner: detected {on['detected']}, growth per stop {on['pos_err_growth_per_stop']:.4f} m "
          f"(without: {off['pos_err_growth_per_stop']:.4f} m), ANIS {on['anis']:.2f} in {on['run_bounds']}")
    assert len(on["stops"]) == 1 and on["frames"]["stationary"] >= 13
    assert on["detected"]["stationary"] >= 0.9 and on["detected"]["cruise"] == 0.0
    assert on["pos_err_growth_per_stop"] < off["pos_err_growth_per_stop"]
