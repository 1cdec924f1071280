"""GNSS antenna positions and headings in the stacked aided update on the device (msckf_b200_aid_stack_update /
_batch_aid_stack_update with ANTENNA_POSITION, CLONE_ANTENNA_POSITION, HEADING, CLONE_HEADING) against numpy fp64 on the fetched
covariance and state: the Joseph-form covariance, the state injection of oracle/msckf_numpy.py and the NIS, with the models of
montecarlo.  Also: the device Jacobians against central differences through montecarlo.perturb (read back through a LINEAR
update), every mask, a stack mixed with odometry against the dense stacked update, batch against single calls bit for bit,
refusals and the degenerate heading (nothing written), and the runner's GNSS."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from oracle.msckf_numpy import quat_to_rot
from tests.test_aid_gpu import CONTRACT, assert_unchanged, snapshot, spd, state_of
from tests.test_batch_stream_gpu import Member
from tests.test_odometry_gpu import H_r as odometry_H_r, body_item, rel_item

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
GNSS = (capi.AID_ANTENNA_POSITION, capi.AID_CLONE_ANTENNA_POSITION, capi.AID_HEADING, capi.AID_CLONE_HEADING)


def H_r(item, imu, poses, n):
    if item["model"] in GNSS:
        return mc.odometry_jacobian(item, imu, poses, n), mc.odometry_residual(item, imu, poses)
    return odometry_H_r(item, imu, poses, n)


def stack_reference(items, imu, poses, P):
    from scipy.linalg import block_diag
    from tests.test_aid_gpu import numpy_update
    Hs, rs = zip(*[H_r(it, imu, poses, P.shape[0]) for it in items])
    return numpy_update(P, imu, poses, np.vstack(Hs), np.concatenate(rs), block_diag(*[it["R"] for it in items]))


def rel_errors(e, res, ref, imu0):
    """relative differences of P, the state, the NIS and |dx| to the numpy reference, as test_odometry_gpu.rel_errors, but with
    |dx| held to the dtype's contract like the others rather than to 1e-9.  Worst differences measured on an H100 80GB HBM3
    (700 W power limit), test_models_match_numpy: fp32 P 1.8e-7, state 1.9e-8, NIS 5.6e-7, |dx| 3.0e-7; fp64 P 6.0e-16,
    state 4.5e-17, NIS 2.4e-14, |dx| 1.2e-14"""
    Pr, imur, posesr, nisr, dxr = ref
    Pd = e.covariance()
    assert np.array_equal(Pd, Pd.T)
    imud, posesd = state_of(e)
    assert np.array_equal(imud[19:29], imu0[19:29])  # the observability copies are not touched
    sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([imur[0:19], posesr.ravel()])
    return {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(), "state": np.abs(sd - sr).max() / np.abs(sr).max(),
            "nis": abs(res["nis"] - nisr) / nisr, "dx": abs(res["dx_norm"] - dxr) / dxr}


def antenna_item(rng, imu, poses, mask=7, clone=None, scale=0.1, lever=None):
    lever = rng.normal(size=3) * 0.5 if lever is None else np.asarray(lever, dtype=np.float64)
    p, q = (imu[0:3], imu[15:19]) if clone is None else (poses[clone, 0:3], poses[clone, 3:7])
    z = np.r_[mc.antenna_position(p, q, lever) + scale * rng.normal(size=3), lever]
    R = spd(rng, bin(mask).count("1"), 0.02)
    if clone is None:
        return {"model": capi.AID_ANTENNA_POSITION, "a": mask, "z": z, "R": R}
    return {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": clone, "b": mask, "z": z, "R": R}


def heading_item(rng, imu, poses, clone=None, scale=0.05, axis=None):
    axis = rng.normal(size=3) if axis is None else np.asarray(axis, dtype=np.float64)
    q = imu[15:19] if clone is None else poses[clone, 3:7]
    z = np.r_[mc.wrap_angle(mc.heading_of(q, axis) + scale * rng.normal()), axis]
    R = np.array([[0.01 + 0.01 * rng.random()]])
    if clone is None:
        return {"model": capi.AID_HEADING, "z": z, "R": R}
    return {"model": capi.AID_CLONE_HEADING, "a": clone, "z": z, "R": R}


def gnss_cases(rng, imu, poses, M):
    out = [antenna_item(rng, imu, poses, 7), antenna_item(rng, imu, poses, 0b011), antenna_item(rng, imu, poses, 0b100, lever=np.zeros(3)),
           heading_item(rng, imu, poses)]
    if M >= 1:
        out += [antenna_item(rng, imu, poses, 7, clone=0), antenna_item(rng, imu, poses, 0b101, clone=M - 1),
                heading_item(rng, imu, poses, clone=M // 2), heading_item(rng, imu, poses, clone=M - 1)]
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_models_match_numpy(dtype):
    rng = np.random.default_rng(41)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0, "dx": 0.0}
    for M, seed in ((0, 1), (1, 6), (3, 2), (12, 3), (40, 4)):
        base = Member(dtype, M, seed=seed)
        imu, poses = state_of(base.e)
        for item in gnss_cases(rng, imu, poses, M):
            mem = base.twin(dtype)
            imu_t, poses_t = state_of(mem.e)  # (the reference linearises at the twin's own state)
            P = mem.e.covariance().astype(np.float64)
            res = mem.e.aid_stack_update([item])
            assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == len(mc.odometry_residual(item, imu_t, poses_t))
            rel = rel_errors(mem.e, res, stack_reference([item], imu_t, poses_t, P), imu_t)
            for k, v in rel.items():
                assert v <= CONTRACT[name], (M, item["model"], k, v)
                worst[k] = max(worst[k], v)
    print(f"gnss rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))


def test_jacobians_match_central_differences():
    """H of the four models by central differences of the residual through montecarlo.perturb, against the numpy H and against
    the device: a LINEAR update with the difference quotient gives the covariance the model's update gives"""
    rng = np.random.default_rng(19)
    M = 12
    base = Member(np.float64, M, seed=9)
    n = 15 + 6 * M
    imu, poses = state_of(base.e)
    est = {"imu": imu[0:19], "poses": poses}
    items = [antenna_item(rng, imu, poses, 7, scale=0.0), antenna_item(rng, imu, poses, 7, clone=5, scale=0.0),
             heading_item(rng, imu, poses, scale=0.0), heading_item(rng, imu, poses, clone=11, scale=0.0),
             heading_item(rng, imu, poses, clone=0, scale=0.0, axis=[0.0, 0.3, 1.0])]
    eps = 1e-6
    worst = 0.0
    for item in items:
        r0 = mc.odometry_residual(item, imu, poses)
        assert np.abs(r0).max() <= 1e-12
        Hcd = np.zeros((len(r0), n))
        for k in range(n):
            e = np.zeros(n); e[k] = eps
            sp, sm = mc.perturb(est, e), mc.perturb(est, -e)
            Hcd[:, k] = -(mc.odometry_residual(item, sp["imu"], sp["poses"]) - mc.odometry_residual(item, sm["imu"], sm["poses"])) / (2 * eps)
        Ha = mc.odometry_jacobian(item, imu, poses, n)
        assert np.abs(Hcd - Ha).max() <= 1e-6, np.abs(Hcd - Ha).max()
        a, b = base.twin(np.float64), base.twin(np.float64)
        ra = a.e.aid_stack_update([item])
        rb = b.e.aid_update(capi.AID_LINEAR, r0, item["R"], H=Hcd)
        Pa, Pb = a.e.covariance(), b.e.covariance()
        d = np.abs(Pa - Pb).max() / np.abs(Pa).max()
        assert d <= 1e-8, (item["model"], d)
        assert abs(ra["nis"] - rb["nis"]) <= 1e-8 * max(rb["nis"], 1e-12)
        worst = max(worst, d)
    print(f"gnss device H vs central differences: P rel {worst:.3e}")


@pytest.mark.parametrize("model", [capi.AID_ANTENNA_POSITION, capi.AID_CLONE_ANTENNA_POSITION])
def test_every_mask(model):
    rng = np.random.default_rng(7)
    M = 5
    base = Member(np.float64, M, seed=12)
    imu, poses = state_of(base.e)
    for mask in range(1, 8):
        item = antenna_item(rng, imu, poses, mask, clone=None if model == capi.AID_ANTENNA_POSITION else mask % M)
        mem = base.twin(np.float64)
        imu_t, poses_t = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        res = mem.e.aid_stack_update([item])
        assert res["dof"] == bin(mask).count("1") and res["applied"] == 1
        for k, v in rel_errors(mem.e, res, stack_reference([item], imu_t, poses_t, P), imu_t).items():
            assert v <= CONTRACT["float64"], (mask, k, v)


@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_stack_equals_the_dense_stacked_update(dtype):
    rng = np.random.default_rng(29)
    name = np.dtype(dtype).name
    M = 12
    base = Member(dtype, M, seed=5)
    imu, poses = state_of(base.e)
    items = [antenna_item(rng, imu, poses, 7), heading_item(rng, imu, poses, clone=M - 3), body_item(rng, imu, 0b111),
             rel_item(rng, poses, M - 2, M - 1)]
    st = base.twin(dtype)
    imu_t, poses_t = state_of(st.e)
    P = st.e.covariance().astype(np.float64)
    res = st.e.aid_stack_update(items)
    assert res["dof"] == 3 + 1 + 3 + 6 and res["applied"] == 1
    rel = rel_errors(st.e, res, stack_reference(items, imu_t, poses_t, P), imu_t)
    print(f"gnss mixed stack rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in rel.items()))
    for k, v in rel.items():
        assert v <= CONTRACT[name], (k, v)


def _random_stack(rng, imu, poses, M, k):
    """k items (rows <= 32) valid for a window of M clones: GNSS models mixed with odometry"""
    out, rows = [], 0
    while len(out) < k:
        kind = rng.integers(0, 6)
        if kind == 0:
            it = antenna_item(rng, imu, poses, int(rng.integers(1, 8)))
        elif kind == 1 and M >= 1:
            it = antenna_item(rng, imu, poses, int(rng.integers(1, 8)), clone=int(rng.integers(0, M)))
        elif kind == 2:
            it = heading_item(rng, imu, poses)
        elif kind == 3 and M >= 1:
            it = heading_item(rng, imu, poses, clone=int(rng.integers(0, M)))
        elif kind == 4 and M >= 2:
            a, b = rng.choice(M, size=2, replace=False)
            it = rel_item(rng, poses, int(a), int(b))
        else:
            it = body_item(rng, imu, int(rng.integers(1, 8)))
        m = len(it["R"])
        if rows + m > 32:
            break
        rows += m
        out.append(it)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(18)
    mem = [Member(dtype, Ms[i % 4], seed=290 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    stacks = []
    for i, m in enumerate(mem):
        k = [1, 2, 3, 8, 0][i % 5]  # (k = 0: the member is left alone)
        imu, poses = state_of(m.e)
        stacks.append(_random_stack(rng, imu, poses, m.e.num_clones(), k) if k else None)
    assert stacks[32] is not None
    assert {it["model"] for s in stacks if s for it in s} >= set(GNSS)
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.aid_stack_update(s) for t, s in zip(twins, stacks)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.aid_stack_update(stacks)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, stacks)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        assert got[i] == single[i] and got[i]["applied"] == 1, i
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


def test_refusals_and_the_degenerate_heading_write_nothing():
    rng = np.random.default_rng(23)
    M = 4
    mem = [Member(np.float64, M, seed=60 + i) for i in range(3)]
    lib = capi.lib()
    imu, poses = state_of(mem[0].e)
    ant, cant = antenna_item(rng, imu, poses, 7), antenna_item(rng, imu, poses, 3, clone=2)
    hd, chd = heading_item(rng, imu, poses), heading_item(rng, imu, poses, clone=1)
    before = [snapshot(m.e) for m in mem]
    sentinel = capi.AidResult(7.0, 7.0, 7, 7, 7)

    def raw(e, items, chi2_max=0.0):
        arr, keep = capi.aid_items(items)
        out = capi.AidResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_aid_stack_update(e.h, arr, C.c_int(len(items)), C.c_double(chi2_max), C.byref(out)), out

    bad = [dict(ant, a=0), dict(ant, a=8), dict(cant, b=0), dict(cant, b=9), dict(cant, a=-1), dict(cant, a=M), dict(chd, a=M),
           dict(chd, a=-1), dict(hd, z=np.r_[hd["z"][0], 0.0, 0.0, 0.0]), dict(chd, z=np.r_[1.0, 0.0, 0.0, 0.0]),
           dict(hd, a=1), dict(hd, b=2), dict(ant, b=1), dict(chd, b=3)]
    for i in range(6):
        z = ant["z"].copy(); z[i] = np.nan
        bad.append(dict(ant, z=z))
        z = cant["z"].copy(); z[i] = np.inf
        bad.append(dict(cant, z=z))
    for i in range(4):
        z = hd["z"].copy(); z[i] = np.nan
        bad.append(dict(hd, z=z))
        z = chd["z"].copy(); z[i] = -np.inf
        bad.append(dict(chd, z=z))
    R_nan = np.eye(2); R_nan[1, 0] = np.nan
    bad.append(dict(cant, R=R_nan))
    pose = {"model": capi.AID_POSE, "z": np.r_[imu[0:3], imu[15:19]], "R": np.eye(6)}
    stacks = [[b] for b in bad] + [[ant] * 8 + [hd], [pose] * 5 + [ant], [pose] * 5 + [cant, hd]]  # 9 items; 33 rows; 33 rows
    for items in stacks:
        rc, out = raw(mem[0].e, items)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), [(it["model"], it.get("a"), it.get("b")) for it in items]
    assert raw(mem[0].e, [ant, hd], chi2_max=np.nan)[0] == -3
    # msckf_b200_aid_update refuses the stack-only models
    for it in (ant, cant, hd, chd):
        with pytest.raises(RuntimeError, match="rc=-3"):
            mem[0].e.aid_update(it["model"], it["z"], it["R"], clone=it.get("a", 0))
    assert_unchanged(snapshot(mem[0].e), before[0])
    # a heading axis along the vertical: status 2, NIS NaN, nothing written -- alone, and inside a stack
    up = quat_to_rot(imu[15:19]) @ np.array([0.0, 0.0, 1.0])  # C(q_IG) e_z: d = C^T f is vertical
    upc = quat_to_rot(poses[3, 3:7]) @ np.array([0.0, 0.0, 2.0])
    vert = [[dict(hd, z=np.r_[0.3, up])], [ant, dict(chd, a=3, z=np.r_[0.3, upc]), body_item(rng, imu, 7)]]
    for items in vert:
        rc, out = raw(mem[0].e, items)
        assert rc == 0 and out.status == 2 and out.applied == 0 and np.isnan(out.nis) and out.dx_norm == 0.0
        assert out.dof == sum(len(it["R"]) for it in items)
    # just off the vertical (about 2e-3 rad): a valid heading
    tilt = quat_to_rot(imu[15:19]) @ np.array([2e-3, 0.0, 1.0])
    tw = mem[0].twin(np.float64)  # (held: the twin owns its engine)
    assert tw.e.aid_stack_update([dict(hd, z=np.r_[0.3, tilt])])["status"] == 0
    assert_unchanged(snapshot(mem[0].e), before[0])
    # in a batch the degenerate member reports status 2 and is left alone; the others are applied
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_stack_update([[ant], [dict(cant, a=M)], [hd]])
    for m, b in zip(mem, before):
        assert_unchanged(snapshot(m.e), b)
    i1, p1 = state_of(mem[1].e)
    res = batch.aid_stack_update([[ant, hd], [dict(hd, z=np.r_[1.0, quat_to_rot(i1[15:19]) @ np.array([0.0, 0.0, 1.0])])],
                                  [antenna_item(rng, *state_of(mem[2].e), 7)]])
    batch.close()
    assert [r["status"] for r in res] == [0, 2, 0] and [r["applied"] for r in res] == [1, 0, 1]
    assert_unchanged(snapshot(mem[1].e)[:3], before[1][:3])
    assert not np.array_equal(snapshot(mem[0].e)[2], before[0][2])


def test_runner_with_gnss():
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, gnss_every=1, gnss_delay=2, heading_every=5, gnss_lever=(0.3, -0.2, 0.5))
    s = mc.summarize(rec)
    g = s["gnss"]
    assert len(g["anis"]) >= 50 and all(np.isfinite(g["anis"])) and g["applied"] == 1.0 and g["degenerate"] == 0
    print(f"gnss: ANIS {g['mean_anis']:.3f} per stack ({g['mean_dof']:.2f} dof, run bounds [{g['run_bounds'][0]:.3f}, "
          f"{g['run_bounds'][1]:.3f}]), updates inside {g['updates_inside']:.2f}; ANEES imu "
          f"{s['components']['imu']['mean_anees']:.3f}; position RMSE {s['pos_rmse_run']:.4f} m")
    assert np.isfinite(s["components"]["imu"]["mean_anees"]) and s["pos_rmse_run"] < 1.0
