"""Radio ranges and rangefinder distances in the stacked aided update on the device (msckf_b200_aid_stack_update /
_batch_aid_stack_update with RANGE, CLONE_RANGE, PLANE_RANGE, CLONE_PLANE_RANGE) against numpy fp64 on the fetched covariance
and state: the Joseph-form covariance, the state injection of oracle/msckf_numpy.py and the NIS, with the models of montecarlo.
Also: the device Jacobians against central differences through montecarlo.perturb (read back through a LINEAR update), a stack
mixed with odometry and GNSS against the dense stacked update, batch against single calls bit for bit, refusals and the
degenerate ranges (nothing written), and the runner's ranging."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from oracle.msckf_numpy import quat_to_rot
from tests.test_aid_gpu import CONTRACT, assert_unchanged, snapshot, state_of
from tests.test_batch_stream_gpu import Member
from tests.test_gnss_gpu import H_r as gnss_H_r, antenna_item, heading_item, rel_errors
from tests.test_odometry_gpu import body_item, rel_item

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
RANGES = (capi.AID_RANGE, capi.AID_CLONE_RANGE, capi.AID_PLANE_RANGE, capi.AID_CLONE_PLANE_RANGE)


def H_r(item, imu, poses, n):
    if item["model"] in RANGES:
        return mc.odometry_jacobian(item, imu, poses, n), mc.odometry_residual(item, imu, poses)
    return gnss_H_r(item, imu, poses, n)


def stack_reference(items, imu, poses, P):
    from scipy.linalg import block_diag
    from tests.test_aid_gpu import numpy_update
    Hs, rs = zip(*[H_r(it, imu, poses, P.shape[0]) for it in items])
    return numpy_update(P, imu, poses, np.vstack(Hs), np.concatenate(rs), block_diag(*[it["R"] for it in items]))


def _body(imu, poses, clone):
    return (imu[0:3], imu[15:19]) if clone is None else (poses[clone, 0:3], poses[clone, 3:7])


def range_item(rng, imu, poses, clone=None, scale=0.05, lever=None, anchor=None):
    """a range to an anchor 2..6 m from the body (or at `anchor`), lever in the body frame"""
    lever = rng.normal(size=3) * 0.3 if lever is None else np.asarray(lever, dtype=np.float64)
    p, q = _body(imu, poses, clone)
    if anchor is None:
        u = rng.normal(size=3)
        anchor = p + (2.0 + 4.0 * rng.random()) * u / np.linalg.norm(u)
    z = np.r_[mc.range_of(p, q, lever, anchor) + scale * rng.normal(), anchor, lever]
    R = np.array([[0.005 + 0.01 * rng.random()]])
    if clone is None:
        return {"model": capi.AID_RANGE, "z": z, "R": R}
    return {"model": capi.AID_CLONE_RANGE, "a": clone, "z": z, "R": R}


def plane_item(rng, imu, poses, clone=None, scale=0.02, lever=None, beam=None, dist=None, length=None):
    """a plane range along the beam direction `beam` in G (default: down, tilted by up to ~0.4 rad), the axis given in the body
    frame with a random length, to a level plane that the beam meets dist (1..3 m) from the sensor"""
    lever = rng.normal(size=3) * 0.2 if lever is None else np.asarray(lever, dtype=np.float64)
    p, q = _body(imu, poses, clone)
    beam = np.r_[0.4 * rng.normal(size=2), -1.0] if beam is None else np.asarray(beam, dtype=np.float64)
    beam = beam / np.linalg.norm(beam)
    axis = quat_to_rot(q) @ beam * (0.5 + rng.random() if length is None else length)
    dist = 1.0 + 2.0 * rng.random() if dist is None else dist
    h = mc.antenna_position(p, q, lever)[2] + dist * beam[2]
    z = np.r_[mc.plane_range_of(p, q, h, lever, axis) + scale * rng.normal(), h, lever, axis]
    R = np.array([[0.0004 + 0.001 * rng.random()]])
    if clone is None:
        return {"model": capi.AID_PLANE_RANGE, "z": z, "R": R}
    return {"model": capi.AID_CLONE_PLANE_RANGE, "a": clone, "z": z, "R": R}


def range_cases(rng, imu, poses, M):
    out = [range_item(rng, imu, poses), range_item(rng, imu, poses, lever=np.zeros(3)),
           plane_item(rng, imu, poses, beam=[0.0, 0.0, -1.0], lever=np.zeros(3)), plane_item(rng, imu, poses),
           plane_item(rng, imu, poses, beam=[0.3, -0.2, 1.0])]  # (a ceiling above)
    if M >= 1:
        out += [range_item(rng, imu, poses, clone=0), range_item(rng, imu, poses, clone=M - 1),
                plane_item(rng, imu, poses, clone=M // 2), plane_item(rng, imu, poses, clone=M - 1)]
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_models_match_numpy(dtype):
    """Worst relative differences to numpy measured on an H100 80GB HBM3 (700 W power limit): fp32 P 3.9e-7, state 2.4e-8,
    NIS 2.7e-7, |dx| 1.7e-7; fp64 P 1.0e-15, state 9.1e-17, NIS 2.4e-13, |dx| 1.2e-13"""
    rng = np.random.default_rng(43)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0, "dx": 0.0}
    for M, seed in ((0, 1), (1, 6), (3, 2), (12, 3), (40, 4)):
        base = Member(dtype, M, seed=seed)
        imu, poses = state_of(base.e)
        for item in range_cases(rng, imu, poses, M):
            mem = base.twin(dtype)
            imu_t, poses_t = state_of(mem.e)  # (the reference linearises at the twin's own state)
            P = mem.e.covariance().astype(np.float64)
            res = mem.e.aid_stack_update([item])
            assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == 1
            rel = rel_errors(mem.e, res, stack_reference([item], imu_t, poses_t, P), imu_t)
            for k, v in rel.items():
                assert v <= CONTRACT[name], (M, item["model"], k, v)
                worst[k] = max(worst[k], v)
    print(f"range rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))


def test_jacobians_match_central_differences():
    """H of the four models by central differences of the residual through montecarlo.perturb, against the numpy H and against
    the device: a LINEAR update with the difference quotient gives the covariance the model's update gives"""
    rng = np.random.default_rng(19)
    M = 12
    base = Member(np.float64, M, seed=9)
    n = 15 + 6 * M
    imu, poses = state_of(base.e)
    est = {"imu": imu[0:19], "poses": poses}
    items = [range_item(rng, imu, poses, scale=0.0), range_item(rng, imu, poses, clone=5, scale=0.0),
             plane_item(rng, imu, poses, scale=0.0), plane_item(rng, imu, poses, clone=11, scale=0.0),
             plane_item(rng, imu, poses, clone=0, scale=0.0, beam=[0.5, 0.3, -1.0], lever=[0.2, -0.4, 0.3])]
    eps = 1e-6
    worst = 0.0
    for item in items:
        r0 = mc.odometry_residual(item, imu, poses)
        assert np.abs(r0).max() <= 1e-12
        Hcd = np.zeros((1, n))
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
    print(f"range device H vs central differences: P rel {worst:.3e}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_stack_equals_the_dense_stacked_update(dtype):
    rng = np.random.default_rng(31)
    name = np.dtype(dtype).name
    M = 12
    base = Member(dtype, M, seed=5)
    imu, poses = state_of(base.e)
    items = [range_item(rng, imu, poses) for _ in range(2)] + [range_item(rng, imu, poses, clone=M - 3), plane_item(rng, imu, poses),
             plane_item(rng, imu, poses, clone=M - 2), antenna_item(rng, imu, poses, 7), body_item(rng, imu, 0b111),
             rel_item(rng, poses, M - 2, M - 1)]
    st = base.twin(dtype)
    imu_t, poses_t = state_of(st.e)
    P = st.e.covariance().astype(np.float64)
    res = st.e.aid_stack_update(items)
    assert res["dof"] == 5 + 3 + 3 + 6 and res["applied"] == 1
    rel = rel_errors(st.e, res, stack_reference(items, imu_t, poses_t, P), imu_t)
    print(f"range mixed stack rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in rel.items()))
    for k, v in rel.items():
        assert v <= CONTRACT[name], (k, v)


def _random_stack(rng, imu, poses, M, k):
    """k items (rows <= 32) valid for a window of M clones: range models mixed with GNSS and odometry"""
    out, rows = [], 0
    while len(out) < k:
        kind = rng.integers(0, 8)
        if kind == 0:
            it = range_item(rng, imu, poses)
        elif kind == 1 and M >= 1:
            it = range_item(rng, imu, poses, clone=int(rng.integers(0, M)))
        elif kind == 2:
            it = plane_item(rng, imu, poses)
        elif kind == 3 and M >= 1:
            it = plane_item(rng, imu, poses, clone=int(rng.integers(0, M)))
        elif kind == 4:
            it = antenna_item(rng, imu, poses, int(rng.integers(1, 8)))
        elif kind == 5 and M >= 1:
            it = heading_item(rng, imu, poses, clone=int(rng.integers(0, M)))
        elif kind == 6 and M >= 2:
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
    rng = np.random.default_rng(21)
    mem = [Member(dtype, Ms[i % 4], seed=390 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    stacks = []
    for i, m in enumerate(mem):
        k = [1, 2, 3, 8, 0][i % 5]  # (k = 0: the member is left alone)
        imu, poses = state_of(m.e)
        stacks.append(_random_stack(rng, imu, poses, m.e.num_clones(), k) if k else None)
    assert stacks[32] is not None
    assert {it["model"] for s in stacks if s for it in s} >= set(RANGES)
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


def test_refusals_and_the_degenerate_ranges_write_nothing():
    rng = np.random.default_rng(23)
    M = 4
    mem = [Member(np.float64, M, seed=60 + i) for i in range(3)]
    lib = capi.lib()
    imu, poses = state_of(mem[0].e)
    rg, crg = range_item(rng, imu, poses), range_item(rng, imu, poses, clone=2)
    pl, cpl = plane_item(rng, imu, poses), plane_item(rng, imu, poses, clone=1)
    before = [snapshot(m.e) for m in mem]
    sentinel = capi.AidResult(7.0, 7.0, 7, 7, 7)

    def raw(e, items, chi2_max=0.0):
        arr, keep = capi.aid_items(items)
        out = capi.AidResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_aid_stack_update(e.h, arr, C.c_int(len(items)), C.c_double(chi2_max), C.byref(out)), out

    bad = [dict(crg, a=-1), dict(crg, a=M), dict(cpl, a=-1), dict(cpl, a=M),  # a clone outside the window
           dict(rg, a=1), dict(rg, b=1), dict(crg, b=2), dict(pl, a=3), dict(pl, b=1), dict(cpl, b=1),  # unused a / b
           dict(pl, z=np.r_[pl["z"][0:5], 0.0, 0.0, 0.0]), dict(cpl, z=np.r_[cpl["z"][0:5], 0.0, 0.0, 0.0])]  # a zero beam axis
    for i in range(7):
        z = rg["z"].copy(); z[i] = np.nan
        bad.append(dict(rg, z=z))
        z = crg["z"].copy(); z[i] = np.inf
        bad.append(dict(crg, z=z))
    for i in range(8):
        z = pl["z"].copy(); z[i] = -np.inf
        bad.append(dict(pl, z=z))
        z = cpl["z"].copy(); z[i] = np.nan
        bad.append(dict(cpl, z=z))
    bad += [dict(rg, R=np.array([[np.nan]])), dict(cpl, R=np.array([[np.inf]]))]
    pose = {"model": capi.AID_POSE, "z": np.r_[imu[0:3], imu[15:19]], "R": np.eye(6)}
    stacks = [[b] for b in bad] + [[rg] * 8 + [pl], [pose] * 5 + [rg, crg, pl]]  # 9 items; 33 rows
    for items in stacks:
        rc, out = raw(mem[0].e, items)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), [(it["model"], it.get("a"), it.get("b")) for it in items]
    assert raw(mem[0].e, [rg, pl], chi2_max=np.nan)[0] == -3
    # msckf_b200_aid_update refuses the stack-only models
    for it in (rg, crg, pl, cpl):
        with pytest.raises(RuntimeError, match="rc=-3"):
            mem[0].e.aid_update(it["model"], it["z"], it["R"], clone=it.get("a", 0))
    assert_unchanged(snapshot(mem[0].e), before[0])
    # a range with 7 doubles of z whose last four (the anchor's height and the lever) are zero is not a zero quaternion
    zq = range_item(rng, imu, poses, lever=np.zeros(3), anchor=np.r_[imu[0:2] + [3.0, -1.0], 0.0])
    assert np.all(zq["z"][3:7] == 0.0)
    tw = mem[0].twin(np.float64)  # (held: the twin owns its engine)
    assert tw.e.aid_stack_update([zq])["applied"] == 1
    # degenerate: an antenna on its anchor, a beam parallel to the plane, a plane behind the sensor -- status 2, NIS NaN, nothing
    # written, alone and inside a stack
    lever = np.array([0.2, -0.1, 0.3])
    on_anchor = range_item(rng, imu, poses, lever=lever, anchor=mc.antenna_position(imu[0:3], imu[15:19], lever))
    on_anchor_c = range_item(rng, imu, poses, clone=3, lever=lever, anchor=mc.antenna_position(poses[3, 0:3], poses[3, 3:7], lever))
    level_beam = dict(pl, z=np.r_[1.0, pl["z"][1:5], quat_to_rot(imu[15:19]) @ np.array([0.6, 0.8, 0.0])])
    behind = plane_item(rng, imu, poses, clone=2, dist=-1.0)  # the plane 1 m behind along the beam
    assert mc.range_of(imu[0:3], imu[15:19], lever, on_anchor["z"][1:4]) <= 1e-12
    cases = [[on_anchor], [on_anchor_c], [level_beam], [behind],
             [rg, dict(behind), body_item(rng, imu, 7)], [antenna_item(rng, imu, poses, 7), pl, on_anchor_c], [crg, level_beam, cpl]]
    for items in cases:
        rc, out = raw(mem[0].e, items)
        assert rc == 0 and out.status == 2 and out.applied == 0 and np.isnan(out.nis) and out.dx_norm == 0.0, [it["model"] for it in items]
        assert out.dof == sum(len(it["R"]) for it in items)
    assert_unchanged(snapshot(mem[0].e), before[0])
    # just off parallel (about 2e-3 rad, b_z^2 = 4e-6): a valid plane range, applied
    off = np.array([1.0, 0.0, -2e-3])
    near = dict(pl, z=np.r_[5.0, mc.antenna_position(imu[0:3], imu[15:19], pl["z"][2:5])[2] - 0.01, pl["z"][2:5],
                            quat_to_rot(imu[15:19]) @ (off / np.linalg.norm(off))])
    assert mc.plane_range_of(imu[0:3], imu[15:19], near["z"][1], near["z"][2:5], near["z"][5:8]) > 4.0
    tw2 = mem[0].twin(np.float64)
    r = tw2.e.aid_stack_update([near])
    assert r["status"] == 0 and r["applied"] == 1 and np.isfinite(r["nis"])
    assert_unchanged(snapshot(mem[0].e), before[0])
    # in a batch the degenerate member reports status 2 and is left alone; the others are applied
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_stack_update([[rg], [dict(crg, a=M)], [pl]])
    for m, b in zip(mem, before):
        assert_unchanged(snapshot(m.e), b)
    i1, p1 = state_of(mem[1].e)
    i2, p2 = state_of(mem[2].e)
    res = batch.aid_stack_update([[rg, pl], [range_item(rng, i1, p1), range_item(rng, i1, p1, anchor=mc.antenna_position(i1[0:3], i1[15:19], np.zeros(3)),
                                                                                   lever=np.zeros(3))],
                                  [range_item(rng, i2, p2), plane_item(rng, i2, p2, clone=1)]])
    batch.close()
    assert [r["status"] for r in res] == [0, 2, 0] and [r["applied"] for r in res] == [1, 0, 1]
    assert_unchanged(snapshot(mem[1].e)[:3], before[1][:3])
    assert not np.array_equal(snapshot(mem[0].e)[2], before[0][2]) and not np.array_equal(snapshot(mem[2].e)[2], before[2][2])


def test_runner_with_ranging():
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, range_every=1, range_delay=2, plane_every=1)
    s = mc.summarize(rec)
    g = s["range"]
    assert len(g["anis"]) >= 50 and all(np.isfinite(g["anis"])) and g["applied"] == 1.0 and g["degenerate"] == 0
    assert g["mean_dof"] == 5.0 and "gnss" not in s
    base, _ = mc.run(range(8), truth, dtype=np.float64)
    s0 = mc.summarize(base)
    print(f"range: ANIS {g['mean_anis']:.3f} per stack ({g['mean_dof']:.2f} dof, run bounds [{g['run_bounds'][0]:.3f}, "
          f"{g['run_bounds'][1]:.3f}]), updates inside {g['updates_inside']:.2f}; ANEES imu "
          f"{s['components']['imu']['mean_anees']:.3f}; position RMSE {s['pos_rmse_run']:.4f} m against {s0['pos_rmse_run']:.4f} m "
          f"without aids")
    assert np.isfinite(s["components"]["imu"]["mean_anees"]) and s["pos_rmse_run"] < s0["pos_rmse_run"]
