"""Stacked aided updates on the device (msckf_b200_aid_stack_update / _batch_aid_stack_update, MSCKF::aidedUpdate(items),
MSCKFBatch::aidedUpdate(items)) with the odometry models BODY_VELOCITY and RELATIVE_POSE, against numpy fp64 on the fetched
covariance and state: the Joseph-form covariance, the state injection of oracle/msckf_numpy.py and the NIS.  Also: the model
Jacobians against central differences through montecarlo.perturb (read back through a LINEAR update), a stack of one against
msckf_b200_aid_update, a stack of three against the dense stacked update, batch against single calls bit for bit, updates that
must write nothing, ERR_NUMERIC and the runner's odometry."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import block_diag

from msckf_mono_b200 import capi, montecarlo as mc
from msckf_mono_b200.montecarlo import odometry_jacobian as jacobian, odometry_residual as residual
from oracle.msckf_numpy import quat_to_rot
from tests.test_aid_gpu import CONTRACT, assert_unchanged, make_spec, numpy_update, snapshot, spd, state_of
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]


def H_r(item, imu, poses, n):
    """(H, r) of any stack item"""
    if item["model"] in (capi.AID_BODY_VELOCITY, capi.AID_RELATIVE_POSE):
        return jacobian(item, imu, poses, n), residual(item, imu, poses)
    spec = dict(item, clone=item.get("a", 0))
    z = np.asarray(item["z"], dtype=np.float64)
    if item["model"] in (capi.AID_VELOCITY, capi.AID_POSITION):
        o, c = (3, 6) if item["model"] == capi.AID_VELOCITY else (0, 12)
        r, cols = z - imu[o:o + 3], list(range(c, c + 3))
    else:
        p, q = (imu[0:3], imu[15:19]) if item["model"] == capi.AID_POSE else (poses[spec["clone"], 0:3], poses[spec["clone"], 3:7])
        r = np.concatenate([mc.quat_error(z[3:7], q), z[0:3] - p])
        cols = [0, 1, 2, 12, 13, 14] if item["model"] == capi.AID_POSE else list(range(15 + 6 * spec["clone"], 21 + 6 * spec["clone"]))
    H = np.zeros((len(r), n))
    H[np.arange(len(r)), cols] = 1.0
    return H, r


def body_item(rng, imu, mask, scale=0.1):
    rows = [j for j in range(3) if (mask >> j) & 1]
    v = quat_to_rot(imu[15:19]) @ imu[3:6]
    return {"model": capi.AID_BODY_VELOCITY, "a": mask, "z": v + scale * rng.normal(size=3), "R": spd(rng, len(rows), 0.02)}


def rel_item(rng, poses, a, b, scale=0.05):
    p, q = mc.relative_pose(poses[a], poses[b])
    q = mc.quat_mul(mc.quat_of_error(scale * rng.normal(size=3)), q)
    return {"model": capi.AID_RELATIVE_POSE, "a": a, "b": b, "z": np.r_[p + scale * rng.normal(size=3), q / np.linalg.norm(q)],
            "R": spd(rng, 6, 0.02)}


def stack_reference(items, imu, poses, P):
    n = P.shape[0]
    Hs, rs = zip(*[H_r(it, imu, poses, n) for it in items])
    return numpy_update(P, imu, poses, np.vstack(Hs), np.concatenate(rs), block_diag(*[it["R"] for it in items]))


def rel_errors(e, res, ref, imu0):
    Pr, imur, posesr, nisr, dxr = ref
    Pd = e.covariance()
    assert np.array_equal(Pd, Pd.T)
    imud, posesd = state_of(e)
    assert np.array_equal(imud[19:29], imu0[19:29])  # the observability copies are not touched
    sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([imur[0:19], posesr.ravel()])
    assert abs(res["dx_norm"] - dxr) <= 1e-9 * dxr
    return {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(), "state": np.abs(sd - sr).max() / np.abs(sr).max(),
            "nis": abs(res["nis"] - nisr) / nisr}


@pytest.mark.parametrize("dtype", DTYPES)
def test_models_match_numpy(dtype):
    rng = np.random.default_rng(31)
    name = np.dtype(dtype).name
    worst = {"P": 0.0, "state": 0.0, "nis": 0.0}
    for M, seed in ((0, 1), (3, 2), (12, 3), (40, 4)):
        base = Member(dtype, M, seed=seed)
        cases = [("bv", m) for m in (0b111, 0b110, 0b001)]
        if M >= 2:
            cases += [("rel", (0, M - 1)), ("rel", (M - 1, 0)), ("rel", (M // 2, 1 if M // 2 != 1 else 0))]
        for kind, arg in cases:
            mem = base.twin(dtype)
            imu, poses = state_of(mem.e)
            P = mem.e.covariance().astype(np.float64)
            item = body_item(rng, imu, arg) if kind == "bv" else rel_item(rng, poses, *arg)
            res = mem.e.aid_stack_update([item])
            assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == len(residual(item, imu, poses))
            rel = rel_errors(mem.e, res, stack_reference([item], imu, poses, P), imu)
            for k, v in rel.items():
                assert v <= CONTRACT[name], (M, kind, arg, k, v)
                worst[k] = max(worst[k], v)
    print(f"odometry rel vs numpy {name}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))


def test_jacobians_match_central_differences():
    """H of both models by central differences of the residual through montecarlo.perturb (the inverse of the error-state
    convention), against the numpy H above and against the device: a LINEAR update with the difference quotient gives the
    covariance the model's update gives (P does not depend on r)"""
    rng = np.random.default_rng(17)
    M = 12
    base = Member(np.float64, M, seed=9)
    n = 15 + 6 * M
    imu, poses = state_of(base.e)
    est = {"imu": imu[0:19], "poses": poses}
    # (at zero residual: the rotation rows' H, like POSE's, is the derivative there)
    for item in (body_item(rng, imu, 0b111, 0.0), body_item(rng, imu, 0b110, 0.0), rel_item(rng, poses, 3, 8, 0.0),
                 rel_item(rng, poses, 11, 2, 0.0)):
        eps = 1e-6
        Hcd = np.zeros((len(residual(item, imu, poses)), n))
        for k in range(n):
            e = np.zeros(n); e[k] = eps
            sp, sm = mc.perturb(est, e), mc.perturb(est, -e)
            Hcd[:, k] = -(residual(item, sp["imu"], sp["poses"]) - residual(item, sm["imu"], sm["poses"])) / (2 * eps)
        Ha = jacobian(item, imu, poses, n)
        assert np.abs(Hcd - Ha).max() <= 1e-6, np.abs(Hcd - Ha).max()
        a, b = base.twin(np.float64), base.twin(np.float64)
        a.e.aid_stack_update([item])
        b.e.aid_update(capi.AID_LINEAR, residual(item, imu, poses), item["R"], H=Hcd)
        Pa, Pb = a.e.covariance(), b.e.covariance()
        assert np.abs(Pa - Pb).max() <= 1e-8 * np.abs(Pa).max(), np.abs(Pa - Pb).max()


@pytest.mark.parametrize("dtype", DTYPES)
def test_stack_of_one_equals_aid_update(dtype):
    rng = np.random.default_rng(5)
    M = 12
    base = Member(dtype, M, seed=7)
    n = 15 + 6 * M
    for model, clone in ((capi.AID_VELOCITY, 0), (capi.AID_POSITION, 0), (capi.AID_POSE, 0), (capi.AID_CLONE_POSE, 4)):
        a, b = base.twin(dtype), base.twin(dtype)
        imu, poses = state_of(a.e)
        spec = make_spec(rng, model, imu, poses, n, clone)[0]
        ra = a.e.aid_update(model, spec["z"], spec["R"], clone=clone)
        rb = b.e.aid_stack_update([{"model": model, "a": clone, "z": spec["z"], "R": spec["R"]}])
        assert ra == rb, model
        for x, y in zip(snapshot(a.e), snapshot(b.e)):
            assert np.array_equal(x, y), model


@pytest.mark.parametrize("dtype", DTYPES)
def test_stack_of_three_equals_the_dense_stacked_update(dtype):
    rng = np.random.default_rng(23)
    name = np.dtype(dtype).name
    M = 12
    base = Member(dtype, M, seed=5)
    imu, poses = state_of(base.e)
    P = base.e.covariance().astype(np.float64)
    items = [body_item(rng, imu, 0b111), rel_item(rng, poses, M - 2, M - 1),
             {"model": capi.AID_POSITION, "z": imu[0:3] + 0.1 * rng.normal(size=3), "R": spd(rng, 3, 0.02)}]
    st = base.twin(dtype)
    res = st.e.aid_stack_update(items)
    assert res["dof"] == 12 and res["applied"] == 1
    rel = rel_errors(st.e, res, stack_reference(items, imu, poses, P), imu)
    for k, v in rel.items():
        assert v <= CONTRACT[name], (k, v)
    # three sequential updates re-linearise at the updated state: outside the stacked update's bounds
    Pr, imur, posesr = stack_reference(items, imu, poses, P)[:3]
    sq = base.twin(dtype)
    for it in items:
        sq.e.aid_stack_update([it])
    imuq, posesq = state_of(sq.e)
    sr, sqs = np.concatenate([imur[0:19], posesr.ravel()]), np.concatenate([imuq[0:19], posesq.ravel()])
    dP = np.abs(sq.e.covariance().astype(np.float64) - Pr).max() / np.abs(Pr).max()
    ds = np.abs(sqs - sr).max() / np.abs(sr).max()
    print(f"sequential vs stacked {name}: P {dP:.3e} state {ds:.3e}")
    assert max(dP, ds) > 10 * CONTRACT[name]


def _random_stack(rng, imu, poses, M, k):
    """k items (rows <= 32) valid for a window of M clones"""
    out, rows = [], 0
    while len(out) < k:
        kind = rng.integers(0, 6)
        if kind == 0:
            it = body_item(rng, imu, int(rng.integers(1, 8)))
        elif kind == 1 and M >= 2:
            a, b = rng.choice(M, size=2, replace=False)
            it = rel_item(rng, poses, int(a), int(b))
        elif kind == 2 and M >= 1:
            it = dict(make_spec(rng, capi.AID_CLONE_POSE, imu, poses, 15 + 6 * M, int(rng.integers(0, M)))[0])
            it["a"] = it.pop("clone")
        else:
            model = (capi.AID_VELOCITY, capi.AID_POSITION, capi.AID_POSE)[kind % 3]
            it = make_spec(rng, model, imu, poses, 15 + 6 * M)[0]
        m = len(it["R"])
        if rows + m > 32:
            break
        rows += m
        out.append(it)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_bit_for_bit(dtype):
    Ms = [0, 5, 30, 90]
    rng = np.random.default_rng(8)
    mem = [Member(dtype, Ms[i % 4], seed=190 + i, max_clones=Ms[i % 4] + 2) for i in range(33)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    stacks = []
    for i, m in enumerate(mem):
        k = [1, 2, 3, 8, 0][i % 5]  # (k = 0: the member is left alone)
        imu, poses = state_of(m.e)
        stacks.append(_random_stack(rng, imu, poses, m.e.num_clones(), k) if k else None)
    assert stacks[32] is not None  # (a member past the first chunk of 32 is updated)
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


def test_updates_that_write_nothing():
    rng = np.random.default_rng(13)
    mem = [Member(np.float64, 4, seed=30 + i) for i in range(3)]
    lib = capi.lib()
    imu, poses = state_of(mem[0].e)
    good = [body_item(rng, imu, 0b110), rel_item(rng, poses, 0, 3)]
    before = [snapshot(m.e) for m in mem]
    # gated out: NIS reported, nothing applied
    r = mem[0].e.aid_stack_update(good, chi2_max=1e-12)
    assert r["applied"] == 0 and r["status"] == 0 and r["nis"] > 1e-12 and r["dx_norm"] == 0.0 and r["dof"] == 8
    # S not positive definite
    r = mem[0].e.aid_stack_update([good[0], dict(good[1], R=-1e6 * np.eye(6))])
    assert r["status"] == 1 and r["applied"] == 0 and np.isnan(r["nis"])
    assert_unchanged(snapshot(mem[0].e), before[0])
    sentinel = capi.AidResult(7.0, 7.0, 7, 7, 7)

    def raw(e, items, chi2_max=0.0):
        arr, keep = capi.aid_items(items)
        out = capi.AidResult.from_buffer_copy(sentinel)
        return lib.msckf_b200_aid_stack_update(e.h, arr, C.c_int(len(items)), C.c_double(chi2_max), C.byref(out)), out

    rel = good[1]
    R_lower_nan = np.eye(6); R_lower_nan[5, 0] = np.nan
    bad = [[dict(rel, model=capi.AID_LINEAR)], [dict(rel, model=9)], [dict(rel, b=4)], [dict(rel, a=-1)], [dict(rel, b=0)],
           [dict(good[0], a=0)], [dict(good[0], a=8)], [rel] * 6, [good[0]] * 9, [dict(rel, z=np.r_[rel["z"][0:3], 0, 0, 0, 0])],
           [dict(good[0], z=[0.0, np.nan, 0.0])], [dict(rel, R=R_lower_nan)], [good[0], {"model": capi.AID_CLONE_POSE, "a": 4,
                                                                                         "z": rel["z"], "R": np.eye(6)}], []]
    for items in bad:
        rc, out = raw(mem[0].e, items)
        assert rc == -3 and out.as_dict() == sentinel.as_dict(), items
    assert raw(mem[0].e, good, chi2_max=np.nan)[0] == -3
    R_upper_nan = np.eye(6); R_upper_nan[0, 5] = np.nan  # (only the lower triangle is read: valid)
    assert mem[0].e.aid_stack_update([dict(rel, R=R_upper_nan)])["applied"] == 1
    before[0] = snapshot(mem[0].e)
    # a batch with one bad member changes no member
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_stack_update([good, [dict(rel, b=0)], good])
    # an un-fetched update (a triangulation of one track) on member 1
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    launched = mem[1].e.launch_count()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.aid_stack_update([good, None, good])
    rc, out = raw(mem[1].e, good)
    assert rc == -5 and out.as_dict() == sentinel.as_dict()
    assert mem[1].e.launch_count() == launched
    mem[1].e.fetch(1)  # (a triangulation writes neither P nor the state)
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)
    batch.close()


def test_non_finite_covariance_is_reported_and_applied():
    rng = np.random.default_rng(4)
    mem = Member(np.float64, 4, seed=3)
    P = mem.e.covariance()
    P[30, 30] = np.inf  # outside the rows a body velocity reads: only the downdate meets it
    mem.e.set_covariance(P)
    imu, _ = state_of(mem.e)
    with pytest.raises(RuntimeError, match="rc=-6"):
        mem.e.aid_stack_update([body_item(rng, imu, 0b111)])
    assert not np.array_equal(state_of(mem.e)[0], imu)  # applied, like the vision update's ERR_NUMERIC


def test_runner_with_odometry():
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, odo_every=1)
    s = mc.summarize(rec)
    o = s["odometry"]
    assert len(o["anis"]) == 60 and all(np.isfinite(o["anis"])) and o["applied"] == 1.0
    print(f"odometry: ANIS {o['mean_anis']:.3f} per stack ({o['mean_dof']:.2f} dof, run bounds [{o['run_bounds'][0]:.3f}, "
          f"{o['run_bounds'][1]:.3f}]), updates inside {o['updates_inside']:.2f}; ANEES imu "
          f"{s['components']['imu']['mean_anees']:.3f}; position RMSE {s['pos_rmse_run']:.4f} m")
    lo, hi = o["run_bounds"]
    assert lo <= o["mean_anis"] <= hi
