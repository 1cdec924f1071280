"""The side updates at every window, row count, storage path and cap their kernels dispatch on (tests/side_shapes.py), in fp64
and fp32, against dense fp64 references on the engine's fetched state:
  * k_aid: each row count 1 .. 32 at its last window with W^T and dx in shared memory and its first with them in the global
    workspace, as one LINEAR call and one stack of model items; windows 0, 1, 191, 192; the chi2 gate 1e-6 either side of the
    NIS on both paths; a 33-member device batch whose first launch chunk mixes both paths; the shared memory of each path's
    launch in a profiler trace, plain and FDE (its launch past the default 48 KB);
  * k_nees: windows of 19 .. 192 clones (1 .. 37 panels of the factor), with and without truth poses, a 33-member batch, and a
    first bad pivot past the first panel;
  * k_lmk_*: exact-map rows 30 .. 1152 across the panel edges of k_lmk_gain's factor and k_lmk_downdate's loop, windows 91 ..
    192, 255 and 256 observations of one clone, 4096 of one member (against the information form), gating that leaves the
    used rows a panel below the planned stride, the iterated form at 180 and 1152 rows; map uncertainty with 8-clone groups at
    the end of the window, a group of 256 observations, 256 groups, 1152 rows through groups and the call one step past it;
    a 33-member batch of large and small members.
Integer outputs are compared exactly, P must be exactly symmetric and the observability copies untouched; floating-point
differences are held to the side updates' ceilings and to 10 x the measurement below."""
import json
import os
import tempfile

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from tests import aid_fde_reference as fde_ref, landmark_map_reference as mref, side_shapes as ss
from tests.landmark_iter_reference import iekf
from tests.test_aid_gpu import assert_unchanged, call, make_spec, numpy_update, snapshot, state_of
from tests.test_batch_stream_gpu import Member
from tests.test_gnss_gpu import antenna_item, heading_item, rel_errors as aid_rel_errors, stack_reference
from tests.test_landmark_gpu import R_PIX, dense, make_obs
from tests.test_landmark_iter_gpu import drifted_obs
from tests.test_landmark_map_gpu import scene
from tests.test_nees_gpu import KEYS as NEES_KEYS, as_row, est_of, numpy_nees
from tests.test_odometry_gpu import body_item, rel_item

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
CONTRACT = {"float32": 1e-5, "float64": 1e-9}  # P, the state, the NIS (and |dx|, gamma): fp64 arithmetic, one rounding to the type
# worst relative differences to the references, measured on an H100 80GB HBM3 (700 W power limit) by this file; asserted at 10 x
# (fp32: P and the state are rounded to float32 once; aid's NIS and |dx| are the GNSS models' residuals at the float32 state)
MEASURED = {
    "aid": {"float32": {"P": 2.35e-7, "state": 5.55e-8, "nis": 5.74e-7, "dx": 1.84e-7},
            "float64": {"P": 3.89e-14, "state": 1.87e-15, "nis": 5.06e-14, "dx": 2.75e-14}},
    "nees": {"float32": {"nees": 2.53e-15}, "float64": {"nees": 6.31e-15}},
    "lmk": {"float32": {"P": 5.66e-8, "state": 5.11e-8, "nis": 5.76e-11, "dx": 7.45e-10, "gamma": 7.95e-16},
            "float64": {"P": 4.05e-14, "state": 1.77e-12, "nis": 3.22e-11, "dx": 4.20e-10, "gamma": 1.86e-12}},
    "lmk_iter": {"float32": {"P": 5.50e-8, "state": 4.87e-8, "nis": 3.62e-12, "dx": 3.55e-12, "gamma": 4.99e-16},
                 "float64": {"P": 6.51e-12, "state": 3.38e-12, "nis": 4.53e-12, "dx": 1.79e-12, "gamma": 1.13e-14}},
    "map": {"float32": {"P": 5.62e-8, "state": 4.92e-8, "nis": 9.18e-12, "dx": 3.57e-10, "gamma": 6.49e-16},
            "float64": {"P": 2.01e-12, "state": 1.63e-12, "nis": 4.20e-11, "dx": 3.02e-10, "gamma": 4.40e-12}},
}
CHI2 = 1e-3  # gamma of an observation pushed 0.5 off is ~0.1 at these P; of one at the pixel noise, ~1e-5
_BASE = {}


def cap(M):
    """max_clones of a window of M (the default M + 8 passes the hard limit of 192 from 185 clones on)"""
    return min(M + 2, ss.K["kMaxKeep"])


def base(dtype, M):
    """one engine per (dtype, window), built once; tests that write take a twin"""
    key = (np.dtype(dtype).name, M)
    if key not in _BASE:
        _BASE[key] = Member(dtype, M, seed=500 + M, max_clones=cap(M))
    return _BASE[key]


def fresh(dtype, M):
    return base(dtype, M).twin(dtype, max_clones=cap(M))


def settle(worst, rel, name, where):
    for k, v in rel.items():
        assert v <= CONTRACT[name], (where, k, v)
        worst[k] = max(worst.get(k, 0.0), v)


def assert_measured(group, name, worst):
    print(f"MEASURED {group} {name} " + json.dumps({k: float(f"{v:.3g}") for k, v in worst.items()}))
    for k, v in worst.items():
        assert v <= 10 * MEASURED[group][name][k], (group, k, v, MEASURED[group][name][k])


# ---- k_aid -------------------------------------------------------------------------------------------------------------
def stack_items(rng, recipe, imu, poses, M):
    items = []
    for model, rows, clone in recipe:
        k = M - 1 if clone == -1 else clone
        if model == "CLONE_HEADING":
            it = heading_item(rng, imu, poses, clone=k)
        elif model == "HEADING":
            it = heading_item(rng, imu, poses)
        elif model == "CLONE_ANTENNA_POSITION":
            it = antenna_item(rng, imu, poses, 7, clone=k)
        elif model == "ANTENNA_POSITION":
            it = antenna_item(rng, imu, poses, 7)
        elif model == "RELATIVE_POSE":
            it = rel_item(rng, poses, 0, M - 1)
        elif model == "BODY_VELOCITY":
            it = body_item(rng, imu, 0b111)
        else:  # CLONE_POSE, POSE, VELOCITY
            it = dict(make_spec(rng, getattr(capi, "AID_" + model), imu, poses, ss.n_of(M), k or 0)[0])
            it["a"] = it.pop("clone")
        assert len(it["R"]) == rows, model
        items.append(it)
    return items


def aid_checked(name, e, res, ref, imu0, m):
    assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == m, res
    return aid_rel_errors(e, res, ref, imu0)  # (P symmetric, observability copies untouched)


@pytest.mark.parametrize("dtype", DTYPES)
def test_aid_at_both_storage_paths(dtype):
    rng = np.random.default_rng(61)
    name = np.dtype(dtype).name
    worst = {}
    for M, m in ss.aid_cases():
        b = base(dtype, M)
        imu, poses = state_of(b.e)
        P = b.e.covariance().astype(np.float64)
        where = (M, m, "global" if ss.aid_global(M, m) else "shared")
        # one LINEAR call
        spec, H, r = make_spec(rng, capi.AID_LINEAR, imu, poses, ss.n_of(M), m=m)
        ref = numpy_update(P, imu, poses, H, r, spec["R"])
        lin = fresh(dtype, M)
        settle(worst, aid_checked(name, lin.e, call(lin.e, spec), ref, imu, m), name, where + ("LINEAR",))
        # the gate 1e-6 either side of the reference NIS: applied (bit for bit the ungated call) or nothing written
        for f, applied in ((1 + 1e-6, 1), (1 - 1e-6, 0)):
            g = fresh(dtype, M)
            before = snapshot(g.e)
            res = call(g.e, dict(spec, chi2_max=ref[3] * f))
            assert res["applied"] == applied and res["status"] == 0 and res["dof"] == m, (where, f, res)
            if applied:
                for x, y in zip(snapshot(g.e)[:3], snapshot(lin.e)[:3]):
                    assert np.array_equal(x, y), where
            else:
                assert res["dx_norm"] == 0.0 and abs(res["nis"] - ref[3]) <= CONTRACT[name] * ref[3]
                assert_unchanged(snapshot(g.e), before)
        # one stack of model items with the same m
        items = stack_items(rng, ss.aid_stack(M, m), imu, poses, M)
        st = fresh(dtype, M)
        res = st.e.aid_stack_update(items)
        settle(worst, aid_checked(name, st.e, res, stack_reference(items, imu, poses, P), imu, m), name, where + ("stack",))
    assert_measured("aid", name, worst)


@pytest.mark.parametrize("dtype", DTYPES)
def test_aid_batch_mixing_both_paths(dtype):
    rng = np.random.default_rng(62)
    name = np.dtype(dtype).name
    worst = {}
    mem = [fresh(dtype, M) for M, _ in ss.AID_BATCH]
    twins = [fresh(dtype, M) for M, _ in ss.AID_BATCH]
    specs, refs = [], []
    for (M, m), b in zip(ss.AID_BATCH, mem):
        imu, poses = state_of(b.e)
        P = b.e.covariance().astype(np.float64)
        spec, H, r = make_spec(rng, capi.AID_LINEAR, imu, poses, ss.n_of(M), m=m)
        specs.append(spec)
        refs.append((numpy_update(P, imu, poses, H, r, spec["R"]), imu))
    single = [call(t.e, s) for t, s in zip(twins, specs)]
    batch = capi.Batch([b.e for b in mem])
    got = batch.aid_update(specs)
    batch.close()
    for i, ((M, m), b, t) in enumerate(zip(ss.AID_BATCH, mem, twins)):
        assert got[i] == single[i], i
        for x, y in zip(b.e.state() + (b.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i
        settle(worst, aid_checked(name, b.e, got[i], refs[i][0], refs[i][1], m), name, (i, M, m))
    assert_measured("aid", name, worst)


def test_aid_launch_shared_memory_follows_the_storage_path():
    """k_aid's shared memory per launch in a torch.profiler trace: the launch of a member on the shared side carries
    aid_ws_bytes(n, m) dynamic bytes more than the launch of a member on the global side"""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    M0, M1 = ss.AID_EDGES[3]
    cases = [(M0, 3), (M1, 3)]
    mems = [fresh(np.float64, M) for M, _ in cases]
    rng = np.random.default_rng(63)
    specs = []
    for (M, m), b in zip(cases, mems):
        imu, poses = state_of(b.e)
        specs.append(make_spec(rng, capi.AID_LINEAR, imu, poses, ss.n_of(M), m=m)[0])
    torch.cuda.init()
    smem = []
    with tempfile.TemporaryDirectory() as tmp:
        for b, s in zip(mems, specs):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(b.e, s)
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as fh:
                ev = [e for e in json.load(fh).get("traceEvents", []) if "k_aid" in str(e.get("name", ""))]
            if not ev or "shared memory" not in ev[0].get("args", {}):
                pytest.skip("the profiler trace carries no k_aid launch with its shared memory")
            smem.append(int(ev[0]["args"]["shared memory"]))
    assert ss.aid_global(M1, 3) and not ss.aid_global(M0, 3)
    assert smem[0] - smem[1] == ss.aid_dynamic_smem(M0, 3) == ss.aid_ws_bytes(ss.n_of(M0), 3), smem


def test_aid_fde_launch_shared_memory_past_the_default_limit():
    """the same for k_aid<S, 1, true> at the same two windows (m = 3 at window 168 is one of ss.AID_OPT_IN): the shared-side
    launch carries aid_ws_bytes(n, 3) more, and where the trace counts static shared memory, it is over the default 48 KB"""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    M0, M1 = ss.AID_EDGES[3]
    assert (M0, 3) in ss.AID_OPT_IN
    rng = np.random.default_rng(76)
    chi2 = capi.fde_thresholds(0.01)
    torch.cuda.init()
    smem = []
    with tempfile.TemporaryDirectory() as tmp:
        for M in (M0, M1):
            b = fresh(np.float64, M)
            imu, poses = state_of(b.e)
            items = fde_ref.recipe_items(rng, ss.fde_stack(M, 3), imu, poses, M)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                got = b.e.aid_stack_update(items, fde={"chi2": chi2, "max_exclude": 1})
            assert got["applied"] == 1
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as fh:
                ev = [e for e in json.load(fh).get("traceEvents", []) if "k_aid" in str(e.get("name", ""))]
            if not ev or "shared memory" not in ev[0].get("args", {}):
                pytest.skip("the profiler trace carries no k_aid launch with its shared memory")
            smem.append(int(ev[0]["args"]["shared memory"]))
    print(f"k_aid FDE launch shared memory: window {M0} {smem[0]} B, window {M1} {smem[1]} B")
    assert ss.aid_global(M1, 3) and not ss.aid_global(M0, 3)
    assert smem[0] - smem[1] == ss.aid_ws_bytes(ss.n_of(M0), 3), smem
    if smem[1] >= ss.AID_STATIC_SMEM["fde"]:
        assert smem[0] > ss.AID_DEFAULT_SMEM, smem


# ---- k_nees ------------------------------------------------------------------------------------------------------------
def nees_perm(n):
    """engine index of each NEES-order index: [dtheta_I, dp_I, dv, db_g, db_a, clones] from [dtheta, db_g, dv, db_a, dp, clones]"""
    head = [o + r for o in (0, 12, 6, 3, 9) for r in range(3)]
    return np.array(head + list(range(15, n)))


def first_bad_pivot(P):
    """the first non-positive pivot of P's Cholesky factor: the smallest j whose leading (j + 1) block does not factor"""
    def ok(j):
        try:
            np.linalg.cholesky(P[:j, :j])
            return True
        except np.linalg.LinAlgError:
            return False
    if ok(len(P)):
        return -1
    lo, hi = 0, len(P)  # ok(lo), not ok(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


def nees_rel(r, ref, full):
    out = {}
    for k in NEES_KEYS:
        if k == "full" and not full:
            assert np.isnan(r[k])
            continue
        out[k] = abs(r[k] - ref[k]) / ref[k]
    return {"nees": max(out.values())}


@pytest.mark.parametrize("dtype", DTYPES)
def test_nees_at_every_panel_count(dtype):
    rng = np.random.default_rng(64)
    name = np.dtype(dtype).name
    worst = {}
    truths, refs = [], []
    for M in ss.NEES_WINDOWS:
        m = base(dtype, M)
        n = ss.n_of(M)
        est = est_of(m.e)
        truth = mc.perturb(est, 0.05 * rng.standard_normal(n))
        ref = numpy_nees(m.e.covariance().astype(np.float64), mc.error_state(truth, est), True)
        for poses in (truth["poses"], None):
            r = m.e.nees(truth["imu"], poses)
            assert r["first_bad_pivot"] == -1 and r["dim_full"] == (n if poses is not None else 0), (M, r)
            settle(worst, nees_rel(r, ref, poses is not None), name, M)
        truths.append(truth)
        refs.append(ref)
    # one batch of 33 members over these windows (two launch chunks), every third without truth poses
    W = len(ss.NEES_WINDOWS)
    mem = [fresh(dtype, ss.NEES_WINDOWS[i % W]) for i in range(33)]
    tp = [None if i % 3 == 0 else truths[i % W]["poses"] for i in range(33)]
    single = [as_row(m.e.nees(truths[i % W]["imu"], tp[i])) for i, m in enumerate(mem)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.nees([truths[i % W]["imu"] for i in range(33)], tp)
    batch.close()
    for i, r in enumerate(got):
        assert np.array_equal(as_row(r), single[i], equal_nan=True), i
        assert r["first_bad_pivot"] == -1
        settle(worst, nees_rel(r, refs[i % W], tp[i] is not None), name, (i, ss.NEES_WINDOWS[i % W]))
    assert_measured("nees", name, worst)


@pytest.mark.parametrize("dtype", DTYPES)
def test_nees_first_bad_pivot_past_the_first_panel(dtype):
    rng = np.random.default_rng(65)
    M, k = ss.NEES_BREAK
    n = ss.n_of(M)
    b0 = 15 + 6 * k
    for rows in (slice(b0, b0 + 6), slice(b0 + 3, b0 + 4)):  # the clone's whole block; one diagonal entry inside it
        m = fresh(dtype, M)
        P = m.e.covariance().astype(np.float64)
        P[rows, rows] = -1e3 * np.eye(rows.stop - rows.start)
        m.e.set_covariance(P)
        P = m.e.covariance().astype(np.float64)
        est = est_of(m.e)
        truth = mc.perturb(est, 0.02 * rng.standard_normal(n))
        r = m.e.nees(truth["imu"], truth["poses"])
        p = nees_perm(n)
        want = first_bad_pivot(P[np.ix_(p, p)])
        assert want == rows.start and r["first_bad_pivot"] == want, (r["first_bad_pivot"], want)
        assert ss.chunks(want + 1) > 1 and np.isnan(r["full"]) and r["dim_full"] == n
        ref = numpy_nees(P, mc.error_state(truth, est), False)
        for key in ("orientation", "position", "pose", "imu"):
            assert np.isfinite(r[key]) and abs(r[key] - ref[key]) <= 1e-9 * ref[key], (key, r[key], ref[key])


# ---- mapped landmarks, exact map ---------------------------------------------------------------------------------------
def lmk_obs(rng, poses, counts, push=(), behind=None):
    """make_obs of `counts`; the observations of the clones in `push` moved 0.5 off (gated at CHI2); `behind` (clone -> count)
    adds landmarks behind those clones (flag 2)"""
    clone, z, p_L = make_obs(rng, poses, counts)
    for k in push:
        z[clone == k] += 0.5
    if behind:
        bc, bz, bp = make_obs(rng, poses, behind)
        bp = np.array([2 * poses[k, 0:3] - pl for k, pl in zip(bc, bp)])
        clone, z, p_L = np.concatenate([clone, bc]), np.vstack([z, bz]), np.vstack([p_L, bp])
        o = rng.permutation(len(clone))
        clone, z, p_L = clone[o], z[o], p_L[o]
    return clone, z, p_L


def lmk_reference(P, imu, poses, clone, z, p_L, chi2):
    """(the update's tuple, gamma, flag): the dense Joseph form, or the information form past 2048 rows (dense() taken over
    chunks of observations: it builds R (x) I of all it is given)"""
    parts = [dense(P, poses, clone[i:i + 512], z[i:i + 512], p_L[i:i + 512], R_PIX, chi2) for i in range(0, len(clone), 512)]
    H, r = np.vstack([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    gam, flag = np.concatenate([p[3] for p in parts]), np.concatenate([p[4] for p in parts])
    if chi2 > 0:  # no observation near the gate
        ok = np.isfinite(gam)
        assert np.all(np.abs(np.log(gam[ok] / chi2)) > 0.5)
    if len(r) > 2048:
        return ss.information_update(P, imu, poses, H, r, np.broadcast_to(R_PIX, (len(r) // 2, 2, 2))), gam, flag
    return numpy_update(P, imu, poses, H, r, np.kron(np.eye(len(r) // 2), R_PIX)), gam, flag


def lmk_checked(res, e, ref, gam, flag, imu0, rows):
    assert np.array_equal(res["flag"], flag)
    used = int(np.sum(flag == 0))
    assert res["used"] == used and res["dof"] == 2 * used and res["rows"] == rows, (res["rows"], rows)
    assert res["applied"] == 1 and res["status"] == 0
    Pr, imur, posesr, nisr, dxr = ref
    Pd = e.covariance()
    assert np.array_equal(Pd, Pd.T)
    imud, posesd = state_of(e)
    assert np.array_equal(imud[19:29], imu0[19:29])  # the observability copies are not touched
    sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([imur[0:19], posesr.ravel()])
    ok = np.isfinite(gam)
    assert np.array_equal(np.isfinite(res["gamma"]), ok)
    return {"P": np.abs(Pd.astype(np.float64) - Pr).max() / np.abs(Pr).max(), "state": np.abs(sd - sr).max() / np.abs(sr).max(),
            "nis": abs(res["nis"] - nisr) / nisr, "dx": abs(res["dx_norm"] - dxr) / dxr,
            "gamma": float(np.max(np.abs(res["gamma"][ok] - gam[ok]) / gam[ok]))}


def lmk_cases(M0):
    """(M, counts, push, behind, rows) of the single exact-map calls; push and behind as lmk_obs"""
    out = [(M0, ss.sweep_counts(M0, rows), (), None, rows) for rows in ss.LMK_SWEEP_ROWS]
    out += [(M, {0: 3, M // 2: 1, M - 1: 2}, (), None, 12) for M in ss.LMK_WINDOWS]
    out += [(192, {191: c, 0: 1}, (), None, 8) for c in ss.LMK_PER_CLONE]
    out.append((192, dict(ss.LMK_FULL), (), None, 96))
    for counts in ss.LMK_GATE:
        clones = sorted(counts)
        mid = clones[len(clones) // 2]
        rows = ss.lmk_rows({k: a for k, a in counts.items() if k != mid})
        out.append((192, counts, (mid,), {clones[0]: 2, clones[-1]: 1}, rows))  # behind: the planned rows stay
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_landmarks_at_every_row_count_and_cap(dtype):
    rng = np.random.default_rng(66)
    name = np.dtype(dtype).name
    worst = {}
    for M, counts, push, behind, rows in lmk_cases(ss.LMK_WINDOW):
        mem = fresh(dtype, M)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        chi2 = CHI2 if push else 0.0
        clone, z, p_L = lmk_obs(rng, poses, counts, push, behind)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, chi2_obs=chi2)
        ref, gam, flag = lmk_reference(P, imu, poses, clone, z, p_L, chi2)
        if push:
            assert np.all(flag[np.isin(clone, push)] != 0) and np.any(flag == 2)
            assert ss.chunks(ss.lmk_rows({k: int(np.sum(clone == k)) for k in counts})) > ss.chunks(rows)
        settle(worst, lmk_checked(res, mem.e, ref, gam, flag, imu, rows), name, (M, len(clone), rows))
    assert_measured("lmk", name, worst)


def iter_steps(P, imu, poses, clone, z, p_L):
    """the iteration's step after linearisations 1, 2 and 3 (tol = 0)"""
    return [iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=j, tol=0.0)["step"] for j in (2, 3, 4)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_iterated_landmarks_at_180_and_1152_rows(dtype):
    rng = np.random.default_rng(67)
    name = np.dtype(dtype).name
    worst = {}
    for rows in ss.LMK_ITER_ROWS:
        mem = fresh(dtype, ss.LMK_WINDOW)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        clone, z, p_L = drifted_obs(rng, poses, ss.spread(ss.LMK_WINDOW, rows // 6), 3, 0.3)
        # tol between the two consecutive steps that differ most: converged at a known iteration, far from the threshold
        s = iter_steps(P, imu, poses, clone, z, p_L)
        j = int(np.argmax([s[i] / s[i + 1] for i in range(2)]))
        assert s[j] / s[j + 1] >= 4, s  # (tol a factor >= 2 from either step; the steps agree far closer than that)
        tol = float(np.sqrt(s[j] * s[j + 1]))
        want = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=4, tol=tol)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, max_iter=4, tol=tol)
        assert want["converged"] == 1 and want["iterations"] == j + 2
        assert res["status"] == 0
        for key in ("iterations", "converged", "used", "dof", "applied"):
            assert res[key] == want[key], (rows, key, res[key], want[key])
        ref = (want["P"], want["imu"], want["poses"], want["nis"], float(np.linalg.norm(want["dx"])))
        settle(worst, lmk_checked(res, mem.e, ref, want["gamma"], want["flag"], imu, rows), name, rows)
    assert_measured("lmk_iter", name, worst)


# ---- mapped landmarks, map uncertainty ---------------------------------------------------------------------------------
def map_checked(res, e, P, imu, poses, clone, z, p_L, lm, Sig, rows):
    H, r, Rb, F, lmu, gam, flag = mref.dense(P, poses, clone, z, p_L, lm, Sig, R_PIX)
    assert mref.rows(clone, lm, flag) == rows
    return lmk_checked(res, e, numpy_update(P, imu, poses, H, r, Rb), gam, flag, imu, rows)


@pytest.mark.parametrize("dtype", DTYPES)
def test_map_landmarks_at_every_group_cap(dtype):
    rng = np.random.default_rng(68)
    name = np.dtype(dtype).name
    worst = {}
    M = ss.LMK_WINDOW
    for sets in (ss.MAP_END, ss.MAP_FULL_SET, ss.MAP_SETS, ss.MAP_ROWS):
        mem = fresh(dtype, M)
        imu, poses = state_of(mem.e)
        P = mem.e.covariance().astype(np.float64)
        clone, z, p_L, lm, Sig = scene(rng, poses, sets)
        res = mem.e.landmark_update(clone, z, p_L, R=R_PIX, landmark=lm, Sigma_L=Sig)
        settle(worst, map_checked(res, mem.e, P, imu, poses, clone, z, p_L, lm, Sig, ss.map_rows(sets)), name, len(sets))
    # two rows past the cap (the next count the planned rows can take): refused, nothing written
    mem = fresh(dtype, M)
    _, poses = state_of(mem.e)
    clone, z, p_L, lm, Sig = scene(rng, poses, ss.MAP_PAST)
    before = snapshot(mem.e)
    with pytest.raises(RuntimeError, match="rc=-3"):
        mem.e.landmark_update(clone, z, p_L, R=R_PIX, landmark=lm, Sigma_L=Sig)
    assert b"rows" in capi.lib().msckf_b200_last_error()
    assert_unchanged(snapshot(mem.e), before)
    assert_measured("map", name, worst)


# ---- one landmark batch of large and small members ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_landmark_batch_of_large_and_small_members(dtype):
    rng = np.random.default_rng(69)
    name = np.dtype(dtype).name
    worst = {"lmk": {}, "map": {}}
    large = [("exact", ss.sweep_counts(192, 1152), 1152), ("exact", dict(ss.LMK_FULL), 96), ("exact", {191: 256}, 6),
             ("map", ss.MAP_ROWS, 1152), ("map", ss.MAP_SETS, 1024)]
    plan = []
    for i in range(33):
        if i % 7 == 0 and i // 7 < len(large):
            plan.append((192,) + large[i // 7])
        else:
            M = (3, 12, 40, 91)[i % 4]
            counts = {int(k): int(rng.integers(1, 5)) for k in rng.choice(M, size=min(M, 1 + i % 9), replace=False)}
            plan.append((M, "map" if i % 5 == 1 else "exact", counts if i % 5 != 1 else [[k] for k in counts] + [[0, M - 1]] * 2, None))
    mem = [fresh(dtype, p[0]) for p in plan]
    twins = [fresh(dtype, p[0]) for p in plan]
    specs, inputs = [], []
    for (M, kind, what, rows), m in zip(plan, mem):
        imu, poses = state_of(m.e)
        P = m.e.covariance().astype(np.float64)
        if kind == "exact":
            clone, z, p_L = make_obs(rng, poses, what)
            specs.append({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX})
        else:
            clone, z, p_L, lm, Sig = scene(rng, poses, what)
            specs.append({"clone": clone, "z": z, "p_L": p_L, "R": R_PIX, "landmark": lm, "Sigma_L": Sig})
        inputs.append((P, imu, poses, rows if rows is not None else (ss.lmk_rows(what) if kind == "exact" else ss.map_rows(what))))
    single = [t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], landmark=s.get("landmark"), Sigma_L=s.get("Sigma_L"))
              for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t, s, (P, imu, poses, rows)) in enumerate(zip(mem, twins, specs, inputs)):
        for key in ("nis", "dx_norm", "dof", "rows", "used", "applied", "status"):
            assert got[i][key] == single[i][key], (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"]) and np.array_equal(got[i]["flag"], single[i]["flag"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i
        if "Sigma_L" in s:
            rel = map_checked(got[i], m.e, P, imu, poses, s["clone"], s["z"], s["p_L"], s["landmark"], s["Sigma_L"], rows)
            settle(worst["map"], rel, name, i)
        else:
            ref, gam, flag = lmk_reference(P, imu, poses, s["clone"], s["z"], s["p_L"], 0.0)
            settle(worst["lmk"], lmk_checked(got[i], m.e, ref, gam, flag, imu, rows), name, i)
    for group, w in worst.items():
        assert_measured(group, name, w)
