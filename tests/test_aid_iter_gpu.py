"""The iterated stacked aided update on the device (msckf_b200_aid_stack_update_iter / _fde_iter and their batch forms) in fp32
and fp64 against the dense numpy IEKF of tests/aid_iter_reference.py:
  * windows of 0, 1, 20 and 40 clones, stacks of ranges, a plane range, a GNSS antenna with a 0.5 m lever, a heading, a body
    velocity, a relative pose and a clone range measured at truths drifted by 0.05, 0.3 and 1 m from the estimate, plain and
    with fault detection and exclusion (FDE); iterations and converged equal, P, the state, the NIS and the step within 10 x
    the measurements below;
  * max_iter 0 and 1 bit for bit the calls without _iter; VELOCITY / POSITION stacks keep one linearisation's P bit for bit;
    a 33-member batch over two launch chunks with mixed max_iter bit for bit single calls;
  * a plane that an iterate puts behind the sensor (the previous linearisation is applied), gated-out, rejected and not
    positive definite stacks (nothing written), refusals (nothing written, no launch) and ERR_NUMERIC;
  * every shape the iterated form dispatches on: each row count at its last shared and first global window, windows 0, 1, 191
    and 192 (tests/side_shapes.py), and every shape whose FDE launch passes the default 48 KB of shared memory."""
import ctypes as C
import gc

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from tests import aid_iter_reference as ref, side_shapes as ss
from tests.aid_fde_reference import fde as fde_rounds, recipe_items
from tests.test_aid_gpu import assert_unchanged, snapshot, state_of
from tests.test_batch_stream_gpu import Member
from tests.test_range_gpu import plane_item, range_item

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
WINDOWS = [0, 1, 20, 40]
DRIFTS = [0.05, 0.3, 1.0]
CHI2 = capi.fde_thresholds(0.01)
PASS = {"chi2": [1e12] * 32, "max_exclude": 2}  # FDE whose gate every stack passes: the iteration over all items
MAX_ITER, TOL = 8, 1e-9
CONTRACT = {"float32": 1e-5, "float64": 1e-9}
# worst relative differences to the reference, measured on an H100 80GB HBM3 (700 W power limit) by this file; asserted at 10 x
# (P: of max |P|; state: of max |x|; nis: relative; step: relative to max |delta|; dx: |dx| relative)
MEASURED = {"float32": {"P": 1.26e-7, "state": 5.70e-8, "nis": 2.19e-7, "step": 1.49e-8, "dx": 3.43e-8},
            "float64": {"P": 7.09e-15, "state": 6.79e-16, "nis": 3.85e-14, "step": 2.19e-14, "dx": 1.59e-14}}
# k_aid's static shared memory under IT (-Xptxas -v, sm_90a, both dtypes, NM = 1 and 32): a launch past 48 KB needs the raised limit
IT_STATIC_SMEM = {"plain": 15136, "fde": 18064}
IT_OPT_IN = [(M, m) for M in range(ss.K["kMaxKeep"] + 1) for m in range(1, ss.K["kAidMaxRows"] + 1)
             if not ss.aid_global(M, m) and IT_STATIC_SMEM["fde"] + ss.aid_dynamic_smem(M, m) > ss.AID_DEFAULT_SMEM]
_BASE = {}
WORST = {}


@pytest.fixture(autouse=True, scope="module")
def _free_engines():
    yield
    _BASE.clear()
    gc.collect()
    for k, v in sorted(WORST.items()):
        print(f"aid iter worst {k}: " + ", ".join(f"{a} {b:.2e}" for a, b in v.items()))


def base(dtype, M, drift):
    """one engine per (dtype, window, drift) with a prior of that drift (ref.drift_prior), built once; tests take twins"""
    key = (np.dtype(dtype).name, M, drift)
    if key not in _BASE:
        b = Member(dtype, M, seed=900 + M, max_clones=min(M + 2, ss.K["kMaxKeep"]))
        b.e.set_covariance(ref.drift_prior(np.random.default_rng(M), M, drift))
        _BASE[key] = b
    return _BASE[key]


def fresh(dtype, M, drift):
    b = base(dtype, M, drift)
    return b.twin(dtype, max_clones=min(M + 2, ss.K["kMaxKeep"]))


def prior_of(e):
    imu, poses = state_of(e)
    return imu, poses, e.covariance().astype(np.float64)


def truth_of(rng, imu, poses, P):
    """a truth the estimate has drifted from: the estimate moved by a draw from P"""
    return ref.boxplus(imu, poses, np.linalg.cholesky(P) @ rng.normal(size=len(P)))


def clear(want, tol=TOL):
    """no step of the reference within a factor 2 of tol (iterations and converged are decisions the device must share)"""
    return all(not (tol / 2 <= s <= tol * 2) for s in want["steps"])


def errors(e, got, want, imu0):
    Pd, (imud, posesd) = e.covariance().astype(np.float64), state_of(e)
    assert np.array_equal(imud[19:29], imu0[19:29])  # the observability copies are not touched
    sd, sr = np.concatenate([imud[0:19], posesd.ravel()]), np.concatenate([want["imu"][0:19], want["poses"].ravel()])
    return {"P": np.abs(Pd - want["P"]).max() / np.abs(want["P"]).max(), "state": np.abs(sd - sr).max() / np.abs(sr).max(),
            "nis": abs(got["nis"] - want["nis"]) / want["nis"], "step": abs(got["step"] - want["step"]) / np.abs(want["dx"]).max(),
            "dx": abs(got["dx_norm"] - want["dx_norm"]) / want["dx_norm"]}


def check(dtype, err, what):
    name = np.dtype(dtype).name
    w = WORST.setdefault(f"{name} {what}", {})
    for k, v in err.items():
        w[k] = max(w.get(k, 0.0), v)
        bound = min(CONTRACT[name], 10 * MEASURED[name][k])
        assert v <= bound, (what, k, v, bound)


def compare(dtype, e, got, want, imu0, what):
    assert got["applied"] == 1 and got["status"] == 0
    assert (got["iterations"], got["converged"], got["dof"]) == (want["iterations"], want["converged"], want["dof"]), (what, got, {
        k: want[k] for k in ("iterations", "converged", "dof", "steps")})
    check(dtype, errors(e, got, want, imu0), what)


def drawn(rng, e, M, draw_items, kept=None, max_iter=MAX_ITER, tol=TOL, tries=20):
    """(items, kept indices, the reference) at engine e's prior, items measured at a drifted truth; drawn again until no step
    of the reference is near tol and (FDE) every decision is 5 % from its threshold"""
    imu, poses, P = prior_of(e)
    for _ in range(tries):
        items = draw_items(rng, *truth_of(rng, imu, poses, P))
        if any(ref.degenerate(it, imu, poses) for it in items):  # (a plane the drift put behind the sensor)
            continue
        keep = list(range(len(items)))
        if kept is not None:
            rounds = fde_rounds(items, imu, poses, P, kept["chi2"], kept["max_exclude"])
            if rounds["margin"] < 0.05 or rounds["outcome"] > 1:
                continue
            keep = rounds["kept"]
        want = ref.iekf([items[k] for k in keep], imu, poses, P, max_iter=max_iter, tol=tol)
        if clear(want, tol):
            return items, keep, want
    pytest.fail("no case away from the decisions")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("form", ["plain", "fde", "fde_fault"])
@pytest.mark.parametrize("M", WINDOWS)
def test_matches_the_dense_reference(dtype, form, M):
    rng = np.random.default_rng(10 * M + len(form))
    most = 0
    for drift in DRIFTS:
        b = base(dtype, M, drift)

        def items_at(rng, t_imu, t_poses):
            items = ref.scene(rng, t_imu, t_poses, M)
            if form == "fde_fault":  # the first range 10 m long: excluded at linearisation 0, the rest iterated
                items[0]["z"] = np.r_[items[0]["z"][0] + 10.0, items[0]["z"][1:]]
            return items

        fde = {"plain": None, "fde": PASS, "fde_fault": {"chi2": CHI2, "max_exclude": 2}}[form]
        items, keep, want = drawn(rng, b.e, M, items_at, kept=fde)
        a = b.twin(dtype, max_clones=min(M + 2, ss.K["kMaxKeep"]))
        imu0, _ = state_of(a.e)
        got = a.e.aid_stack_update(items, fde=fde, max_iter=MAX_ITER, tol=TOL)
        if fde is not None:
            assert got["outcome"] == (1 if form == "fde_fault" else 0), got["outcome"]
            assert [k for k, it in enumerate(got["items"]) if it["state"] == 0] == keep
        compare(dtype, a.e, got, want, imu0, f"{form} M={M} drift={drift}")
        most = max(most, got["iterations"])
    assert most >= 3  # the drifted stacks do relinearise


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_linearisation_is_the_existing_call_bit_for_bit(dtype):
    rng = np.random.default_rng(21)
    for M in (0, 20):
        b = base(dtype, M, 0.3)
        imu, poses, P = prior_of(b.e)
        items = ref.scene(rng, *truth_of(rng, imu, poses, P), M)
        for fde in (None, PASS, {"chi2": CHI2, "max_exclude": 1}):
            for max_iter in (0, 1):
                x, y = b.twin(dtype, max_clones=M + 2), b.twin(dtype, max_clones=M + 2)
                got = x.e.aid_stack_update(items, fde=fde, max_iter=max_iter, tol=TOL)
                want = y.e.aid_stack_update(items, fde=fde)
                assert (got.pop("iterations"), got.pop("converged"), got.pop("step")) == (want["applied"], 0, 0.0)
                assert got == want or _same(got, want)
                assert_unchanged(snapshot(x.e)[:3], snapshot(y.e)[:3])
        x, y = b.twin(dtype, max_clones=M + 2), b.twin(dtype, max_clones=M + 2)  # the plain gate passes through
        g = y.e.aid_stack_update(items, chi2_max=1e-3)
        got = x.e.aid_stack_update(items, chi2_max=1e-3, max_iter=1)
        assert got["applied"] == g["applied"] == 0 and got["iterations"] == 0
        assert_unchanged(snapshot(x.e)[:3], snapshot(y.e)[:3])


def _same(a, b):
    for k in b:
        if k == "items":
            for x, y in zip(a[k], b[k]):
                assert all(x[j] == y[j] or (np.isnan(x[j]) and np.isnan(y[j])) for j in y), (x, y)
        else:
            assert a[k] == b[k] or (np.isnan(a[k]) and np.isnan(b[k])), (k, a[k], b[k])
    return True


@pytest.mark.parametrize("dtype", DTYPES)
def test_linear_models_keep_one_linearisations_covariance(dtype):
    rng = np.random.default_rng(31)
    b = base(dtype, 20, 1.0)
    imu, poses, P = prior_of(b.e)
    t_imu, _ = truth_of(rng, imu, poses, P)
    items = [{"model": capi.AID_POSITION, "z": t_imu[0:3] + 0.1 * rng.normal(size=3), "R": 0.01 * np.eye(3)},
             {"model": capi.AID_VELOCITY, "z": t_imu[3:6] + 0.1 * rng.normal(size=3), "R": 0.04 * np.eye(3)}]
    for fde in (None, PASS):
        x, y = b.twin(dtype, max_clones=22), b.twin(dtype, max_clones=22)
        got = x.e.aid_stack_update(items, fde=fde, max_iter=MAX_ITER, tol=TOL)
        one = y.e.aid_stack_update(items, fde=fde)
        assert got["iterations"] == 2 and got["converged"] == 1 and got["step"] <= 1e-12
        assert np.array_equal(x.e.covariance(), y.e.covariance())
        assert got["nis"] == one["nis"] and got["dof"] == one["dof"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fde", [None, PASS])
def test_batch_equals_single_calls_bit_for_bit(dtype, fde):
    """33 members (two launch chunks) at windows 0, 1, 20 and 40, max_iter 0 .. 16 mixed, converging at different iterations,
    every fifth member left alone"""
    rng = np.random.default_rng(41)
    Ms, iters = [0, 1, 20, 40], [0, 1, 2, 3, 8, 16, 5]
    mem, stacks, mi = [], [], []
    for i in range(33):
        M, drift = Ms[i % 4], DRIFTS[i % 3]
        m = base(dtype, M, drift).twin(dtype, max_clones=M + 2)
        mem.append(m)
        imu, poses, P = prior_of(m.e)
        stacks.append(None if i % 5 == 4 else ref.scene(rng, *truth_of(rng, imu, poses, P), M))
        mi.append(iters[i % 7])
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    tol = [TOL if i % 2 else 1e-6 for i in range(33)]
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.aid_stack_update(s, fde=fde, max_iter=k, tol=tl) for t, s, k, tl in zip(twins, stacks, mi, tol)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.aid_stack_update(stacks, fde=fde, max_iter=mi, tol=tol)
    batch.close()
    assert len({g["iterations"] for g in got if g}) >= 4
    for i, (m, t, s) in enumerate(zip(mem, twins, stacks)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        assert got[i].keys() == single[i].keys() and _same(got[i], single[i]), i
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fde", [None, PASS])
def test_a_degenerate_iterate_applies_the_previous_linearisation(dtype, fde):
    """a rangefinder 0.05 m above a floor that reads -0.4 m: the first step puts the floor behind the sensor, so linearisation
    1 is applied; numpy stops at the same iterate"""
    rng = np.random.default_rng(51)
    b = base(dtype, 3, 1.0)
    imu, poses, P = prior_of(b.e)
    plane = plane_item(rng, imu, poses, dist=0.05, beam=np.array([0.0, 0.0, -1.0]))
    plane["z"] = np.r_[-0.4, plane["z"][1:]]
    items = [range_item(rng, imu, poses), plane, range_item(rng, imu, poses)]
    assert not ref.degenerate(plane, imu, poses)
    want = ref.iekf(items, imu, poses, P, max_iter=MAX_ITER, tol=TOL)
    assert want["iterations"] == 1 and ref.degenerate(plane, *ref.boxplus(imu, poses, want["dx"]))
    a = b.twin(dtype, max_clones=5)
    imu0, _ = state_of(a.e)
    got = a.e.aid_stack_update(items, fde=fde, max_iter=MAX_ITER, tol=TOL)
    assert got["iterations"] == 1 and got["converged"] == 0
    compare(dtype, a.e, got, want, imu0, "degenerate iterate")


@pytest.mark.parametrize("dtype", DTYPES)
def test_stacks_that_write_nothing_make_no_iterations(dtype):
    rng = np.random.default_rng(61)
    b = base(dtype, 4, 0.3)
    imu, poses, P = prior_of(b.e)
    items = ref.scene(rng, *truth_of(rng, imu, poses, P), 4)
    neg = items[:-1] + [dict(items[-1], R=np.array([[-1e6]]))]
    lever = np.array([0.2, -0.1, 0.3])
    on_anchor = {"model": capi.AID_RANGE, "a": 0, "b": 0, "R": np.array([[0.01]]),
                 "z": np.r_[1.0, mc.antenna_position(imu[0:3], imu[15:19], lever), lever]}
    cases = [(items, {"chi2_max": 1e-6}, 0), (items, {"fde": {"chi2": [1e-6] * 32, "max_exclude": 0}}, 0),
             (items, {"fde": {"chi2": [1e-6] * 32, "max_exclude": 2}}, 0), (neg, {}, 1), (neg, {"fde": PASS}, 1),
             (items[:2] + [on_anchor], {}, 2), ([on_anchor], {"fde": PASS}, 2)]
    for its, kw, status in cases:
        a = b.twin(dtype, max_clones=6)
        before = snapshot(a.e)
        got = a.e.aid_stack_update(its, max_iter=MAX_ITER, tol=TOL, **kw)
        assert got["applied"] == 0 and got["status"] == status and got["dx_norm"] == 0.0, (kw, got)
        assert (got["iterations"], got["converged"], got["step"]) == (0, 0, 0.0)
        if "fde" in kw and status == 0:
            assert got["outcome"] in (2, 3)
        assert_unchanged(snapshot(a.e), before)


def test_refusals_write_nothing():
    rng = np.random.default_rng(71)
    M = 3
    mem = [fresh(np.float64, M, 0.3) for _ in range(2)]
    lib = capi.lib()
    imu, poses, P = prior_of(mem[0].e)
    good = ref.scene(rng, *truth_of(rng, imu, poses, P), M)
    before = [snapshot(m.e) for m in mem]
    sent, isent = capi.AidFdeResult(), capi.AidIterResult()
    C.memset(C.addressof(sent), 0x5a, C.sizeof(sent))
    C.memset(C.addressof(isent), 0x5a, C.sizeof(isent))

    def raw(e, items, it, fde, null_out=False):
        arr, keep = capi.aid_items(items)
        out, iout = capi.AidFdeResult.from_buffer_copy(sent), capi.AidIterResult.from_buffer_copy(isent)
        ip = None if it is None else C.byref(capi.AidIter(*it))
        io = None if null_out else C.byref(iout)
        if fde:
            rc = lib.msckf_b200_aid_stack_update_fde_iter(e.h, arr, C.c_int(len(items)), C.byref(capi.fde_struct(PASS)), ip,
                                                           C.byref(out), io)
        else:
            rc = lib.msckf_b200_aid_stack_update_iter(e.h, arr, C.c_int(len(items)), C.c_double(0.0), ip, C.byref(out.stack), io)
        return rc, bytes(out), bytes(iout)

    refused = (-3, bytes(sent), bytes(isent))
    for fde in (False, True):
        for it in (None, (-1, 0.0), (17, 0.0), (4, np.nan), (4, np.inf), (4, -1e-3), (4, -np.inf)):
            assert raw(mem[0].e, good, it, fde) == refused, (fde, it)
        assert raw(mem[0].e, good, (4, 0.0), fde, null_out=True) == refused
        assert raw(mem[0].e, [], (4, 0.0), fde) == refused
        assert raw(mem[0].e, [dict(good[0], a=1)], (4, 0.0), fde) == refused  # (a range at the IMU takes a = 0)
        assert raw(mem[0].e, good + good, (4, 0.0), fde) == refused  # more than 8 items
    assert_unchanged(snapshot(mem[0].e), before[0])
    batch = capi.Batch([m.e for m in mem])
    for fde in (None, PASS):
        with pytest.raises(RuntimeError, match="rc=-3"):
            batch.aid_stack_update([good, good], fde=fde, max_iter=[4, 17], tol=0.0)
        with pytest.raises(RuntimeError, match="rc=-3"):
            batch.aid_stack_update([good, good], fde=fde, max_iter=4, tol=[0.0, np.nan])
    # an un-fetched update: ERR_STATE, no launch
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    launched = mem[1].e.launch_count()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.aid_stack_update([good, None], max_iter=4, tol=0.0)
    assert raw(mem[1].e, good, (4, 0.0), False) == (-5, bytes(sent), bytes(isent))
    assert mem[1].e.launch_count() == launched
    mem[1].e.fetch(1)
    batch.close()
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)


def test_non_finite_covariance_is_reported_and_applied():
    rng = np.random.default_rng(81)
    m = fresh(np.float64, 4, 0.3)
    imu, poses, P = prior_of(m.e)
    items = ref.scene(rng, *truth_of(rng, imu, poses, P), 4, kinds=("range",))
    P[30, 30] = np.inf  # outside the rows a range at the IMU reads: only the downdate meets it
    m.e.set_covariance(P)
    with pytest.raises(RuntimeError, match="rc=-6"):
        m.e.aid_stack_update(items, max_iter=4, tol=TOL)
    assert not np.array_equal(state_of(m.e)[0], imu)  # applied, like the vision update's ERR_NUMERIC


def _shape_case(dtype, M, m, fde, seed):
    rng = np.random.default_rng(seed)
    recipe = ss.fde_stack(M, m)
    b = base(dtype, M, 0.3)
    items, keep, want = drawn(rng, b.e, M, lambda r, ti, tp: recipe_items(r, recipe, ti, tp, M), max_iter=4)
    a = b.twin(dtype, max_clones=min(M + 2, ss.K["kMaxKeep"]))
    imu0, _ = state_of(a.e)
    got = a.e.aid_stack_update(items, fde=PASS if fde else None, max_iter=4, tol=TOL)
    compare(dtype, a.e, got, want, imu0, f"shape M={M} m={m} fde={fde}")
    return got


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ss.aid_cases(), ids=str)
def test_every_window_and_row_count(dtype, case):
    """each row count at its last window with W^T, dx in shared memory and its first in the global workspace (the iterated
    form keeps delta_i in dx, so it has the plain form's byte count and boundary), and windows 0, 1, 191 and 192"""
    M, m = case
    for fde in (False, True):
        _shape_case(dtype, M, m, fde, seed=M * 100 + m)
    if M in (191, 192):
        _BASE.pop((np.dtype(dtype).name, M, 0.3), None)


@pytest.mark.parametrize("case", IT_OPT_IN, ids=str)
def test_shapes_past_the_default_shared_memory(case):
    """every shape whose iterated FDE launch takes more than 48 KB (18 064 B static): the raised limit; fp32 and fp64 in turn"""
    M, m = case
    dtype = DTYPES[IT_OPT_IN.index(case) % 2]
    _shape_case(dtype, M, m, True, seed=M * 100 + m + 7)
    _BASE.pop((np.dtype(dtype).name, M, 0.3), None)


def test_runner_first_ranging_after_an_outage():
    """8 trials x 60 frames, four ranges every frame from frame 30 on, iterated up to 8 linearisations: the first stack after
    the outage relinearises, and the ANIS of the run's stacks lies inside its bounds widened by 3 % (as DESIGN 4.15 widens them)"""
    truth = mc.make_truth(n_frames=60, seq=8)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, range_every=1, range_start=30, aid_iterations=8)
    s = mc.summarize(rec)
    g, first = s["range"], s["range_first"]
    one, _ = mc.run(range(8), truth, dtype=np.float64, range_every=1, range_start=30)
    s1 = mc.summarize(one)
    print(f"first ranging stack after frame 30: linearisations {first['iterations']:.2f}, converged {first['converged']:.2f}, "
          f"position RMSE {first['pos_rmse_before']:.3f} -> {first['pos_rmse_after']:.3f} m (one linearisation "
          f"{s1['range_first']['pos_rmse_after']:.3f} m), IMU NEES after {first['imu_anees']:.2f} (one linearisation "
          f"{s1['range_first']['imu_anees']:.2f}, bounds {first['imu_bounds']}); run ANIS {g['mean_anis']:.3f} for "
          f"{g['mean_dof']:.2f} dof, bounds {g['run_bounds']}")
    assert first["frame"] == 30 and first["iterations"] > 1 and first["converged"] > 0
    assert g["run_bounds"][0] * 0.97 <= g["mean_anis"] <= g["run_bounds"][1] * 1.03
