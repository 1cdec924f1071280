"""Fault detection and exclusion (k_aid<S, NM, true>) and the range models at every window, row count, item count and exclusion
depth k_aid dispatches on (tests/side_shapes.py), in fp32 and fp64, against the dense numpy rounds of tests/aid_fde_reference.py
and the Joseph-form update of the kept items:
  * every grid case (each row count at its last shared and first global window, windows 0, 1, 191 and 192), with no fault, a
    fault on the last item, on a 6-row item, and two faults apart (the kept rows gathered around a hole) at max_exclude 2 and 1;
    the applied update also bit for bit against the plain stack of the kept items;
  * 1 to 7 exclusion rounds at m = 32 on both storage sides, one round short (rejected), every item faulty, and a stack no
    single item explains;
  * degenerate items (an antenna on its anchor, a level beam, a plane behind the sensor) first, in the middle and last, with a
    real fault elsewhere;
  * every shape whose launch takes more than the default 48 KB of shared memory, and a 33-member batch mixing them with both
    storage paths (the shared memory of such a launch in a profiler trace: tests/test_side_shapes_gpu.py).
Decisions (outcome, excluded items and rounds, item states) are compared exactly; every drawn case has each decision at least
5 % from its threshold or a tie (drawn again otherwise)."""
import gc
import json

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from oracle.msckf_numpy import quat_to_rot
from tests import aid_fde_reference as ref, side_shapes as ss
from tests.test_aid_gpu import assert_unchanged, snapshot, state_of
from tests.test_gnss_gpu import rel_errors
from tests.test_range_gpu import plane_item, range_item, stack_reference
from tests.test_batch_stream_gpu import Member
from tests.test_side_shapes_gpu import cap, settle

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
CHI2 = capi.fde_thresholds(0.01)
# t_j and the item NIS: relative in fp64; in fp32 relative to max(|w|, 1), the scale of the thresholds they meet
STAT_TOL = {"float32": (1e-4, 1.0), "float64": (1e-9, 1e-12)}
RATIOS = {"none": (), "last": (40.0,), "six": (40.0,), "pair": (60.0, 20.0)}  # each fault alone, in thresholds of its item
# worst relative differences to the references, measured on an H100 80GB HBM3 (700 W power limit) by this file; asserted at 10 x
# (the worst over the file's tests; stat: t_j and the item NIS, as STAT_TOL measures them)
MEASURED = {"float32": {"stat": 7.86e-6, "P": 3.03e-7, "state": 5.63e-8, "nis": 5.45e-7, "dx": 1.52e-7},
            "float64": {"stat": 4.10e-11, "P": 5.94e-14, "state": 6.78e-15, "nis": 5.53e-12, "dx": 2.77e-12}}
NAN_OUT = {"nis", "test"}
_BASE = {}


@pytest.fixture(autouse=True, scope="module")
def _free_engines():
    """the file's engines go with it: the files after it start from the device state they would have without it"""
    yield
    _BASE.clear()
    gc.collect()


def base(dtype, M):
    """one engine per (dtype, window), built once (as test_side_shapes_gpu.base); tests that write take a twin"""
    key = (np.dtype(dtype).name, M)
    if key not in _BASE:
        _BASE[key] = Member(dtype, M, seed=500 + M, max_clones=cap(M))
    return _BASE[key]


def fresh(dtype, M):
    return base(dtype, M).twin(dtype, max_clones=cap(M))


def draw(rng, recipe, faults, ratios, M, e, K, degenerate=None):
    """(items, the reference's rounds) of a recipe at engine e's state with the faults; degenerate = (item, kind) puts a
    degenerate item there.  Drawn again until every decision is 5 % from its threshold or a tie."""
    imu, poses = state_of(e)
    P = e.covariance().astype(np.float64)
    dropped = () if degenerate is None else (degenerate[0],)
    for _ in range(40):
        items = ref.with_faults(rng, ref.recipe_items(rng, recipe, imu, poses, M), faults, ratios, imu, poses, P, CHI2)
        if degenerate is not None:
            items[degenerate[0]] = degenerate_item(rng, degenerate[1], imu, poses, M)
        want = ref.fde(items, imu, poses, P, CHI2, K, dropped=dropped)
        if want["margin"] >= 0.05:
            return items, want
    pytest.fail(f"no case away from the thresholds: {recipe} {faults}")


def degenerate_item(rng, kind, imu, poses, M):
    """a range whose prediction is undefined: an antenna on its anchor, a beam parallel to the plane, the plane behind the sensor"""
    lever = np.array([0.2, -0.1, 0.3])
    if kind == "on_anchor":
        return range_item(rng, imu, poses, lever=lever, anchor=mc.antenna_position(imu[0:3], imu[15:19], lever))
    if kind == "level_beam":
        pl = plane_item(rng, imu, poses)
        return dict(pl, z=np.r_[1.0, pl["z"][1:5], quat_to_rot(imu[15:19]) @ np.array([0.6, 0.8, 0.0])])
    assert kind == "behind"
    return plane_item(rng, imu, poses, clone=M - 1, dist=-1.0)


def checked(got, want, items, e, before, name, worst, where, dropped=()):
    """one FDE result against the reference: the decisions exactly, t_j and the item NIS to STAT_TOL, an applied update against
    numpy within the side updates' ceilings, a rejected one writing nothing"""
    imu, poses, P = before[0].astype(np.float64), before[1].astype(np.float64), before[2].astype(np.float64)
    assert got["status"] == 0 and got["outcome"] == want["outcome"], (where, got["outcome"], want["outcome"], want["excluded"])
    assert got["n_excluded"] == len(want["excluded"]) and got["dof"] == want["dof"], (where, got, want)
    exc = dict(want["excluded"])
    assert len(got["items"]) == len(items)
    tol, floor = STAT_TOL[name]
    for j, it in enumerate(got["items"]):
        state = 2 if j in dropped else 1 if j in exc else (0 if want["outcome"] <= 1 else 3)
        assert it["state"] == state and it["round"] == exc.get(j, -1), (where, j, it, state)
        for k, w in (("nis", want["item_nis"][j]), ("test", want["tests"][j])):
            if np.isnan(w):
                assert np.isnan(it[k]), (where, j, k, it[k])
                continue
            rel = abs(it[k] - w) / max(abs(w), floor)
            worst["stat"] = max(worst.get("stat", 0.0), rel)
            assert rel <= tol, (where, j, k, it[k], w)
    assert abs(got["nis"] - want["nis"]) <= tol * max(abs(want["nis"]), floor), (where, got["nis"], want["nis"])
    if want["outcome"] <= 1:
        assert got["applied"] == 1
        kept = [items[j] for j in want["kept"]]
        settle(worst, rel_errors(e, got, stack_reference(kept, imu, poses, P), imu), name, where)
    else:
        assert got["applied"] == 0 and got["dx_norm"] == 0.0
        assert_unchanged(snapshot(e)[:3], before[:3])


def single(dtype, M, items, want, K, worst, where, dropped=()):
    """an FDE call on a fresh engine, checked; applied: bit for bit the plain stack of the kept items on another"""
    name = np.dtype(dtype).name
    a, b = fresh(dtype, M), fresh(dtype, M)
    before = snapshot(a.e)
    got = a.e.aid_stack_update(items, fde={"chi2": CHI2, "max_exclude": K})
    checked(got, want, items, a.e, before, name, worst, where, dropped)
    if got["applied"]:
        plain = b.e.aid_stack_update([items[j] for j in want["kept"]])
        for k in ("nis", "dx_norm", "dof", "applied", "status"):
            assert got[k] == plain[k], (where, k, got[k], plain[k])
        for x, y in zip(a.e.state() + (a.e.covariance(),), b.e.state() + (b.e.covariance(),)):
            assert np.array_equal(x, y), where
    return got


def assert_measured(name, worst):
    print(f"MEASURED fde {name} " + json.dumps({k: float(f"{v:.3g}") for k, v in worst.items()}))
    for k, v in worst.items():
        assert v <= 10 * MEASURED[name][k], (k, v, MEASURED[name][k])


@pytest.mark.parametrize("dtype", DTYPES)
def test_fde_at_every_grid_case(dtype):
    rng = np.random.default_rng(71)
    name = np.dtype(dtype).name
    worst = {}
    seen = set()
    for M, m in ss.aid_cases():
        recipe = ss.fde_stack(M, m)
        e = base(dtype, M).e
        side = "global" if ss.aid_global(M, m) else "shared"
        for pattern, faults, K in ss.fde_faults(recipe):
            where = (M, m, side, pattern, faults, K)
            items, want = draw(rng, recipe, faults, RATIOS[pattern], M, e, K)
            single(dtype, M, items, want, K, worst, where)
            seen.add(want["outcome"])
            if pattern == "none":  # the plain stack of the recipe (the range models at both paths and clone 191) against numpy
                st = fresh(dtype, M)
                imu, poses = state_of(st.e)
                P = st.e.covariance().astype(np.float64)
                res = st.e.aid_stack_update(items)
                assert res["applied"] == 1 and res["status"] == 0 and res["dof"] == m, (where, res)
                settle(worst, rel_errors(st.e, res, stack_reference(items, imu, poses, P), imu), name, where + ("plain",))
    assert seen == {0, 1, 2, 3}, seen
    assert_measured(name, worst)


@pytest.mark.parametrize("dtype", DTYPES)
def test_exclusion_depth(dtype):
    """k = 1..7 faults of decreasing size leave in that order (k = 7: one item left); max_exclude = k - 1 rejects; every item
    faulty rejects at max_exclude 7; 8 items each 0.75 thresholds off fail the stack with none explaining it (outcome 3)"""
    rng = np.random.default_rng(72)
    name = np.dtype(dtype).name
    worst = {}
    for M in ss.FDE_DEPTH_WINDOWS:
        e = base(dtype, M).e
        for k in range(1, 8):
            faults, ratios = list(range(k)), ss.FDE_DEPTH_RATIOS[:k]
            items, want = draw(rng, ss.FDE_DEPTH, faults, ratios, M, e, k)
            assert want["outcome"] == 1 and want["excluded"] == [(j, j) for j in range(k)] and len(want["kept"]) == 8 - k, want
            single(dtype, M, items, want, k, worst, (M, k, k))
            want = ref.fde(items, *state_of(e), e.covariance().astype(np.float64), CHI2, k - 1)
            assert want["outcome"] == 2 and len(want["excluded"]) == k - 1
            single(dtype, M, items, want, k - 1, worst, (M, k, k - 1))
        items, want = draw(rng, ss.FDE_DEPTH, list(range(8)), ss.FDE_DEPTH_RATIOS, M, e, 7)
        assert want["outcome"] == 2 and len(want["excluded"]) == 7, want
        single(dtype, M, items, want, 7, worst, (M, 8, 7))
        for _ in range(20):
            items, want = draw(rng, ss.FDE_DEPTH, list(range(8)), [ss.FDE_SPREAD_RATIO] * 8, M, e, 7)
            if want["outcome"] == 3 and len(want["kept"]) >= 2:
                break
        else:
            pytest.fail("no stack that no single item explains")
        got = single(dtype, M, items, want, 7, worst, (M, "spread"))
        assert got["outcome"] == 3 and [it["state"] for it in got["items"]].count(3) >= 2
    assert_measured(name, worst)


@pytest.mark.parametrize("dtype", DTYPES)
def test_degenerate_items_with_exclusions(dtype):
    """a degenerate item first, in the middle and last, a real fault elsewhere: state 2, NIS NaN, not counted toward max_exclude,
    the rounds of the reference with the item dropped"""
    rng = np.random.default_rng(73)
    name = np.dtype(dtype).name
    worst = {}
    for M in ss.FDE_DEPTH_WINDOWS:
        e = base(dtype, M).e
        for pos, kind, fault in ((0, "on_anchor", 3), (3, "level_beam", 5), (7, "behind", 1)):
            items, want = draw(rng, ss.FDE_DEPTH, [fault], [40.0], M, e, 1, degenerate=(pos, kind))
            assert want["outcome"] == 1 and want["excluded"] == [(fault, 0)], want
            got = single(dtype, M, items, want, 1, worst, (M, pos, kind), dropped=(pos,))
            assert got["items"][pos]["state"] == 2 and np.isnan(got["items"][pos]["nis"]) and got["n_excluded"] == 1
    assert_measured(name, worst)


def test_every_opt_in_shape():
    """each shape whose FDE launch takes more than the default 48 KB of shared memory: no fault (applied), one fault on the last
    item (excluded), each bit for bit the plain stack of the kept items"""
    rng = np.random.default_rng(74)
    worst = {}
    for M, m in ss.AID_OPT_IN:
        assert ss.aid_launch_smem(M, m, True) > ss.AID_DEFAULT_SMEM and not ss.aid_global(M, m)
        recipe = ss.fde_stack(M, m)
        e = base(np.float64, M).e
        for pattern, faults, K in (("none", (), 2), ("last", (len(recipe) - 1,), 1)):
            items, want = draw(rng, recipe, faults, RATIOS[pattern], M, e, K)
            assert want["outcome"] == (0 if pattern == "none" else 1) and [j for j, _ in want["excluded"]] == list(faults), want
            single(np.float64, M, items, want, K, worst, (M, m, pattern))
    assert_measured("float64", worst)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_equals_single_calls_and_the_reference(dtype):
    rng = np.random.default_rng(75)
    name = np.dtype(dtype).name
    worst = {}
    plan = [ss.FDE_BATCH[i % len(ss.FDE_BATCH)] for i in range(33)]
    mem = [fresh(dtype, M) for M, _ in plan]
    twins = [fresh(dtype, M) for M, _ in plan]
    K = 2
    stacks, wants = [], []
    for i, ((M, m), b) in enumerate(zip(plan, mem)):
        recipe = ss.fde_stack(M, m)
        pattern, faults, _ = ss.fde_faults(recipe)[(0, 1, -2)[i % 3]]
        items, want = draw(rng, recipe, faults, RATIOS[pattern], M, b.e, K)
        stacks.append(items)
        wants.append(want)
    before = [snapshot(b.e) for b in mem]
    fde = {"chi2": CHI2, "max_exclude": K}
    single_res = [t.e.aid_stack_update(s, fde=fde) for t, s in zip(twins, stacks)]
    batch = capi.Batch([b.e for b in mem])
    got = batch.aid_stack_update(stacks, fde=fde)
    batch.close()
    for i, (b, t) in enumerate(zip(mem, twins)):
        assert got[i].keys() == single_res[i].keys()
        for k in got[i]:
            if k != "items":
                assert got[i][k] == single_res[i][k] or (np.isnan(got[i][k]) and np.isnan(single_res[i][k])), (i, k)
        for x, y in zip(got[i]["items"], single_res[i]["items"]):
            assert all(x[k] == y[k] or (k in NAN_OUT and np.isnan(x[k]) and np.isnan(y[k])) for k in x), (i, x, y)
        for x, y in zip(b.e.state() + (b.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i
        checked(got[i], wants[i], stacks[i], b.e, before[i], name, worst, (i,) + plan[i])
    assert {w["outcome"] for w in wants} >= {0, 1}
    assert_measured(name, worst)

