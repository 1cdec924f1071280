"""Fault detection and exclusion over a stack's items on the device (msckf_b200_aid_stack_update_fde / _batch_..._fde) in
fp32 and fp64 at windows of 0, 1, 20 and 40 clones (W^T in shared memory and in the global workspace): max_exclude = 0 against
the plain stack's gate, injected range and GNSS faults against the numpy rounds of tests/aid_fde_reference.py and bit for bit
against the plain stack on the kept items, the rejections, the degenerate items, batches against single calls and refusals."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from tests import aid_fde_reference as ref
from tests.test_aid_gpu import assert_unchanged, snapshot, state_of
from tests.test_batch_stream_gpu import Member

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
WINDOWS = [0, 1, 20, 40]
CHI2 = capi.fde_thresholds(0.01)
NAN_OUT = {"nis", "test"}


def _stack(rng, imu, poses, M, faults=(), jump=0.0, wide=False):
    """four ranges, a GNSS antenna fix and a body velocity (and at M >= 1 a clone range); wide adds a relative pose so that
    m = 17 rows (W^T in the global workspace at 40 clones)"""
    items = ref.range_scene(rng, imu, poses, faults=faults, gnss=True, jump=jump, odometry=True, clone=M - 1 if M >= 1 else None)
    if wide and M >= 2:
        p, q = mc.relative_pose(poses[0], poses[M - 1])
        items.append({"model": capi.AID_RELATIVE_POSE, "a": 0, "b": M - 1, "z": np.r_[p + 0.01 * rng.normal(size=3), q],
                      "R": 1e-4 * np.eye(6)})
    return items


def _same_result(a, b):
    for k in ("nis", "dx_norm", "dof", "applied", "status"):
        assert a[k] == b[k] or (np.isnan(a[k]) and np.isnan(b[k])), (k, a[k], b[k])


def _assert_same_filter(e1, e2):
    for x, y in zip(e1.state() + (e1.covariance(),), e2.state() + (e2.covariance(),)):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", WINDOWS)
def test_max_exclude_zero_is_the_stack_gate(dtype, M):
    """both sides of chi2[m - 1]: bit-identical to msckf_b200_aid_stack_update with chi2_max = chi2[m - 1]"""
    rng = np.random.default_rng(100 + M)
    base = Member(dtype, M, seed=7 + M)
    imu, poses = state_of(base.e)
    for wide in (False, True):
        items = _stack(rng, imu, poses, M, faults=(1,), wide=wide)
        m = sum(len(it["R"]) for it in items)
        probe = base.twin(dtype)
        g = probe.e.aid_stack_update(items)["nis"]
        for side in (0.95, 1.05):
            chi2 = list(CHI2)
            chi2[m - 1] = g * side
            a, b = base.twin(dtype), base.twin(dtype)
            got = a.e.aid_stack_update(items, fde={"chi2": chi2, "max_exclude": 0})
            want = b.e.aid_stack_update(items, chi2_max=chi2[m - 1])
            _same_result(got, want)
            _assert_same_filter(a.e, b.e)
            assert got["applied"] == (side > 1.0) and got["outcome"] == (0 if side > 1.0 else 2) and got["n_excluded"] == 0
            assert all(np.isnan(it["test"]) and it["round"] == -1 for it in got["items"])
            assert [it["state"] for it in got["items"]] == [0 if side > 1.0 else 3] * len(items)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", WINDOWS)
def test_injected_faults_match_numpy(dtype, M):
    """the excluded set and outcome of numpy; P, state and NIS of the plain stack on the kept items bit for bit; t_j and the item
    NIS to 1e-9 relative in fp64.  Cases with a decision within 5 % of a threshold or a tie are skipped (drawn again)."""
    rng = np.random.default_rng(200 + M)
    base = Member(dtype, M, seed=11 + M)
    imu, poses = state_of(base.e)
    P = base.e.covariance().astype(np.float64)
    # fp64: relative; fp32: relative to max(|w|, 1), the scale of the thresholds the statistics meet (small t_j of the fp32
    # covariance were 3e-3 apart relative, 3e-8 absolute, on an H100)
    tol, floor = (1e-9, 1e-12) if dtype == np.float64 else (1e-4, 1.0)
    seen, worst = {0: 0, 1: 0, 2: 0, 3: 0}, 0.0
    cases = [((), 0.0), ((2,), 0.0), ((), 3.0), ((0,), 3.0), ((1, 3), 0.0), ((0, 2), 4.0)]
    for wide in (False, True):
        for faults, jump in cases:
            for K in (1, 2, 3):
                for _ in range(20):
                    items = _stack(rng, imu, poses, M, faults=faults, jump=jump, wide=wide)
                    want = ref.fde(items, imu, poses, P, CHI2, K)
                    if want["margin"] >= 0.05:
                        break
                else:
                    pytest.fail("no case away from the thresholds")
                a, b = base.twin(dtype), base.twin(dtype)
                got = a.e.aid_stack_update(items, fde={"chi2": CHI2, "max_exclude": K})
                assert got["outcome"] == want["outcome"], (faults, jump, K, got, want)
                assert got["n_excluded"] == len(want["excluded"])
                for j, rnd in want["excluded"]:
                    assert got["items"][j]["state"] == 1 and got["items"][j]["round"] == rnd
                seen[got["outcome"]] += 1
                for j, it in enumerate(got["items"]):
                    for k, w in (("nis", want["item_nis"][j]), ("test", want["tests"][j])):
                        if np.isnan(w):
                            assert np.isnan(it[k]), (j, k)
                        else:
                            worst = max(worst, abs(it[k] - w) / max(abs(w), floor))
                            assert abs(it[k] - w) <= tol * max(abs(w), floor), (j, k, it[k], w)
                if got["outcome"] <= 1:
                    assert [j for j, it in enumerate(got["items"]) if it["state"] == 0] == want["kept"]
                    plain = b.e.aid_stack_update([items[j] for j in want["kept"]])
                    _same_result(got, plain)
                    _assert_same_filter(a.e, b.e)
                    assert got["dof"] == want["dof"]
                else:
                    assert got["applied"] == 0 and [it["state"] for it in got["items"]].count(0) == 0
                    _assert_same_filter(a.e, b.e)
    assert seen[0] and seen[1] and seen[2], seen
    print(f"fde {np.dtype(dtype).name} M={M}: outcomes {seen}, worst t_j / item NIS rel to numpy {worst:.2e}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_rejections_and_degenerate_items(dtype):
    rng = np.random.default_rng(300)
    M = 4
    base = Member(dtype, M, seed=31)
    imu, poses = state_of(base.e)
    fde = {"chi2": CHI2, "max_exclude": 2}
    lever = np.array([0.2, -0.1, 0.3])
    on_anchor = {"model": capi.AID_RANGE, "a": 0, "b": 0, "R": np.array([[0.01]]),
                 "z": np.r_[1.0, mc.antenna_position(imu[0:3], imu[15:19], lever), lever]}
    # a one-item stack that fails: not identifiable (3); two faults with max_exclude 1: rejected at max_exclude (2)
    P = base.e.covariance().astype(np.float64)
    for items, K, outcome in ((ref.range_scene(rng, imu, poses, n_ranges=1, faults=(0,), bias=20.0), 2, 3),
                              (ref.range_scene(rng, imu, poses, n_ranges=6, faults=(1, 4), bias=5.0), 1, 2)):
        assert ref.fde(items, imu, poses, P, CHI2, K)["outcome"] == outcome
        a = base.twin(dtype)
        before = snapshot(a.e)
        got = a.e.aid_stack_update(items, fde={"chi2": CHI2, "max_exclude": K})
        assert got["outcome"] == outcome and got["applied"] == 0 and got["status"] == 0 and got["dx_norm"] == 0.0
        assert_unchanged(snapshot(a.e)[:3], before[:3])
    # a degenerate item among good ones: dropped (state 2, not counted), the rest applied as their plain stack
    good = _stack(rng, imu, poses, M)
    for pos in (0, 3, len(good)):
        items = good[:pos] + [on_anchor] + good[pos:]
        a, b = base.twin(dtype), base.twin(dtype)
        got = a.e.aid_stack_update(items, fde={"chi2": [1e6] * 32, "max_exclude": 0})
        assert got["outcome"] == 0 and got["n_excluded"] == 0 and got["status"] == 0
        assert got["items"][pos]["state"] == 2 and np.isnan(got["items"][pos]["nis"])
        _same_result(got, b.e.aid_stack_update(good))
        _assert_same_filter(a.e, b.e)
    # S_AA not positive definite (an item with a negative R): status 1, outcome -1, nothing written
    a = base.twin(dtype)
    before = snapshot(a.e)
    neg = dict(good[0], R=np.array([[-1e6]]))
    got = a.e.aid_stack_update(good[1:] + [neg], fde=fde)
    assert got["status"] == 1 and got["outcome"] == -1 and got["applied"] == 0 and np.isnan(got["nis"]) and got["dx_norm"] == 0.0
    assert got["dof"] == sum(len(it["R"]) for it in good)
    assert_unchanged(snapshot(a.e)[:3], before[:3])
    # every item degenerate: status 2, nothing written
    a = base.twin(dtype)
    before = snapshot(a.e)
    got = a.e.aid_stack_update([on_anchor, on_anchor], fde=fde)
    assert got["status"] == 2 and got["outcome"] == -1 and np.isnan(got["nis"]) and got["applied"] == 0
    assert [it["state"] for it in got["items"]] == [2, 2]
    assert_unchanged(snapshot(a.e)[:3], before[:3])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nf", [1, 8, 33])
def test_batch_equals_single_calls_bit_for_bit(dtype, nf):
    Ms = [0, 1, 20, 40]
    rng = np.random.default_rng(400 + nf)
    mem = [Member(dtype, Ms[i % 4], seed=500 + i, max_clones=Ms[i % 4] + 2) for i in range(nf)]
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    fde = {"chi2": CHI2, "max_exclude": 2}
    stacks = []
    for i, m in enumerate(mem):
        imu, poses = state_of(m.e)
        skip = nf > 1 and i % 5 == 4
        stacks.append(None if skip else _stack(rng, imu, poses, m.e.num_clones(), faults=((i % 4,) if i % 3 else ()),
                                                 jump=3.0 * (i % 2), wide=i % 2 == 0))
    before = [snapshot(m.e) for m in mem]
    single = [None if s is None else t.e.aid_stack_update(s, fde=fde) for t, s in zip(twins, stacks)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.aid_stack_update(stacks, fde=fde)
    batch.close()
    for i, (m, t, s) in enumerate(zip(mem, twins, stacks)):
        if s is None:
            assert got[i] is None
            assert_unchanged(snapshot(m.e), before[i])
            continue
        assert got[i].keys() == single[i].keys()
        for k in got[i]:
            if k != "items":
                assert got[i][k] == single[i][k] or (np.isnan(got[i][k]) and np.isnan(single[i][k])), (i, k)
        for x, y in zip(got[i]["items"], single[i]["items"]):
            assert all(x[k] == y[k] or (k in NAN_OUT and np.isnan(x[k]) and np.isnan(y[k])) for k in x), (i, x, y)
        _assert_same_filter(m.e, t.e)


def test_refusals_write_nothing():
    rng = np.random.default_rng(600)
    M = 3
    mem = [Member(np.float64, M, seed=70 + i) for i in range(2)]
    lib = capi.lib()
    imu, poses = state_of(mem[0].e)
    good = _stack(rng, imu, poses, M, faults=(1,))
    before = [snapshot(m.e) for m in mem]
    sentinel = capi.AidFdeResult()
    C.memset(C.addressof(sentinel), 0x5a, C.sizeof(sentinel))

    def raw(e, items, f):
        arr, keep = capi.aid_items(items)
        out = capi.AidFdeResult.from_buffer_copy(sentinel)
        fp = None if f is None else C.byref(capi.fde_struct(f))
        rc = lib.msckf_b200_aid_stack_update_fde(e.h, arr, C.c_int(len(items)), fp, C.byref(out))
        return rc, bytes(out)

    bad_fde = [None, {"chi2": CHI2, "max_exclude": -1}, {"chi2": CHI2, "max_exclude": 8}]
    for d, v in ((0, np.nan), (5, np.inf), (31, 0.0), (2, -1.0), (7, -np.inf)):
        c = list(CHI2)
        c[d] = v
        bad_fde.append({"chi2": c, "max_exclude": 1})
    for f in bad_fde:
        assert raw(mem[0].e, good, f) == (-3, bytes(sentinel)), f
    f = {"chi2": CHI2, "max_exclude": 1}
    bad_items = [[], good + good, [dict(good[6], a=M)], [dict(good[0], z=np.r_[np.nan, good[0]["z"][1:]])],
                 [dict(good[0], R=np.array([[np.inf]]))], [{"model": capi.AID_LINEAR, "a": 0, "b": 0, "z": np.zeros(1), "R": np.eye(1)}]]
    for items in bad_items:
        assert raw(mem[0].e, items, f) == (-3, bytes(sentinel)), [it["model"] for it in items]
    assert_unchanged(snapshot(mem[0].e), before[0])
    # in a batch, one bad member refuses the call for all; an un-fetched update returns ERR_STATE
    batch = capi.Batch([m.e for m in mem])
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_stack_update([good, [dict(good[6], a=M)]], fde=f)
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.aid_stack_update([good, good], fde={"chi2": CHI2, "max_exclude": 9})
    tb = capi.TrackBatch([0, 3], np.full(6, 0.01), [0, 1, 2], np.float64)
    mem[1].e.stage(capi.TRIANGULATE, tb)
    mem[1].e.launch()
    launched = mem[1].e.launch_count()
    with pytest.raises(RuntimeError, match="rc=-5"):
        batch.aid_stack_update([good, None], fde=f)
    assert raw(mem[1].e, good, f) == (-5, bytes(sentinel))
    assert mem[1].e.launch_count() == launched
    mem[1].e.fetch(1)
    batch.close()
    for i, (m, b) in enumerate(zip(mem, before)):
        assert_unchanged(snapshot(m.e)[:3] if i == 1 else snapshot(m.e), b[:3] if i == 1 else b)


def test_runner_with_nlos_ranges():
    """8 trials x 60 frames, four ranges and a plane range every frame, 10 % of the ranges 1 m long: FDE (alpha 0.01, two
    exclusions) excludes most injected faults and the ANIS of the applied stacks lies inside the bounds DESIGN 4.15 records"""
    truth = mc.make_truth(n_frames=60, seq=8)
    kw = dict(range_every=1, plane_every=1, range_outlier_rate=0.1, range_outlier_bias=1.0)
    rec, _ = mc.run(range(8), truth, dtype=np.float64, fde_alpha=0.01, fde_max_exclude=2, **kw)
    g = mc.summarize(rec)["range"]
    raw, _ = mc.run(range(8), truth, dtype=np.float64, **kw)
    g0 = mc.summarize(raw)["range"]
    print(f"NLOS run: FDE injected {g['injected']} excluded {g['faults_excluded']} clean excluded {g['clean_excluded']} missed "
          f"{g['faults_missed']} rejected {g['stacks_rejected']} ANIS {g['mean_anis']:.3f} ({g['mean_dof']:.2f} dof) bounds "
          f"{g['run_bounds']}; ungated injected {g0['injected']} missed {g0['faults_missed']} ANIS {g0['mean_anis']:.3f}")
    assert g["injected"] == g0["injected"] > 50
    assert g["faults_excluded"] >= 0.8 * g["injected"] and g["clean_excluded"] <= 0.05 * 5 * 480
    assert g["run_bounds"][0] * 0.97 <= g["mean_anis"] <= g["run_bounds"][1] * 1.03
