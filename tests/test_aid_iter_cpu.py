"""The dense iterated stacked aided update (tests/aid_iter_reference.py) without a device: one linearisation is the Joseph-form
update, linear models converge at once, converged results are Gauss-Newton stationary points, and on the anchor toy the
iteration restores the consistency one linearisation loses after drift.  Also what the class and C view forms send to the
C-ABI, through a recording fake of the iterated entry points (tests/stub/stub_aid_iter.cpp), and the runner's trial inputs
with --range-start / --gnss-start."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests import aid_iter_reference as ref
from tests.aid_fde_reference import linearise
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)
from tests.test_shim_bookkeeping_cpu import shim_filter


def _drifted(rng, M, drift, kinds=None):
    """(items measured at a truth, the estimate imu / poses, P): the truth is the estimate moved by a draw from P"""
    imu = np.zeros(19)
    imu[0:3], imu[3:6] = [1.0, 2.0, 1.5], [0.5, -0.2, 0.1]
    q = rng.normal(size=4)
    imu[15:19] = q / np.linalg.norm(q)
    poses = np.zeros((M, 7))
    for k in range(M):
        poses[k, 0:3] = imu[0:3] + 0.3 * rng.normal(size=3)
        qk = rng.normal(size=4)
        poses[k, 3:7] = qk / np.linalg.norm(qk)
    P = ref.drift_prior(rng, M, drift)
    t_imu, t_poses = ref.boxplus(imu, poses, np.linalg.cholesky(P) @ rng.normal(size=len(P)))
    items = ref.scene(rng, t_imu, t_poses, M) if kinds is None else ref.scene(rng, t_imu, t_poses, M, kinds)
    return items, imu, poses, P


@pytest.mark.parametrize("M", [0, 1, 3])
def test_one_linearisation_is_the_joseph_update(M):
    rng = np.random.default_rng(1 + M)
    for drift in (0.05, 0.3, 1.0):
        items, imu, poses, P = _drifted(rng, M, drift)
        for max_iter in (0, 1):
            got = ref.iekf(items, imu, poses, P, max_iter=max_iter)
            Pj, dx, nis = ref.one_linearisation(items, imu, poses, P)
            assert np.abs(got["P"] - Pj).max() <= 1e-12 * np.abs(Pj).max()
            assert np.abs(got["dx"] - dx).max() <= 1e-12 * max(np.abs(dx).max(), 1.0)
            assert abs(got["nis"] - nis) <= 1e-12 * max(nis, 1.0)
            assert (got["iterations"], got["converged"], got["step"]) == (1, 0, 0.0)


def test_linear_models_converge_at_the_second_linearisation():
    """VELOCITY / POSITION: H does not depend on the state, so delta_2 = delta_1 and P is one linearisation's"""
    rng = np.random.default_rng(7)
    imu = np.zeros(19)
    imu[0:3], imu[3:6], imu[18] = [1.0, 2.0, 1.5], [0.5, -0.2, 0.1], 1.0
    poses = np.zeros((2, 7))
    poses[:, 6] = 1.0
    P = ref.drift_prior(rng, 2, 1.0)
    items = [{"model": capi.AID_POSITION, "a": 0, "b": 0, "z": imu[0:3] + rng.normal(size=3), "R": 0.01 * np.eye(3)},
             {"model": capi.AID_VELOCITY, "a": 0, "b": 0, "z": imu[3:6] + rng.normal(size=3), "R": 0.04 * np.eye(3)}]
    one = ref.iekf(items, imu, poses, P, max_iter=1)
    got = ref.iekf(items, imu, poses, P, max_iter=8, tol=1e-12)
    assert got["iterations"] == 2 and got["converged"] == 1 and got["step"] <= 1e-14
    assert np.abs(got["P"] - one["P"]).max() <= 1e-14 * np.abs(one["P"]).max()


@pytest.mark.parametrize("drift", [0.05, 0.3, 1.0])
def test_converged_results_are_stationary(drift):
    """P^-1 delta = H^T R^-1 r with H, r at the last iterate (Gauss-Newton on the MAP cost)"""
    rng = np.random.default_rng(int(drift * 100))
    seen = 0
    for M in (0, 1, 2, 3, 4, 5):
        items, imu, poses, P = _drifted(rng, M, drift)
        got = ref.iekf(items, imu, poses, P, max_iter=16, tol=1e-11)
        if not got["converged"]:
            continue
        seen += 1
        H, r = ref.stacked(items, *ref.boxplus(imu, poses, got["dx"]), len(P))
        assert ref.stationarity(P, H, r, got["R"], got["dx"]) <= 1e-9
    assert seen >= (3 if drift < 1.0 else 1)  # (at 1 m the heading's pull makes the convergence slow: 1 of these 6 in 16)


def test_iterate_linearises_where_the_device_does():
    """the iterate of a clone and of the IMU: montecarlo's injection, the clone quaternion renormalised, the IMU's not"""
    rng = np.random.default_rng(3)
    _, imu, poses, P = _drifted(rng, 2, 0.3)
    d = np.linalg.cholesky(P) @ rng.normal(size=len(P))
    i2, p2 = ref.boxplus(imu, poses, d)
    assert np.allclose(np.linalg.norm(p2[:, 3:7], axis=1), 1.0, atol=1e-15)
    assert np.allclose(mc.error_state({"imu": i2, "poses": p2}, {"imu": imu, "poses": poses}), d, atol=1e-9)
    items = ref.scene(rng, i2, p2, 2)
    assert len(items) == 8 and sum(len(h) for h, _ in linearise(items, i2, p2, len(P))) == 17


def test_anchor_toy_consistency():
    """four anchors, range sigma 0.1 m, P = sigma_p^2 I: at sigma_p = 1 m one linearisation is far outside the 95 % bounds of
    the ANEES (3 dof, 2000 draws) and four linearisations are inside them"""
    lo, hi = mc.chi2_bounds(3 * 2000, 2000)
    one = ref.anchor_toy(np.random.default_rng(2024), 1.0, 1)
    four = ref.anchor_toy(np.random.default_rng(2024), 1.0, 4)
    print(f"anchor toy sigma_p 1 m: ANEES one linearisation {one:.2f}, four {four:.2f}, bounds [{lo:.2f}, {hi:.2f}]")
    assert one > hi
    assert lo <= four <= hi


# ---- the class and C view forms over a fake of the iterated entry points -------------------------------------------------------


def _recorded(f):
    """(single calls, batched calls, IMU readings handed over before the last iterated call, max_iter, tol, chi2_max (NaN:
    FDE), max_exclude (-1: no FDE), the item models) of the fake for filter f"""
    rec = (C.c_double * 13)()
    f.lib.msckf_b200_stub_aid_iter_calls(C.c_void_p(f.engineHandle()), rec)
    r = list(rec)
    return (int(r[0]), int(r[1]), int(r[2]), r[3], r[4], r[5], r[6], [int(m) for m in r[8:8 + int(r[7])]])


def _filters(lib, n, dtype, frames=4):
    wl = synth.make_stream_workload(n_frames=frames + 1, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:frames]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs, wl


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_views_pass_the_iteration_options_through(stub_view, dtype):
    """MSCKF::aidedUpdate(items, chi2_max | fde, iter, iter_out) and the MSCKFBatch forms through the C view: one C-ABI call per
    class call with the IMU queue handed over first, max_iter / tol / chi2_max / fde passed as given, the results returned;
    options the C-ABI would refuse throw std::invalid_argument in the class before any call"""
    fs, wl = _filters(stub_view, 3, dtype)
    rng = np.random.default_rng(9)
    stack = [{"model": capi.AID_RANGE, "z": rng.normal(size=7), "R": np.array([[0.01]])},
             {"model": capi.AID_CLONE_PLANE_RANGE, "a": 2, "z": rng.normal(size=8), "R": np.array([[0.03]])},
             {"model": capi.AID_ANTENNA_POSITION, "a": 7, "z": rng.normal(size=6), "R": np.diag([0.1, 0.2, 0.3])}]
    fde = {"chi2": [float(x) for x in 1.0 + rng.random(32)], "max_exclude": 3}
    models = [it["model"] for it in stack]
    base = [_recorded(f)[:2] for f in fs]  # (the fake's records outlive the filters: a handle may reuse a freed address)
    count = lambda f, i: tuple(c - b for c, b in zip(_recorded(f)[:2], base[i]))  # noqa: E731
    for (omega, a, dT) in wl["frames"][4]["imu"][:3]:
        fs[0].propagate(omega, a, dT)
    r = fs[0].aid_stack_update(stack, chi2_max=7.5, max_iter=6, tol=1e-8)
    _, _, readings, mi, tol, chi2_max, K, got = _recorded(fs[0])
    assert count(fs[0], 0) == (1, 0) and (mi, tol, chi2_max, K, got) == (6.0, 1e-8, 7.5, -1.0, models)
    assert readings >= 3  # the queued readings reached the engine before the update
    assert (r["iterations"], r["converged"], r["step"], r["applied"], r["dof"]) == (6, 1, 5e-9, 1, 3)
    r = fs[0].aid_stack_update(stack, fde=fde, max_iter=0, tol=0.0)
    _, _, _, mi, tol, chi2_max, K, _ = _recorded(fs[0])
    assert count(fs[0], 0) == (2, 0) and (mi, tol, K) == (0.0, 0.0, 3.0) and np.isnan(chi2_max)
    assert r["outcome"] == 0 and r["iterations"] == 1 and len(r["items"]) == 3
    fb = FilterBatch(fs)
    res = fb.aid_stack_update([stack, None, stack[:1]], chi2_max=2.0, max_iter=[4, 0, 16], tol=[1e-6, 0.0, 1e-3])
    assert res[1] is None and (res[0]["iterations"], res[2]["iterations"]) == (4, 16) and res[2]["step"] == 5e-4
    assert [count(f, i)[1] for i, f in enumerate(fs)] == [1, 0, 1]
    assert _recorded(fs[0])[3:6] == (4.0, 1e-6, 2.0) and _recorded(fs[2])[3:5] == (16.0, 1e-3)
    res = fb.aid_stack_update([None, stack, stack], fde=fde, max_iter=2, tol=1e-9)
    assert res[0] is None and res[1]["outcome"] == 0 and _recorded(fs[1])[6] == 3.0
    assert fb.lib.msckf_b200_stub_batch_aid_iter_calls(C.c_void_p(fb.handle())) == 2
    # refused in the class: nothing reaches the C-ABI
    err = fs[0].lib.msckf_mono_last_error
    err.restype = C.c_char_p
    calls = [count(f, i) for i, f in enumerate(fs)]
    for mi, tol in ((-1, 0.0), (17, 0.0), (4, np.nan), (4, np.inf), (4, -1e-3)):
        with pytest.raises(RuntimeError):
            fs[0].aid_stack_update(stack, max_iter=mi, tol=tol)
        assert "iter" in err().decode()
        with pytest.raises(RuntimeError):
            fs[0].aid_stack_update(stack, fde=fde, max_iter=mi, tol=tol)
        with pytest.raises(RuntimeError):
            fb.aid_stack_update([stack, None, stack], max_iter=[4, 4, mi], tol=[0.0, 0.0, tol])
        assert "iter" in err().decode()
        with pytest.raises(RuntimeError):
            fb.aid_stack_update([stack, None, stack], fde=fde, max_iter=mi, tol=tol)
    fb.aid_stack_update([stack, None, None], max_iter=[4, -1, 99], tol=[0.0, np.nan, -1.0])  # (not read for filters left alone)
    assert [count(f, i) for i, f in enumerate(fs)] == [(calls[0][0], calls[0][1] + 1)] + calls[1:]
    fb.close()
    for f in fs:
        f.close()


# ---- the Monte-Carlo runner ----------------------------------------------------------------------------------------------------
def test_runner_trial_inputs_do_not_depend_on_the_start_or_the_iterations():
    """--range-start / --gnss-start only blank the epochs before the start (the noise is drawn all the same), and the iteration
    options change no trial input"""
    truth = mc.make_truth(n_frames=40, seq=8)
    kw = dict(range_every=1, plane_every=2, gnss_every=1, heading_every=3)
    a = mc.make_trial(truth, 3, 0, **kw)
    b = mc.make_trial(truth, 3, 0, range_start=30, gnss_start=20, **kw)
    for key in ("range", "plane", "gnss", "heading"):
        start = 30 if key in ("range", "plane") else 20
        for f, (x, y) in enumerate(zip(a[key], b[key])):
            if f < start:
                assert y is None
            else:
                assert (x is None and y is None) or np.array_equal(x, y), (key, f)
    for fa, fb_ in zip(a["frames"], b["frames"]):
        for (wa, aa, da), (wb, ab, db) in zip(fa["imu"], fb_["imu"]):
            assert np.array_equal(wa, wb) and np.array_equal(aa, ab) and da == db
        assert np.array_equal(fa["update"][0], fb_["update"][0]) and np.array_equal(fa["add"][0], fb_["add"][0])
    assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
    for k in a["injected"]:
        assert np.array_equal(a["injected"][k], b["injected"][k])
