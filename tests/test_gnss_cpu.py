"""Host side of the GNSS and heading models of the stacked aided update without a GPU: the numpy models of montecarlo
(ANTENNA_POSITION, CLONE_ANTENNA_POSITION, HEADING, CLONE_HEADING) against the truth stream and against central differences,
the heading wrap, what the class forms (MSCKF::antennaPositionUpdate, cloneAntennaPositionUpdate, headingUpdate,
cloneHeadingUpdate) and MSCKFBatch::aidedUpdate(items) send to the C-ABI, and the Monte-Carlo runner's GNSS inputs and summary.

The C view is linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp)
plus tests/stub/stub_gnss_stack.cpp, which records every stacked item in full and calls the class forms on a view handle."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.test_shim_bookkeeping_cpu import shim_filter

GNSS = (capi.AID_ANTENNA_POSITION, capi.AID_CLONE_ANTENNA_POSITION, capi.AID_HEADING, capi.AID_CLONE_HEADING)
LEVER = np.array([0.3, -0.2, 0.5])
AXIS = np.array([1.0, 0.0, 0.0])


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_gnss_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / n for n in ("stub_engine.cpp", "stub_batch_state.cpp", "stub_aid.cpp", "stub_gnss_stack.cpp")]
    src += [csrc / n for n in ("filter_capi.cpp", "batch_capi.cpp", "aid_capi.cpp", "aid_stack_capi.cpp")]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", f"-I{csrc}", *map(str, src),
                               "-o", str(so)])
    return so


def _recorded(f):
    """([single calls, batched calls] naming f, the items of its last stacked call as dicts model, a, b, z, R)"""
    out = (C.c_longlong * 2)()
    rec = (C.c_double * (20 * 8))()
    n = f.lib.msckf_b200_stub_gnss_calls(C.c_void_p(f.engineHandle()), out, rec, 8)
    items = []
    for k in range(n):
        r = np.array(rec[20 * k:20 * k + 20])
        z, R = r[3:11], r[11:20]
        items.append({"model": int(r[0]), "a": int(r[1]), "b": int(r[2]), "z": z[np.isfinite(z)], "R": R[np.isfinite(R)]})
    return [out[0], out[1]], items


def _class_call(f, which, state_id=0, p=(0.0, 0.0, 0.0), v=(0.0, 0.0, 0.0), R=np.eye(3), mask=7, psi=0.0, var=1.0):
    R = np.ascontiguousarray(R, dtype=np.float64)
    res = capi.AidResult()
    rc = f.lib.msckf_b200_stub_gnss_class_call(f.h, C.c_int(which), C.c_int(state_id), (C.c_double * 3)(*p), (C.c_double * 3)(*v),
                                               R.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(R.shape[0]), C.c_int(mask),
                                               C.c_double(psi), C.c_double(var), C.byref(res))
    return rc, res


def _filters(lib, n, dtype, frames=4):
    wl = synth.make_stream_workload(n_frames=frames + 1, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        for fr in wl["frames"][:frames]:
            f.augmentState(fr["state_id"], fr["time"])
    return fs, wl


# ---- the numpy models ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("delay", [0, 1, 2, 3])
def test_truth_models_have_zero_residual(delay):
    """noise-free items of gnss_items from truth_imu at epoch g = f - delay against the truth state of frame f (its IMU state
    and its window of truth camera poses, synth.cam_pose): zero residual for all four models"""
    truth = mc.make_truth(n_frames=30, seq=8)
    lever_sets = (LEVER, np.zeros(3))
    for f in (5, 17, 29):
        g = f - delay
        ids = list(range(f - 4, f + 1))
        imu, poses = truth["truth_imu"][f], truth["truth_pose"][ids]
        for lever in lever_sets:
            for clone in ((None, ids.index(g)) if delay == 0 else (ids.index(g),)):
                items = mc.gnss_items(truth["truth_imu"][g], truth["camera"], np.zeros(3), np.zeros(1), 0.1, lever, 0.01, AXIS, clone)
                want = (capi.AID_ANTENNA_POSITION, capi.AID_HEADING) if clone is None else (capi.AID_CLONE_ANTENNA_POSITION, capi.AID_CLONE_HEADING)
                assert [it["model"] for it in items] == list(want)
                for it in items:
                    r = mc.odometry_residual(it, imu, poses)
                    assert np.abs(r).max() <= 1e-12, (f, delay, clone, it["model"], r)
    # the truth antenna position is p + C(q_IG)^T l with synth's own rotation, and the heading is the yaw of the IMU's x axis
    t = truth["frames"][7]["time"]
    R_GI = truth["traj"].R_GI(t)
    items = mc.gnss_items(truth["truth_imu"][7], truth["camera"], np.zeros(3), np.zeros(1), 0.1, LEVER, 0.01, AXIS)
    assert np.abs(items[0]["z"][0:3] - (truth["traj"].pos(t) + R_GI @ LEVER)).max() <= 1e-12
    assert abs(items[1]["z"][0] - math.atan2(R_GI[1, 0], R_GI[0, 0])) <= 1e-12


def _random_state(rng, M):
    imu = np.concatenate([rng.normal(size=15), rng.normal(size=4)])
    imu[15:19] /= np.linalg.norm(imu[15:19])
    poses = np.concatenate([rng.normal(size=(M, 3)), rng.normal(size=(M, 4))], axis=1)
    poses[:, 3:7] /= np.linalg.norm(poses[:, 3:7], axis=1, keepdims=True)
    return imu, poses


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(11)
    M = 6
    n = 15 + 6 * M
    imu, poses = _random_state(rng, M)
    est = {"imu": imu, "poses": poses}
    items = []
    for mask in range(1, 8):
        items.append({"model": capi.AID_ANTENNA_POSITION, "a": mask, "z": np.r_[rng.normal(size=3), rng.normal(size=3)], "R": np.eye(3)})
        items.append({"model": capi.AID_CLONE_ANTENNA_POSITION, "a": mask % M, "b": mask, "z": np.r_[rng.normal(size=3), rng.normal(size=3)],
                      "R": np.eye(3)})
    for k in range(M):
        items.append({"model": capi.AID_CLONE_HEADING, "a": k, "z": np.r_[0.3, rng.normal(size=3)], "R": np.eye(1)})
    items.append({"model": capi.AID_HEADING, "z": np.r_[-1.0, rng.normal(size=3)], "R": np.eye(1)})
    eps = 1e-6
    for it in items:
        m = len(mc.odometry_residual(it, imu, poses))
        Hcd = np.zeros((m, n))
        for k in range(n):
            e = np.zeros(n); e[k] = eps
            sp, sm = mc.perturb(est, e), mc.perturb(est, -e)
            dr = mc.odometry_residual(it, sp["imu"], sp["poses"]) - mc.odometry_residual(it, sm["imu"], sm["poses"])
            Hcd[:, k] = -np.array([mc.wrap_angle(x) for x in dr]) / (2 * eps)
        Ha = mc.odometry_jacobian(it, imu, poses, n)
        assert Ha.shape == (m, n)
        assert np.abs(Hcd - Ha).max() <= 1e-6, (it["model"], np.abs(Hcd - Ha).max())
        # non-zeros only over the pose's [dtheta, dp] (headings: dtheta)
        c0 = 15 + 6 * it["a"] if it["model"] in (capi.AID_CLONE_ANTENNA_POSITION, capi.AID_CLONE_HEADING) else 0
        cols = set(np.flatnonzero(np.abs(Ha).sum(axis=0)))
        allowed = set(range(c0, c0 + 3)) | (set() if it["model"] in (capi.AID_HEADING, capi.AID_CLONE_HEADING)
                                            else set(range(c0 + 3, c0 + 6)) if c0 else {12, 13, 14})
        assert cols <= allowed, (it["model"], cols)


def test_heading_wraps_across_pi():
    assert mc.wrap_angle(math.pi) == math.pi and mc.wrap_angle(-math.pi) == math.pi
    assert abs(mc.wrap_angle(3 * math.pi / 2) + math.pi / 2) <= 1e-15 and mc.wrap_angle(0.25) == 0.25
    for psi_hat, z, want in ((-3.1, 3.1, 6.2 - 2 * math.pi), (3.1, -3.1, 2 * math.pi - 6.2), (0.2, 0.1, -0.1)):
        Rz = np.array([[math.cos(psi_hat), -math.sin(psi_hat), 0.0], [math.sin(psi_hat), math.cos(psi_hat), 0.0], [0.0, 0.0, 1.0]])
        imu = np.zeros(19)
        imu[15:19] = synth.rot_to_quat(Rz.T)  # C(q_IG) = R_GI^T: the IMU's x axis points at yaw psi_hat
        assert abs(mc.heading_of(imu[15:19], AXIS) - psi_hat) <= 1e-12
        r = mc.odometry_residual({"model": capi.AID_HEADING, "z": np.r_[z, AXIS], "R": np.eye(1)}, imu, np.zeros((0, 7)))
        assert abs(r[0] - want) <= 1e-12, (psi_hat, z, r)
    assert abs((6.2 - 2 * math.pi) + 0.0832) < 1e-3


# ---- what the class and the C view send ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_class_forms_send_the_expected_items(stub_view, dtype):
    (f,), _ = _filters(stub_view, 1, dtype)
    ids = [int(x) for x in f.getCamStates()["state_id"]]
    assert len(ids) == 4
    p, lv = np.array([1.0, -2.0, 0.5]), np.array([0.3, -0.2, 0.5])
    R3 = np.array([[0.04, 0.001, 0.0], [0.001, 0.05, 0.002], [0.0, 0.002, 0.09]])
    R2 = R3[0:2, 0:2]
    base = _recorded(f)[0]
    cases = [  # (which, kwargs, expected item)
        (0, dict(p=p, v=lv, R=R3), {"model": capi.AID_ANTENNA_POSITION, "a": 7, "b": 0, "z": np.r_[p, lv], "R": R3.ravel()}),
        (0, dict(p=p, v=lv, R=R2, mask=0b011), {"model": capi.AID_ANTENNA_POSITION, "a": 3, "b": 0, "z": np.r_[p, lv], "R": R2.ravel()}),
        (1, dict(state_id=ids[1], p=p, v=lv, R=R3), {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": 1, "b": 7, "z": np.r_[p, lv], "R": R3.ravel()}),
        (1, dict(state_id=ids[3], p=p, v=np.zeros(3), R=np.eye(1) * 0.25, mask=0b100),
         {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": 3, "b": 4, "z": np.r_[p, 0, 0, 0], "R": np.array([0.25])}),
        (2, dict(psi=2.5, v=AXIS, var=0.01), {"model": capi.AID_HEADING, "a": 0, "b": 0, "z": np.r_[2.5, AXIS], "R": np.array([0.01])}),
        (3, dict(state_id=ids[2], psi=-1.0, v=lv, var=0.02), {"model": capi.AID_CLONE_HEADING, "a": 2, "b": 0, "z": np.r_[-1.0, lv],
                                                              "R": np.array([0.02])}),
    ]
    for k, (which, kw, want) in enumerate(cases):
        rc, res = _class_call(f, which, **kw)
        assert rc == 0 and res.applied == 1 and res.dof == round(math.sqrt(len(want["R"]))), (which, rc)
        calls, got = _recorded(f)
        assert calls == [base[0] + k + 1, base[1]]  # one C-ABI call per class call
        assert len(got) == 1
        for key in ("model", "a", "b"):
            assert got[0][key] == want[key], (which, key)
        assert np.array_equal(got[0]["z"], want["z"]) and np.array_equal(got[0]["R"], want["R"]), which
    n_calls = _recorded(f)[0]
    # refused before any device call: an id that is not in the window, a mask outside 1..7, R of the wrong size
    err = f.lib.msckf_mono_last_error
    err.restype = C.c_char_p
    for which, kw, msg in ((1, dict(state_id=max(ids) + 1, R=R3), "not in the window"), (3, dict(state_id=-5), "not in the window"),
                           (0, dict(mask=0, R=np.eye(1)), "mask"), (1, dict(state_id=ids[0], mask=8, R=R3), "mask"),
                           (0, dict(R=R2), "wrong shape"), (1, dict(state_id=ids[0], R=np.eye(1), mask=3), "wrong shape")):
        rc, _ = _class_call(f, which, **kw)
        assert rc == -1 and msg in err().decode(), (which, kw, err())
    assert _recorded(f)[0] == n_calls
    f.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_views_pass_items_through_unchanged(stub_view, dtype):
    """the C view's single and batched stacked calls (MSCKF::aidedUpdate(items), MSCKFBatch::aidedUpdate(items)) hand GNSS
    items to the C-ABI exactly as given, mixed with odometry, and leave unnamed members alone"""
    fs, wl = _filters(stub_view, 3, dtype)
    rng = np.random.default_rng(4)
    stack = [{"model": capi.AID_ANTENNA_POSITION, "a": 5, "z": rng.normal(size=6), "R": np.diag([0.1, 0.2])},
             {"model": capi.AID_CLONE_HEADING, "a": 2, "z": rng.normal(size=4), "R": np.array([[0.03]])},
             {"model": capi.AID_BODY_VELOCITY, "a": 0b110, "z": rng.normal(size=3), "R": np.eye(2)},
             {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": 3, "b": 6, "z": rng.normal(size=6), "R": np.array([[0.5, 0.1], [0.1, 0.7]])},
             {"model": capi.AID_HEADING, "z": rng.normal(size=4), "R": np.array([[0.02]])}]

    def check(f, items):
        got = _recorded(f)[1]
        assert len(got) == len(items)
        for g, it in zip(got, items):
            assert g["model"] == it["model"] and g["a"] == it.get("a", 0) and g["b"] == it.get("b", 0)
            assert np.array_equal(g["z"], np.asarray(it["z"], dtype=np.float64))
            assert np.array_equal(g["R"], np.asarray(it["R"], dtype=np.float64).ravel())

    base = [_recorded(f)[0] for f in fs]  # (the fake keys its counters by handle address, which a later filter may reuse)
    r = fs[0].aid_stack_update(stack)
    assert r["dof"] == 2 + 1 + 2 + 2 + 1 and _recorded(fs[0])[0] == [base[0][0] + 1, base[0][1]]
    check(fs[0], stack)
    fb = FilterBatch(fs)
    nb = fs[0].lib.msckf_b200_stub_gnss_batch_calls(C.c_void_p(fb.handle()))
    res = fb.aid_stack_update([stack[3:], None, stack[:2]])
    assert res[1] is None and res[0]["dof"] == 3 and res[2]["dof"] == 3
    assert fs[0].lib.msckf_b200_stub_gnss_batch_calls(C.c_void_p(fb.handle())) == nb + 1
    assert [[c[0] - b[0], c[1] - b[1]] for c, b in zip([_recorded(f)[0] for f in fs], base)] == [[1, 1], [0, 0], [0, 1]]
    check(fs[0], stack[3:])
    check(fs[2], stack[:2])
    fb.close()
    for f in fs:
        f.close()


# ---- the runner ------------------------------------------------------------------------------------------------------------
def test_gnss_leaves_the_trial_inputs_unchanged():
    truth = mc.make_truth(n_frames=40, seq=8)
    for k in (0, 3):
        a = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2, odo_every=2)
        b = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2, odo_every=2, gnss_every=3, heading_every=4)
        assert "gnss" not in a and "heading" not in a and len(b["gnss"]) == 40 and len(b["heading"]) == 40
        assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
        for key in a["injected"]:
            assert np.array_equal(a["injected"][key], b["injected"][key]), key
        for fa, fb_ in zip(a["frames"], b["frames"]):
            for key in ("update", "add"):
                assert np.array_equal(fa[key][0], fb_[key][0]) and np.array_equal(fa[key][1], fb_[key][1])
            for ra, rb in zip(fa["imu"], fb_["imu"]):
                assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
        for key in ("fixes", "odometry"):
            assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a[key], b[key])), key
        assert [f for f, n in enumerate(b["gnss"]) if n is not None] == list(range(2, 40, 3))
        assert [f for f, n in enumerate(b["heading"]) if n is not None] == list(range(3, 40, 4))
        assert all(n.shape == (3,) for n in b["gnss"] if n is not None) and all(n.shape == (1,) for n in b["heading"] if n is not None)
        # the fix noise does not depend on whether heading is on, and vice versa
        c = mc.make_trial(truth, k, gnss_every=3)
        d = mc.make_trial(truth, k, heading_every=4)
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(c["gnss"], b["gnss"]))
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(d["heading"], b["heading"]))
    # another trial draws other noise; the same trial the same noise
    g1 = mc.make_trial(truth, 1, gnss_every=1, heading_every=1)
    g0 = mc.make_trial(truth, 0, gnss_every=1, heading_every=1)
    assert not np.array_equal(g1["gnss"][3], g0["gnss"][3]) and not np.array_equal(g1["heading"][3], g0["heading"][3])
    again = mc.make_trial(truth, 1, gnss_every=1, heading_every=1)
    assert np.array_equal(g1["gnss"][3], again["gnss"][3]) and np.array_equal(g1["heading"][3], again["heading"][3])


def test_summary_reports_the_anis_of_the_gnss_stacks():
    from scipy import stats
    rng = np.random.default_rng(3)
    rows = [{c: 1.0 for c in mc.COMPONENTS} | {"dim_full": 21, "first_bad_pivot": -1} for _ in range(5)]
    recs = {}
    for k in range(10):
        dof = [3, 4, 4]
        g = [{"nis": rng.chisquare(d), "dof": d, "applied": 1, "status": 0} for d in dof]
        if k == 0:  # a dropped epoch (its clone had left the window) and a degenerate heading
            g[1] = {"nis": 0.0, "dof": 0, "applied": 0, "status": 0}
            g[2] = {"nis": float("nan"), "dof": 4, "applied": 0, "status": 2}
        recs[k] = mc.trial_record(rows, [0.0] * 5, gnss_rows=g)
    s = mc.summarize(recs)
    o = s["gnss"]
    assert o["dof"] == [30, 36, 36] and len(o["anis"]) == 3 and o["degenerate"] == 1
    assert abs(o["lower"][0] - stats.chi2.ppf(0.025, 30) / 10) < 1e-12 and abs(o["upper"][1] - stats.chi2.ppf(0.975, 36) / 9) < 1e-12
    assert abs(o["anis"][1] - sum(recs[k]["gnss"]["nis"][1] for k in range(1, 10)) / 9) < 1e-12
    assert abs(o["mean_dof"] - (30 + 36 + 36) / 28) < 1e-12 and o["applied"] == 1.0
    assert "gnss" not in mc.summarize({0: mc.trial_record(rows, [0.0] * 5)})
    assert "gnss" not in mc.trial_record(rows, [0.0] * 5)
