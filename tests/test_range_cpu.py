"""Host side of the range models of the stacked aided update without a GPU: the numpy models of montecarlo (RANGE, CLONE_RANGE,
PLANE_RANGE, CLONE_PLANE_RANGE) against the truth stream and against central differences, what the class forms
(MSCKF::rangeUpdate, cloneRangeUpdate, planeRangeUpdate, clonePlaneRangeUpdate) and MSCKFBatch::aidedUpdate(items) send to the
C-ABI, and the Monte-Carlo runner's ranging inputs and summary.

The C view is linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp)
plus tests/stub/stub_range_stack.cpp, which records every stacked item in full and calls the class forms on a view handle."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc, synth
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.test_shim_bookkeeping_cpu import shim_filter

RANGES = (capi.AID_RANGE, capi.AID_CLONE_RANGE, capi.AID_PLANE_RANGE, capi.AID_CLONE_PLANE_RANGE)
LEVER = np.array([0.3, -0.2, 0.5])
PLANE_LEVER = np.array([0.1, 0.2, -0.1])
TILTED = np.array([-1.0, 0.2, 0.1])  # a beam about 13 degrees off the IMU's downward axis


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_range_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / n for n in ("stub_engine.cpp", "stub_batch_state.cpp", "stub_aid.cpp", "stub_range_stack.cpp")]
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
    n = f.lib.msckf_b200_stub_range_calls(C.c_void_p(f.engineHandle()), out, rec, 8)
    items = []
    for k in range(n):
        r = np.array(rec[20 * k:20 * k + 20])
        z, R = r[3:11], r[11:20]
        items.append({"model": int(r[0]), "a": int(r[1]), "b": int(r[2]), "z": z[np.isfinite(z)], "R": R[np.isfinite(R)]})
    return [out[0], out[1]], items


def _class_call(f, which, state_id=0, rho=1.0, h=0.0, anchor=(0.0, 0.0, 0.0), lever=(0.0, 0.0, 0.0), axis=(-1.0, 0.0, 0.0), var=1.0):
    res = capi.AidResult()
    rc = f.lib.msckf_b200_stub_range_class_call(f.h, C.c_int(which), C.c_int(state_id), C.c_double(rho), C.c_double(h),
                                                (C.c_double * 3)(*anchor), (C.c_double * 3)(*lever), (C.c_double * 3)(*axis),
                                                C.c_double(var), C.byref(res))
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
    """noise-free items of range_items from truth_imu at epoch g = f - delay against the truth state of frame f (its IMU state
    and its window of truth camera poses, synth.cam_pose): zero residual for all four models, straight down and on a tilted beam"""
    truth = mc.make_truth(n_frames=30, seq=8)
    for f in (5, 17, 29):
        g = f - delay
        ids = list(range(f - 4, f + 1))
        imu, poses = truth["truth_imu"][f], truth["truth_pose"][ids]
        for lever, plane_lever, axis in ((LEVER, PLANE_LEVER, TILTED), (np.zeros(3), np.zeros(3), np.array(mc.PLANE_AXIS))):
            for clone in ((None, ids.index(g)) if delay == 0 else (ids.index(g),)):
                items = mc.range_items(truth["truth_imu"][g], truth["camera"], np.zeros(len(mc.ANCHORS)), np.zeros(1), 0.1, lever,
                                       0.02, mc.PLANE_HEIGHT, plane_lever, axis, clone)
                want = (capi.AID_RANGE,) * 4 + (capi.AID_PLANE_RANGE,) if clone is None else (capi.AID_CLONE_RANGE,) * 4 + (capi.AID_CLONE_PLANE_RANGE,)
                assert [it["model"] for it in items] == list(want)
                for it in items:
                    r = mc.odometry_residual(it, imu, poses)
                    assert r.shape == (1,) and abs(r[0]) <= 1e-12, (f, delay, clone, it["model"], r)
    # the truth ranges with synth's own rotation: to each anchor, and straight down to the ground at h = -1.5 m
    t = truth["frames"][7]["time"]
    R_GI, p = truth["traj"].R_GI(t), truth["traj"].pos(t)
    items = mc.range_items(truth["truth_imu"][7], truth["camera"], np.zeros(4), np.zeros(1), 0.1, LEVER, 0.02, mc.PLANE_HEIGHT,
                           np.zeros(3), np.array([0.0, 0.0, 0.0]) + mc.PLANE_AXIS)
    for it, a in zip(items[:4], mc.ANCHORS):
        assert abs(it["z"][0] - np.linalg.norm(p + R_GI @ LEVER - a)) <= 1e-12
    b = R_GI @ np.array(mc.PLANE_AXIS)
    assert b[2] < -0.99 and abs(items[4]["z"][0] - (mc.PLANE_HEIGHT - p[2]) / b[2]) <= 1e-12 and 1.2 < items[4]["z"][0] < 1.8
    # the anchors are not coplanar
    A = mc.ANCHORS[1:] - mc.ANCHORS[0]
    assert abs(np.linalg.det(A)) > 1.0


def _random_state(rng, M):
    imu = np.concatenate([rng.normal(size=15), rng.normal(size=4)])
    imu[15:19] /= np.linalg.norm(imu[15:19])
    poses = np.concatenate([rng.normal(size=(M, 3)), rng.normal(size=(M, 4))], axis=1)
    poses[:, 3:7] /= np.linalg.norm(poses[:, 3:7], axis=1, keepdims=True)
    return imu, poses


def _plane_item(rng, q, model, clone, lever, beam_G, length=1.0):
    """a plane range whose beam points along beam_G in G (given in the body frame of q), lever in the body frame, plane 3 m below"""
    axis = mc.quat_to_rot(q) @ (np.asarray(beam_G, dtype=np.float64) / np.linalg.norm(beam_G)) * length
    it = {"model": model, "z": np.r_[1.0 + rng.random(), -3.0, lever, axis], "R": np.eye(1)}
    if clone is not None:
        it["a"] = clone
    return it


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(11)
    M = 6
    n = 15 + 6 * M
    imu, poses = _random_state(rng, M)
    est = {"imu": imu, "poses": poses}
    items = []
    for k in range(M):
        items.append({"model": capi.AID_CLONE_RANGE, "a": k, "z": np.r_[3.0, 4 * rng.normal(size=3), 0.5 * rng.normal(size=3)], "R": np.eye(1)})
        items.append(_plane_item(rng, poses[k, 3:7], capi.AID_CLONE_PLANE_RANGE, k, 0.5 * rng.normal(size=3), [0.4, -0.3, -1.0], 2.5))
    for lever in (np.zeros(3), LEVER):
        items.append({"model": capi.AID_RANGE, "z": np.r_[3.0, 4 * rng.normal(size=3), lever], "R": np.eye(1)})
        for beam in ([0.0, 0.0, -1.0], [0.5, 0.2, -1.0], [0.0, 0.0, 1.0]):  # straight down, tilted, and up at a plane above
            it = _plane_item(rng, imu[15:19], capi.AID_PLANE_RANGE, None, lever, beam, 0.7)
            if beam[2] > 0:
                it["z"][1] = imu[2] + 4.0
            items.append(it)
    eps = 1e-6
    for it in items:
        if it["model"] in (capi.AID_PLANE_RANGE, capi.AID_CLONE_PLANE_RANGE):
            q, p = (imu[15:19], imu[0:3]) if it["model"] == capi.AID_PLANE_RANGE else (poses[it["a"], 3:7], poses[it["a"], 0:3])
            assert mc.plane_range_of(p, q, it["z"][1], it["z"][2:5], it["z"][5:8]) > 0.0  # (a plane in front of the sensor)
        r0 = mc.odometry_residual(it, imu, poses)
        assert r0.shape == (1,)
        Hcd = np.zeros((1, n))
        for k in range(n):
            e = np.zeros(n); e[k] = eps
            sp, sm = mc.perturb(est, e), mc.perturb(est, -e)
            Hcd[:, k] = -(mc.odometry_residual(it, sp["imu"], sp["poses"]) - mc.odometry_residual(it, sm["imu"], sm["poses"])) / (2 * eps)
        Ha = mc.odometry_jacobian(it, imu, poses, n)
        assert Ha.shape == (1, n)
        assert np.abs(Hcd - Ha).max() <= 1e-6, (it["model"], np.abs(Hcd - Ha).max())
        # non-zeros only over the pose's dtheta and dp (plane ranges: dp_z), at most 6
        c0 = 15 + 6 * it["a"] if it["model"] in (capi.AID_CLONE_RANGE, capi.AID_CLONE_PLANE_RANGE) else 0
        cp = c0 + 3 if c0 else 12
        cols = set(np.flatnonzero(Ha[0]))
        allowed = set(range(c0, c0 + 3)) | ({cp + 2} if it["model"] in (capi.AID_PLANE_RANGE, capi.AID_CLONE_PLANE_RANGE) else set(range(cp, cp + 3)))
        assert cols <= allowed, (it["model"], cols)


def test_plane_range_of_a_level_body():
    """a body at height 0.4 m whose beam points straight down sees a plane 1.5 m below at 1.9 m, and 1.9 / cos(t) on a beam
    tilted by t; a beam pointing up sees the floor behind it (a negative range)"""
    q = np.array([0.0, 0.0, 0.0, 1.0])  # C = I: body axes are G's
    p = np.array([3.0, -1.0, 0.4])
    assert abs(mc.plane_range_of(p, q, -1.5, np.zeros(3), [0.0, 0.0, -2.0]) - 1.9) <= 1e-15
    t = 0.3
    assert abs(mc.plane_range_of(p, q, -1.5, np.zeros(3), [math.sin(t), 0.0, -math.cos(t)]) - 1.9 / math.cos(t)) <= 1e-14
    assert abs(mc.plane_range_of(p, q, -1.5, [0.0, 0.0, -0.1], [0.0, 0.0, -1.0]) - 1.8) <= 1e-15
    assert mc.plane_range_of(p, q, -1.5, np.zeros(3), [0.0, 0.0, 1.0]) < 0.0
    assert abs(mc.range_of(p, q, [0.0, 0.0, 0.6], [0.0, 3.0, 1.0]) - 5.0) <= 1e-15


# ---- what the class and the C view send ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_class_forms_send_the_expected_items(stub_view, dtype):
    (f,), _ = _filters(stub_view, 1, dtype)
    ids = [int(x) for x in f.getCamStates()["state_id"]]
    assert len(ids) == 4
    a, lv, ax = np.array([5.0, -5.0, 2.0]), np.array([0.3, -0.2, 0.5]), np.array([-1.0, 0.2, 0.1])
    base = _recorded(f)[0]
    cases = [  # (which, kwargs, expected item)
        (0, dict(rho=7.5, anchor=a, lever=lv, var=0.01), {"model": capi.AID_RANGE, "a": 0, "b": 0, "z": np.r_[7.5, a, lv], "R": [0.01]}),
        (1, dict(state_id=ids[1], rho=6.0, anchor=a, lever=lv, var=0.04),
         {"model": capi.AID_CLONE_RANGE, "a": 1, "b": 0, "z": np.r_[6.0, a, lv], "R": [0.04]}),
        (2, dict(rho=1.4, h=-1.5, lever=lv, axis=ax, var=4e-4),
         {"model": capi.AID_PLANE_RANGE, "a": 0, "b": 0, "z": np.r_[1.4, -1.5, lv, ax], "R": [4e-4]}),
        (3, dict(state_id=ids[3], rho=2.0, h=3.0, lever=np.zeros(3), axis=-ax, var=1e-3),
         {"model": capi.AID_CLONE_PLANE_RANGE, "a": 3, "b": 0, "z": np.r_[2.0, 3.0, 0, 0, 0, -ax], "R": [1e-3]}),
    ]
    for k, (which, kw, want) in enumerate(cases):
        rc, res = _class_call(f, which, **kw)
        assert rc == 0 and res.applied == 1 and res.dof == 1, (which, rc)
        calls, got = _recorded(f)
        assert calls == [base[0] + k + 1, base[1]]  # one C-ABI call per class call
        assert len(got) == 1
        for key in ("model", "a", "b"):
            assert got[0][key] == want[key], (which, key)
        assert np.array_equal(got[0]["z"], want["z"]) and np.array_equal(got[0]["R"], np.array(want["R"])), which
    n_calls = _recorded(f)[0]
    # refused before any device call: an id that is not in the window
    err = f.lib.msckf_mono_last_error
    err.restype = C.c_char_p
    for which, sid in ((1, max(ids) + 1), (3, -5), (1, min(ids) - 1)):
        rc, _ = _class_call(f, which, state_id=sid)
        assert rc == -1 and "not in the window" in err().decode(), (which, sid, err())
    assert _recorded(f)[0] == n_calls
    f.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_views_pass_items_through_unchanged(stub_view, dtype):
    """the C view's single and batched stacked calls (MSCKF::aidedUpdate(items), MSCKFBatch::aidedUpdate(items)) hand range
    items to the C-ABI exactly as given, mixed with odometry and GNSS, and leave unnamed members alone"""
    fs, wl = _filters(stub_view, 3, dtype)
    rng = np.random.default_rng(4)
    stack = [{"model": capi.AID_RANGE, "z": rng.normal(size=7), "R": np.array([[0.01]])},
             {"model": capi.AID_CLONE_PLANE_RANGE, "a": 2, "z": rng.normal(size=8), "R": np.array([[0.03]])},
             {"model": capi.AID_BODY_VELOCITY, "a": 0b110, "z": rng.normal(size=3), "R": np.eye(2)},
             {"model": capi.AID_CLONE_RANGE, "a": 3, "z": rng.normal(size=7), "R": np.array([[0.5]])},
             {"model": capi.AID_ANTENNA_POSITION, "a": 5, "z": rng.normal(size=6), "R": np.diag([0.1, 0.2])},
             {"model": capi.AID_PLANE_RANGE, "z": rng.normal(size=8), "R": np.array([[0.02]])}]

    def check(f, items):
        got = _recorded(f)[1]
        assert len(got) == len(items)
        for g, it in zip(got, items):
            assert g["model"] == it["model"] and g["a"] == it.get("a", 0) and g["b"] == it.get("b", 0)
            assert np.array_equal(g["z"], np.asarray(it["z"], dtype=np.float64))
            assert np.array_equal(g["R"], np.asarray(it["R"], dtype=np.float64).ravel())

    base = [_recorded(f)[0] for f in fs]  # (the fake keys its counters by handle address, which a later filter may reuse)
    r = fs[0].aid_stack_update(stack)
    assert r["dof"] == 1 + 1 + 2 + 1 + 2 + 1 and _recorded(fs[0])[0] == [base[0][0] + 1, base[0][1]]
    check(fs[0], stack)
    fb = FilterBatch(fs)
    nb = fs[0].lib.msckf_b200_stub_range_batch_calls(C.c_void_p(fb.handle()))
    res = fb.aid_stack_update([stack[3:], None, stack[:2]])
    assert res[1] is None and res[0]["dof"] == 4 and res[2]["dof"] == 2
    assert fs[0].lib.msckf_b200_stub_range_batch_calls(C.c_void_p(fb.handle())) == nb + 1
    assert [[c[0] - b[0], c[1] - b[1]] for c, b in zip([_recorded(f)[0] for f in fs], base)] == [[1, 1], [0, 0], [0, 1]]
    check(fs[0], stack[3:])
    check(fs[2], stack[:2])
    fb.close()
    for f in fs:
        f.close()


# ---- the runner ------------------------------------------------------------------------------------------------------------
def test_ranging_leaves_the_trial_inputs_unchanged():
    truth = mc.make_truth(n_frames=40, seq=8)
    for k in (0, 3):
        a = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2, odo_every=2, gnss_every=3, heading_every=4)
        b = mc.make_trial(truth, k, fix_every=5, fix_sigma=0.2, odo_every=2, gnss_every=3, heading_every=4, range_every=2, plane_every=3)
        assert "range" not in a and "plane" not in a and len(b["range"]) == 40 and len(b["plane"]) == 40
        assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
        assert a["imu_state"].keys() == b["imu_state"].keys()
        assert all(np.array_equal(a["imu_state"][key], b["imu_state"][key]) for key in a["imu_state"])
        for key in a["injected"]:
            assert np.array_equal(a["injected"][key], b["injected"][key]), key
        for fa, fb_ in zip(a["frames"], b["frames"]):
            assert fa["state_id"] == fb_["state_id"] and fa["time"] == fb_["time"]
            for key in ("update", "add"):
                assert np.array_equal(fa[key][0], fb_[key][0]) and np.array_equal(fa[key][1], fb_[key][1])
            for ra, rb in zip(fa["imu"], fb_["imu"]):
                assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
        for key in ("fixes", "odometry", "gnss", "heading"):
            assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a[key], b[key])), key
        assert [f for f, n in enumerate(b["range"]) if n is not None] == list(range(1, 40, 2))
        assert [f for f, n in enumerate(b["plane"]) if n is not None] == list(range(2, 40, 3))
        assert all(n.shape == (len(mc.ANCHORS),) for n in b["range"] if n is not None) and all(n.shape == (1,) for n in b["plane"] if n is not None)
        # the range noise does not depend on whether the plane is on, and vice versa
        c = mc.make_trial(truth, k, range_every=2)
        d = mc.make_trial(truth, k, plane_every=3)
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(c["range"], b["range"]))
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(d["plane"], b["plane"]))
    # another trial draws other noise; the same trial the same noise; the streams are not the GNSS streams
    g1 = mc.make_trial(truth, 1, range_every=1, plane_every=1, gnss_every=1, heading_every=1)
    g0 = mc.make_trial(truth, 0, range_every=1, plane_every=1)
    assert not np.array_equal(g1["range"][3], g0["range"][3]) and not np.array_equal(g1["plane"][3], g0["plane"][3])
    again = mc.make_trial(truth, 1, range_every=1, plane_every=1)
    assert np.array_equal(g1["range"][3], again["range"][3]) and np.array_equal(g1["plane"][3], again["plane"][3])
    assert not np.array_equal(g1["range"][3][0:3], g1["gnss"][3]) and not np.array_equal(g1["plane"][3], g1["heading"][3])


def test_summary_reports_the_anis_of_the_ranging_stacks():
    from scipy import stats
    rng = np.random.default_rng(3)
    rows = [{c: 1.0 for c in mc.COMPONENTS} | {"dim_full": 21, "first_bad_pivot": -1} for _ in range(5)]
    recs = {}
    for k in range(10):
        dof = [5, 4, 5]
        r = [{"nis": rng.chisquare(d), "dof": d, "applied": 1, "status": 0} for d in dof]
        g = [{"nis": rng.chisquare(3), "dof": 3, "applied": 1, "status": 0}]
        if k == 0:  # a dropped epoch (its clone had left the window) and a degenerate plane range
            r[1] = {"nis": 0.0, "dof": 0, "applied": 0, "status": 0}
            r[2] = {"nis": float("nan"), "dof": 5, "applied": 0, "status": 2}
        recs[k] = mc.trial_record(rows, [0.0] * 5, gnss_rows=g, range_rows=r)
    s = mc.summarize(recs)
    o = s["range"]
    assert o["dof"] == [50, 36, 45] and len(o["anis"]) == 3 and o["degenerate"] == 1
    assert abs(o["lower"][0] - stats.chi2.ppf(0.025, 50) / 10) < 1e-12 and abs(o["upper"][1] - stats.chi2.ppf(0.975, 36) / 9) < 1e-12
    assert abs(o["anis"][1] - sum(recs[k]["range"]["nis"][1] for k in range(1, 10)) / 9) < 1e-12
    assert abs(o["mean_dof"] - (50 + 36 + 45) / 28) < 1e-12 and o["applied"] == 1.0
    assert o["run_bounds"] == list(mc.chi2_bounds(50 + 36 + 45, 28))
    assert abs(o["mean_anis"] - sum(x for k in recs for x in recs[k]["range"]["nis"] if np.isfinite(x) and x > 0) / 28) < 1e-12
    # the GNSS stacks are summarised beside them, unchanged
    assert s["gnss"]["dof"] == [30] and s["gnss"]["degenerate"] == 0
    assert s["gnss"] == mc.summarize({k: mc.trial_record(rows, [0.0] * 5, gnss_rows=[{"nis": recs[k]["gnss"]["nis"][0], "dof": 3,
                                                                                       "applied": 1, "status": 0}]) for k in recs})["gnss"]
    assert "range" not in mc.summarize({0: mc.trial_record(rows, [0.0] * 5)})
    assert "range" not in mc.trial_record(rows, [0.0] * 5, gnss_rows=[])
