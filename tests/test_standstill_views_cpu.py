"""Host side of the standstill update without a GPU: MSCKF::standstillUpdate, MSCKFBatch::standstillUpdate and the at-rest
class forms through the C view, linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp,
stub_batch_state.cpp) plus tests/stub/stub_standstill.cpp.  The readings, the cfg and the result travel unchanged, queued
IMU readings are handed over first, members without readings are left alone, and bad input is refused before any call."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from msckf_mono_b200 import capi, synth
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.test_shim_bookkeeping_cpu import shim_filter

DTYPES = [np.float32, np.float64]
CFG = {"noise_scale": 1.5, "sigma_v": 0.01, "scatter_max": 2.0, "chi2_max": 30.0}


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_standstill_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / "stub_engine.cpp", ROOT / "tests" / "stub" / "stub_batch_state.cpp",
           ROOT / "tests" / "stub" / "stub_standstill.cpp", csrc / "filter_capi.cpp", csrc / "batch_capi.cpp", csrc / "standstill_capi.cpp"]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", f"-I{csrc}", *map(str, src),
                               "-o", str(so)])
    return so


def _calls(f):
    """(single calls, batched calls, readings handed over before the last call, stacked calls), cfg, readings [k, 7].  (The
    fake keys its records by engine address, which an earlier, closed filter may have had: the tests compare call counts.)"""
    out, cfg, r = (C.c_longlong * 4)(), (C.c_double * 4)(), (C.c_double * (7 * 512))()
    k = f.lib.msckf_b200_stub_standstill_calls(C.c_void_p(f.engineHandle()), out, cfg, r, 512)
    return list(out), list(cfg), np.array(r[:7 * k]).reshape(k, 7)


def _filters(lib, n, dtype):
    wl = synth.make_stream_workload(n_frames=3, seq=2, max_features=10)
    fs = [shim_filter(lib, dtype) for _ in range(n)]
    for f in fs:
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        f.augmentState(wl["frames"][0]["state_id"], wl["frames"][0]["time"])
    return fs


def _readings(rng, k):
    r = np.zeros((k, 7))
    r[:, 0:3] = 1e-3 * rng.normal(size=(k, 3))
    r[:, 3:6] = [0.0, 0.0, 9.81] + 1e-2 * rng.normal(size=(k, 3))
    r[:, 6] = rng.uniform(0.004, 0.006, size=k)
    return r


def _expect(res, k):
    assert res == {"nis": float(k), "dx_norm": 0.5, "dof": 9, "applied": 1, "status": 0, "scatter": k + 0.25, "outcome": 0}


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_filter_sends_readings_and_cfg_after_the_queue(stub_view, dtype):
    (f,) = _filters(stub_view, 1, dtype)
    rng = np.random.default_rng(1)
    r = _readings(rng, 12)
    for j in range(3):  # queued readings: handed over before the standstill call
        f.propagate(r[j, 0:3], r[j, 3:6], r[j, 6])
    before, _, _ = _calls(f)
    _expect(f.standstill_update(r, CFG), 12)
    c, cfg, got = _calls(f)
    assert c[0] - before[0] == 1 and c[1] == before[1]
    assert c[2] == 3  # (a fresh engine: the three queued readings only)
    assert cfg == [CFG["noise_scale"], CFG["sigma_v"], CFG["scatter_max"], CFG["chi2_max"]]
    assert np.array_equal(got, r.astype(dtype).astype(np.float64))


BAD_READINGS = [("one reading", lambda r: r[:1]), ("4097 readings", lambda r: np.tile(r, (410, 1))[:4097]),
                ("zero dT", lambda r: np.vstack([r[:3], np.r_[r[3, :6], 0.0]])), ("negative dT", lambda r: np.vstack([r[:3], np.r_[r[3, :6], -1e-3]])),
                ("NaN", lambda r: np.where(np.arange(7 * len(r)).reshape(-1, 7) == 9, np.nan, r)),
                ("inf dT", lambda r: np.vstack([r[:3], np.r_[r[3, :6], np.inf]]))]
BAD_CFG = [dict(CFG, noise_scale=0.99), dict(CFG, noise_scale=np.nan), dict(CFG, sigma_v=0.0), dict(CFG, sigma_v=np.inf),
           dict(CFG, scatter_max=-1.0), dict(CFG, scatter_max=np.nan), dict(CFG, chi2_max=0.0), dict(CFG, chi2_max=np.inf)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_bad_input_is_refused_before_any_call(stub_view, dtype):
    (f,) = _filters(stub_view, 1, dtype)
    r = _readings(np.random.default_rng(2), 10)
    f.propagate(r[0, 0:3], r[0, 3:6], r[0, 6])
    before = _calls(f)[0]
    for what, bad in BAD_READINGS:
        with pytest.raises(RuntimeError, match="standstillUpdate"):
            f.standstill_update(bad(r), CFG)
    for cfg in BAD_CFG:
        with pytest.raises(RuntimeError, match="standstillUpdate"):
            f.standstill_update(r, cfg)
    assert _calls(f)[0] == before
    # the queued reading is still queued: the next good call hands it over
    f.standstill_update(r, CFG)
    after = _calls(f)[0]
    assert after[0] == before[0] + 1 and after[2] == 1


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_makes_one_call_and_leaves_members_without_readings_alone(stub_view, dtype):
    fs = _filters(stub_view, 3, dtype)
    fb = FilterBatch(fs)
    rng = np.random.default_rng(3)
    rs = [_readings(rng, 5), None, _readings(rng, 40)]
    before = [_calls(f)[0] for f in fs]
    res = fb.standstill_update(rs, CFG)
    assert res[1] is None
    _expect(res[0], 5)
    _expect(res[2], 40)
    assert fs[0].lib.msckf_b200_stub_batch_standstill_calls(C.c_void_p(fb.handle())) == 1
    for i, f in enumerate(fs):
        c, _, got = _calls(f)
        assert c[0] == before[i][0]
        assert c[1] - before[i][1] == (0 if rs[i] is None else 1)
        if rs[i] is not None:
            assert np.array_equal(got, rs[i].astype(dtype).astype(np.float64))
    bad = [rs[0], _readings(rng, 1), None]
    with pytest.raises(RuntimeError, match="standstillUpdate"):
        fb.standstill_update(bad, CFG)
    assert fs[0].lib.msckf_b200_stub_batch_standstill_calls(C.c_void_p(fb.handle())) == 1
    fb.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_at_rest_class_forms_send_one_item_and_check_R(stub_view, dtype):
    (f,) = _filters(stub_view, 1, dtype)
    v = np.array([0.1, -0.2, 9.7])
    R = np.array([[2.0, 0.1, 0.0], [0.1, 3.0, 0.2], [0.0, 0.2, 4.0]]) * 1e-4
    for which, model in ((0, capi.AID_GYRO_AT_REST), (1, capi.AID_ACCEL_AT_REST)):
        out = capi.AidResult()
        rc = f.lib.msckf_b200_stub_at_rest_class_call(f.h, C.c_int(which), (C.c_double * 3)(*v), (C.c_double * 9)(*R.ravel()),
                                                      C.c_int(3), C.byref(out))
        assert rc == 0 and out.dof == 3 and out.applied == 1
        rec = (C.c_double * 15)()
        assert f.lib.msckf_b200_stub_standstill_items(C.c_void_p(f.engineHandle()), rec, 1) == 1
        rec = np.array(rec[:])
        assert rec[0] == model and rec[1] == 0 and rec[2] == 0
        assert np.array_equal(rec[3:6], v) and np.array_equal(rec[6:15], R.ravel())
    stacks = _calls(f)[0][3]
    out = capi.AidResult()
    rc = f.lib.msckf_b200_stub_at_rest_class_call(f.h, C.c_int(0), (C.c_double * 3)(*v), (C.c_double * 4)(*R[:2, :2].ravel()),
                                                  C.c_int(2), C.byref(out))
    assert rc == -1 and _calls(f)[0][3] == stacks


def test_python_structs():
    c = capi.standstill_struct({"sigma_v": 0.02, "scatter_max": 3.0, "chi2_max": 25.0})
    assert (c.noise_scale, c.sigma_v, c.scatter_max, c.chi2_max) == (1.0, 0.02, 3.0, 25.0)
    assert C.sizeof(capi.StandstillResult) == C.sizeof(capi.AidResult) + 16
    assert capi.AID_GYRO_AT_REST == 15 and capi.AID_ACCEL_AT_REST == 16
    o = capi.StandstillResult()
    o.stack.nis, o.stack.dof, o.scatter, o.outcome = 4.0, 9, 0.7, 2
    assert o.as_dict() == {"nis": 4.0, "dx_norm": 0.0, "dof": 9, "applied": 0, "status": 0, "scatter": 0.7, "outcome": 2}
