"""The C view linked against the recording fake of the C-ABI (tests/stub/stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp)
plus tests/stub/stub_aid_stack.cpp, the fake of the stacked aided-update calls with and without FDE: the module fixture that
builds that one library for the CPU tests of odometry, GNSS, ranges and FDE, and the decoder of what the fake recorded."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

CSRC = ROOT / "msckf_mono_b200" / "csrc"
SOURCES = [ROOT / "tests" / "stub" / n for n in ("stub_engine.cpp", "stub_batch_state.cpp", "stub_aid.cpp", "stub_aid_stack.cpp")]
SOURCES += [CSRC / n for n in ("filter_capi.cpp", "batch_capi.cpp", "aid_capi.cpp", "aid_stack_capi.cpp", "fde_capi.cpp")]
HEADERS = [CSRC / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
           ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]


@pytest.fixture(scope="module")
def stub_view():
    so = ROOT / "tests" / "stub" / "libmsckf_aid_stack_view_stub.so"
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in SOURCES + HEADERS):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", f"-I{CSRC}", *map(str, SOURCES),
                               "-o", str(so)])
    return so


def recorded(f):
    """([single calls, batched calls] naming f, the IMU readings handed over before its last stacked call, that call's fde as
    (chi2 [32], max_exclude) or None without FDE, its items as dicts model, a, b, z, R)"""
    out, fde, rec = (C.c_longlong * 3)(), (C.c_double * 33)(), (C.c_double * (20 * 8))()
    n = f.lib.msckf_b200_stub_aid_stack_calls(C.c_void_p(f.engineHandle()), out, fde, rec, 8)
    items = []
    for k in range(n):
        r = np.array(rec[20 * k:20 * k + 20])
        z, R = r[3:11], r[11:20]
        items.append({"model": int(r[0]), "a": int(r[1]), "b": int(r[2]), "z": z[np.isfinite(z)], "R": R[np.isfinite(R)]})
    return [out[0], out[1]], out[2], (list(fde[:32]), int(fde[32])) if np.isfinite(fde[32]) else None, items


def batch_calls(fb):
    """the batched stacked calls made on FilterBatch fb"""
    return fb.lib.msckf_b200_stub_batch_aid_stack_calls(C.c_void_p(fb.handle()))
