"""The recording fake of the engine C-ABI (include/msckf_b200.h) for the CPU tests, and what builds it.

tests/stub/stub_*.cpp are one complete fake without numerics: every msckf_b200_* entry point and every msckf_b200_stub_* test
hook is defined once, and tests/stub/stub.hpp defines its handles.  The session fixture `stub_view` links the fake with every
translation unit of the C view that the product's Makefile links into libmsckf_b200.so (and with the class-form hooks of
tests/stub/class_forms.cpp) into one library; `build_program` links a host program against the fake alone.  Both rebuild
when a fake source, a view source, filter_view.hpp or a header under include/ is newer than what they built.  Also the
decoder of what the fake recorded of the stacked aided calls."""
import ctypes as C
import functools
import re
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

STUB = ROOT / "tests" / "stub"
CSRC = ROOT / "msckf_mono_b200" / "csrc"
FAKE_SOURCES = sorted(STUB.glob("stub_*.cpp"))


def view_sources():
    """the C view's translation units: the host objects of the Makefile's libmsckf_b200.so rule"""
    rule = re.search(r"^\$\(OUT\):(.*)$", (CSRC / "Makefile").read_text(), re.M).group(1)
    return [CSRC / o.replace(".o", ".cpp") for o in rule.split() if o != "engine.o"]


def stale(target, deps=()):
    """target is missing or older than the fake, the C view, or `deps`"""
    deps = [*deps, *STUB.glob("stub*.?pp"), *view_sources(), CSRC / "filter_view.hpp", *(ROOT / "include").rglob("*.h")]
    return not target.exists() or any(d.stat().st_mtime > target.stat().st_mtime for d in deps)


def build_program(exe, sources, deps=(), flags=()):
    """the host program `sources` linked against the fake into exe (rebuilt when stale; `deps`: the headers it includes)"""
    if stale(exe, [*sources, *deps]):
        subprocess.check_call(["g++", "-O1", "-std=c++17", *flags, f"-I{ROOT / 'include'}", *map(str, sources), *map(str, FAKE_SOURCES),
                               "-o", str(exe)])
    return exe


@functools.cache
def _view_library():
    so = STUB / "libmsckf_view_stub.so"
    sources = [*FAKE_SOURCES, STUB / "class_forms.cpp", *view_sources()]
    if stale(so, sources):  # (-z defs: a C-ABI entry point the view calls and the fake lacks fails here, not at load time)
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wl,-z,defs", f"-I{ROOT / 'include'}", f"-I{CSRC}",
                               *map(str, sources), "-o", str(so)])
    return so


@pytest.fixture(scope="session")
def stub_view():
    """the C view of the class shim linked against the fake: a library for msckf_mono_b200.cview"""
    return _view_library()


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
