"""msckf_mono_b200 -- H100-native MSCKF measurement-update engine behind the msckf_mono::MSCKF<_S> surface.

The product is native: hand-written sm_90a kernels + a C-ABI (include/msckf_b200.h) + the drop-in C++ class
(include/msckf_mono/msckf.h), built in-tree as msckf_mono_b200/libmsckf_b200.so.  This Python package only
holds the ctypes view used by the tests and bench.py, and the synthetic workload generator.
There is no CPU fallback: if the library or a CUDA device is missing, construction fails loudly.
"""
from pathlib import Path

import numpy as np

_ROOT = Path(__file__).resolve().parent
LIB_PATH = _ROOT / "libmsckf_b200.so"


def lib_path() -> Path:
    if not LIB_PATH.exists():
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    return LIB_PATH


def engine_filter(dtype=np.float32, device=0, max_clones=0, max_tracks=0, max_obs=0):
    """msckf_mono::MSCKF<float|double> on the H100 engine, through the C view (include/msckf_mono_c.h)."""
    import ctypes as C
    from .cview import CFilter
    f = CFilter(lib_path(), "msckf_mono_", dtype)
    rc = f.lib.msckf_mono_set_engine_options(f.h, C.c_int(device), C.c_int(max_clones), C.c_int(max_tracks), C.c_int(max_obs))
    if rc != 0:
        raise RuntimeError("msckf_mono_set_engine_options failed")
    return f
