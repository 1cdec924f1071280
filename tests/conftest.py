import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle_lib():
    """The CPU oracle is test infrastructure; build it on demand (g++ only)."""
    so = ROOT / "oracle" / "libmsckf_oracle.so"
    src = [ROOT / "oracle" / n for n in ("oracle_capi.cpp", "msckf_oracle.hpp", "chi2_table.inc")]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in src):
        subprocess.check_call(["make", "-C", str(ROOT / "oracle")])
    return so


@pytest.fixture(scope="session")
def engine_lib():
    so = ROOT / "msckf_mono_b200" / "libmsckf_b200.so"
    if not so.exists():
        pytest.fail("libmsckf_b200.so missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    return so
