"""The recording fake of the engine C-ABI is complete: every entry point include/msckf_b200.h declares is defined by the library
the CPU tests of the C view load, so a new entry point without a fake fails here rather than in a test's link step."""
import re
import subprocess

from tests.common import ROOT
from tests.fake_engine import stub_view  # noqa: F401 (the fixture)


def test_fake_defines_every_c_abi_entry_point(stub_view):
    header = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "msckf_b200.h").read_text(), flags=re.S)
    declared = set(re.findall(r"\b(msckf_b200_\w+)\s*\(", header))
    assert len(declared) > 60 and "msckf_b200_create" in declared and "msckf_b200_batch_nees" in declared
    nm = subprocess.run(["nm", "-D", "--defined-only", str(stub_view)], check=True, capture_output=True, text=True).stdout
    defined = {line.split()[-1] for line in nm.splitlines() if line.strip()}
    assert sorted(declared - defined) == []
