#!/usr/bin/env python
"""scripts/measure_parity.py -- runs every parity case of tests/parity_cases.py on the GPU and writes the measured
numbers as JSON (stdout).  The committed copy, tests/golden/parity_measured.json, is what the GPU tests assert against
(value <= 10 x measurement) and what DESIGN.md section 5 quotes.  Test infrastructure: engine vs CPU oracle.

    python scripts/measure_parity.py [case ...] > tests/golden/parity_measured.json
"""
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests import parity_cases as pc  # noqa: E402


def main():
    names = sys.argv[1:] or list(pc.CASES)
    out = {}
    for name in names:
        t0 = time.time()
        try:
            out[name] = pc.run_case(name)
        except Exception as e:  # keep going: one broken case must not hide the others
            out[name] = {"error": f"{type(e).__name__}: {e}"}
        print(f"{name} ({time.time() - t0:.1f} s): {json.dumps(out[name])}", file=sys.stderr, flush=True)
    print(json.dumps(out, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
