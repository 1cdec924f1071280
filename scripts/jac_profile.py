#!/usr/bin/env python
"""scripts/jac_profile.py -- %globaltimer stamps of k_jac's phases for the first track of filter 0 (CTA 0, thread 0) in a
device batch of independent config-B filters (300 x 30 fp32 each), and k_jac's event time.
Usage: python scripts/jac_profile.py [filters ...]   (default: 8; MSCKF_B200_JAC_GROUP pins the threads per track)"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from msckf_mono_b200 import capi, engine_filter, synth  # noqa: E402

PHASES = ["bookkeeping", "X/r", "QR|Y pairs", "Z/Yq, right-hand sides", "gate Cholesky", "outputs"]


def run(nf, nfeat=300, nclones=30, dtype=np.float32, reps=6):
    caps = dict(max_clones=nclones + 8, max_tracks=max(512, nfeat + 16), max_obs=max(512, nfeat + 16) * nclones)
    tmpl, batches, work = [], [], []
    for i in range(nf):
        f = engine_filter(dtype, **caps)
        synth.drive(f, synth.make_window_workload(n_features=nfeat, n_clones=nclones, seq=(i % 16)), marginalize_last=False)
        off, obs, idx = f.packQueued()
        batches.append(capi.TrackBatch(off, obs, idx, dtype))
        tmpl.append((f, capi.Engine(dtype, borrowed=f.engineHandle())))  # (the filter owns the borrowed engine)
        work.append(capi.Engine(dtype, **caps))
    b = capi.Batch(work)
    work[0].set_option(1, 1.0)  # per-kernel events and phase stamps (plain launches on one stream)
    stamps, jac = [], []
    for _ in range(reps):
        for w, (_, t) in zip(work, tmpl):
            w.copy_state_from(t)
        b.stage(capi.MARGINALIZE, batches, threads=4)
        b.launch_timed()
        b.fetch(batches)
        jac.append(dict(b.kernel_times())["k_jac"] * 1e3)
        buf = (C.c_ulonglong * 80)()
        capi.lib().msckf_b200_tail_profile(work[0].h, buf, 80)
        sj = [int(x) for x in list(buf)[40:60] if x]
        stamps.append(np.diff(np.asarray(sj, dtype=np.float64)) / 1e3)
    work[0].set_option(1, 0.0)
    b.close()
    d = np.median(np.stack(stamps[1:]), axis=0)
    return {"filters": nf, "k_jac_us": round(float(np.median(jac[1:])), 1),
            "track0_phase_us": {n: round(float(v), 2) for n, v in zip(PHASES, d)}, "track0_total_us": round(float(d.sum()), 1)}


if __name__ == "__main__":
    for a in (sys.argv[1:] or ["8"]):
        print(json.dumps(run(int(a))), flush=True)
