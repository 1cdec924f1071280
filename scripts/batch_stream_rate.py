#!/usr/bin/env python
"""scripts/batch_stream_rate.py -- n filters streaming bench.py's `stream` workload (E-sim, float32, 200 frames, 10 IMU
readings per frame, window 20; seed 8 + i for filter i) in lockstep on one GPU, two ways:

  (a) per-filter calls, with MSCKFBatch::marginalize() as the only batched step;
  (b) the fully batched step: MSCKFBatch::propagate / augmentState / marginalize / pruneEmptyStates / refreshState.

Per n: filter-frames/s, host wall time per frame split by call (the asynchronous calls' device work is paid by the next call
that synchronises), kernel launches per frame, and whether the final covariances, IMU states and clone poses of (a) and (b)
are equal bit for bit.  Warm-up run of each form, then `--rounds` rounds alternating (a) and (b); the median is reported.
Launches: the batch's counter counts its batched launches; an engine's counter counts its own launches plus every batched
launch it took part in, so (a) = batch + sum(engines) - n * batch and (b) = batch."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from msckf_mono_b200 import capi, engine_filter, synth  # noqa: E402
from msckf_mono_b200.cview import FilterBatch  # noqa: E402

DTYPE = np.float32


def workloads(n):
    wls = []
    for i in range(n):
        wl = synth.make_stream_workload(n_frames=200, seq=8 + i, max_features=60, max_track_length=20, max_cam_states=20)
        wl["noise"] = synth.euroc_noise(tuned=True)
        wls.append(wl)
    return wls


def run(wls, batched):
    fs = [engine_filter(DTYPE) for _ in wls]
    for f, wl in zip(fs, wls):
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    fb = FilterBatch(fs)
    engs = [capi.Engine(DTYPE, borrowed=f.engineHandle()) for f in fs]
    acc = {}

    def timed(name, fn, *a):
        t0 = time.perf_counter()
        fn(*a)
        acc[name] = acc.get(name, 0.0) + time.perf_counter() - t0

    b0 = int(capi.lib().msckf_b200_batch_launch_count(C.c_void_p(fb.handle())))
    e0 = sum(e.launch_count() for e in engs)
    n_frames = len(wls[0]["frames"])
    t0 = time.perf_counter()
    for k in range(n_frames):
        frs = [wl["frames"][k] for wl in wls]
        if batched:
            for i, fr in enumerate(frs):
                for (w, a, dT) in fr["imu"]:
                    timed("propagate", fb.propagate, i, w, a, dT)
            timed("augmentState", fb.augmentState, [fr["state_id"] for fr in frs], [fr["time"] for fr in frs])
        else:
            for f, fr in zip(fs, frs):
                for (w, a, dT) in fr["imu"]:
                    timed("propagate", f.propagate, w, a, dT)
                timed("augmentState", f.augmentState, fr["state_id"], fr["time"])
        for f, fr in zip(fs, frs):
            timed("update", f.update, *fr["update"])
            timed("addFeatures", f.addFeatures, *fr["add"])
        timed("marginalize", fb.marginalize)
        if batched:
            timed("pruneEmptyStates", fb.pruneEmptyStates)
            timed("refreshState", fb.refreshState)
        else:
            for f in fs:
                timed("pruneEmptyStates", f.pruneEmptyStates)
        for f in fs:
            timed("getImuState", f.getImuState)
    dt = time.perf_counter() - t0
    nb = int(capi.lib().msckf_b200_batch_launch_count(C.c_void_p(fb.handle()))) - b0
    ne = sum(e.launch_count() for e in engs) - e0
    launches = nb if batched else nb + ne - len(fs) * nb
    fb.close()
    final = [(f.getCovariance(), np.concatenate([v for v in f.getImuState().values()]),
              np.hstack([f.getCamStates()["p_C_G"], f.getCamStates()["q_CG"]])) for f in fs]
    return {"s": dt, "us_per_frame": {k: 1e6 * v / n_frames for k, v in acc.items()}, "launches_per_frame": launches / n_frames}, final


def gpu_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    capi.lib().msckf_b200_batch_launch_count.restype = C.c_longlong
    hw = gpu_line()
    print("GPU:", hw, flush=True)
    results = []
    for n in args.n:
        wls = workloads(n)
        run(wls, False)
        run(wls, True)  # warm-up of both forms
        rec = {"a": [], "b": []}
        equal = True
        for _ in range(args.rounds):
            ra, fa = run(wls, False)
            rb, fbin = run(wls, True)
            rec["a"].append(ra); rec["b"].append(rb)
            equal &= all(np.array_equal(x, y) for pa, pb in zip(fa, fbin) for x, y in zip(pa, pb))
        row = {"n": n, "gpu": hw, "bit_identical": bool(equal)}
        for key in ("a", "b"):
            rs = sorted(rec[key], key=lambda r: r["s"])
            med = rs[len(rs) // 2]
            row[key] = {"filter_frames_per_s": n * 200 / med["s"], "all_rounds_s": [r["s"] for r in rec[key]],
                        "us_per_frame_by_call": {k: round(v, 1) for k, v in med["us_per_frame"].items()},
                        "launches_per_frame": med["launches_per_frame"]}
        row["speedup_b_over_a"] = row["b"]["filter_frames_per_s"] / row["a"]["filter_frames_per_s"]
        print(json.dumps(row), flush=True)
        results.append(row)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
