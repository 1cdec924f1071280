#!/usr/bin/env python
"""scripts/odometry_rate.py -- wall time of one stacked odometry update (msckf_b200_aid_stack_update for one filter,
msckf_b200_batch_aid_stack_update for more) against the host path a caller had before it: get_state per filter, the body-velocity
and relative-pose rows linearised in numpy (montecarlo.odometry_jacobian), and one caller-linearised aided update
(msckf_b200_aid_update / _batch_aid_update with LINEAR).  fp64 filters at 30 clones (n = 195); the stack is a body velocity
(3 rows) and the relative pose of the two newest clones (6 rows).  Host time around each synchronising call, median of --reps
after a warm-up, at 1 / 8 / 32 members.  Prints one JSON line with the card's name, power limit and max SM clock."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from msckf_mono_b200 import capi, engine_filter, montecarlo as mc, synth  # noqa: E402


def gpu_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def members(n_members, M=30):
    wl = synth.make_window_workload(n_features=4, n_clones=2, seq=3)
    fs, es = [], []
    for _ in range(n_members):
        f = engine_filter(np.float64, max_clones=M + 8)
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        e = capi.Engine(np.float64, borrowed=f.engineHandle())
        for _ in range(M):
            r = np.zeros((2, 7)); r[:, 0] = 0.2; r[:, 3:6] = [0.3, 0, 9.81]; r[:, 6] = 0.005
            e.propagate_n(r)
            e.augment()
        fs.append(f); es.append(e)
    return fs, es


def stack_of(e, sigma=1e3):
    """a body velocity and the relative pose of the two newest clones at the current estimate (large R: P barely moves)"""
    imu, poses = e.state()
    imu, poses = imu.astype(np.float64), poses.astype(np.float64)
    M = len(poses)
    p, q = mc.relative_pose(poses[M - 2], poses[M - 1])
    return [{"model": capi.AID_BODY_VELOCITY, "a": 0b111, "z": mc.body_velocity(imu) + 0.01, "R": sigma * np.eye(3)},
            {"model": capi.AID_RELATIVE_POSE, "a": M - 2, "b": M - 1, "z": np.r_[p + 0.01, q], "R": sigma * np.eye(6)}]


def host_linear(e, items):
    """the host path of one filter: fetch the state, linearise the stack in numpy; the LINEAR spec"""
    imu, poses = e.state()
    imu, poses = imu.astype(np.float64), poses.astype(np.float64)
    n = 15 + 6 * len(poses)
    H = np.vstack([mc.odometry_jacobian(it, imu, poses, n) for it in items])
    r = np.concatenate([mc.odometry_residual(it, imu, poses) for it in items])
    R = np.zeros((len(r), len(r)))
    o = 0
    for it in items:
        k = len(it["R"]); R[o:o + k, o:o + k] = it["R"]; o += k
    return {"model": capi.AID_LINEAR, "z": r, "R": R, "H": H}


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--members", type=int, nargs="+", default=[1, 8, 32])
    args = ap.parse_args()
    res = {"gpu": gpu_line(), "clones": 30, "rows": 9, "reps": args.reps, "calls_ms": {}}
    for nm in args.members:
        fs, es = members(nm)
        stacks = [stack_of(e) for e in es]
        b = capi.Batch(es) if nm > 1 else None
        if b:
            device = lambda: b.aid_stack_update(stacks)  # noqa: E731
            host = lambda: b.aid_update([host_linear(e, s) for e, s in zip(es, stacks)])  # noqa: E731
        else:
            device = lambda: es[0].aid_stack_update(stacks[0])  # noqa: E731
            host = lambda: es[0].aid_update(**host_linear(es[0], stacks[0]))  # noqa: E731
        res["calls_ms"][str(nm)] = {"device_stack": median_ms(device, args.reps), "host_get_state_numpy_linear": median_ms(host, args.reps)}
        if b:
            b.close()
        for f in fs:
            f.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
