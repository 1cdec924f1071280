#!/usr/bin/env python
"""scripts/gnss_rate.py -- wall time of one stacked GNSS update (msckf_b200_aid_stack_update for one filter,
msckf_b200_batch_aid_stack_update for more) against the host path a caller had before it: get_state per filter, the antenna and
heading rows linearised in numpy (montecarlo.odometry_jacobian), and one caller-linearised aided update (msckf_b200_aid_update /
_batch_aid_update with LINEAR).  fp64 filters at 30 clones (n = 195); the stack is an antenna position at the IMU (3 rows), a
heading (1 row) and a delayed antenna position at the clone four images back (3 rows).  Host time around each synchronising
call, median of --reps after a warm-up, at 1 / 8 / 32 members.  Prints one JSON line with the card's name, power limit and max
SM clock."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
from msckf_mono_b200 import capi, montecarlo as mc  # noqa: E402
from odometry_rate import gpu_line, median_ms, members  # noqa: E402

LEVER = np.array([0.3, -0.2, 0.5])
AXIS = np.array([1.0, 0.0, 0.0])


def stack_of(e, sigma=1e3):
    """the three GNSS items at the current estimate (large R: P barely moves)"""
    imu, poses = e.state()
    imu, poses = imu.astype(np.float64), poses.astype(np.float64)
    k = len(poses) - 5
    R3 = sigma * np.eye(3)
    return [{"model": capi.AID_ANTENNA_POSITION, "a": 0b111, "z": np.r_[mc.antenna_position(imu[0:3], imu[15:19], LEVER) + 0.01, LEVER], "R": R3},
            {"model": capi.AID_HEADING, "z": np.r_[mc.heading_of(imu[15:19], AXIS) + 0.01, AXIS], "R": np.array([[sigma]])},
            {"model": capi.AID_CLONE_ANTENNA_POSITION, "a": k, "b": 0b111,
             "z": np.r_[mc.antenna_position(poses[k, 0:3], poses[k, 3:7], LEVER) + 0.01, LEVER], "R": R3}]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--members", type=int, nargs="+", default=[1, 8, 32])
    args = ap.parse_args()
    res = {"gpu": gpu_line(), "clones": 30, "rows": 7, "reps": args.reps, "calls_ms": {}}
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
