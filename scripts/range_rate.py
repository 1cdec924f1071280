#!/usr/bin/env python
"""scripts/range_rate.py -- wall time of one stacked ranging update (msckf_b200_aid_stack_update for one filter,
msckf_b200_batch_aid_stack_update for more) against the host path a caller had before it: get_state per filter, the range rows
linearised in numpy (montecarlo.odometry_jacobian), and one caller-linearised aided update (msckf_b200_aid_update /
_batch_aid_update with LINEAR).  fp64 filters at 30 clones (n = 195); the stack is four radio ranges at the IMU, to the anchors
of montecarlo.ANCHORS placed around the filter's position, and one rangefinder distance to a level plane 1.5 m below (5 rows),
the method of scripts/gnss_rate.py.  Host time around each synchronising call, median of --reps after a warm-up, at 1 / 8 / 32
members.  --fde instead times the plain stack against msckf_b200_aid_stack_update_fde (alpha = 0.01, max_exclude = 2) on the
same five items with R = 0.01 m^2, without a fault and with the first range 1 m long (one exclusion round).  --iterations K ...
instead times msckf_b200_aid_stack_update_iter / _batch_aid_stack_update_iter at each max_iter K on the same five items with
R = 0.01 m^2, the ranges measured from 0.3 m beside the estimate, tol 0 (every call makes its K linearisations unless a step is
exactly zero), and reports the mean linearisations made.
Prints one JSON line with the card's name, power limit and max SM clock."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
from msckf_mono_b200 import capi, montecarlo as mc  # noqa: E402
from gnss_rate import host_linear  # noqa: E402
from odometry_rate import gpu_line, median_ms, members  # noqa: E402

LEVER = np.array([0.3, -0.2, 0.5])


def stack_of(e, sigma=1e3, fault=0.0, offset=0.0):
    """the five range items at the current estimate (large R: P barely moves), the first range `fault` m long, the anchor
    ranges measured from `offset` m beside the estimate (along x)"""
    imu, _ = e.state()
    imu = imu.astype(np.float64)
    p, q = imu[0:3], imu[15:19]
    pm = p + np.array([offset, 0.0, 0.0])
    items = [{"model": capi.AID_RANGE, "z": np.r_[mc.range_of(pm, q, LEVER, p + a) + 0.01, p + a, LEVER], "R": np.array([[sigma]])}
             for a in mc.ANCHORS]
    axis = mc.quat_to_rot(q) @ np.array([0.0, 0.0, -1.0])  # straight down in G
    h = mc.antenna_position(p, q, LEVER)[2] - 1.5
    items.append({"model": capi.AID_PLANE_RANGE, "z": np.r_[1.51, h, LEVER, axis], "R": np.array([[sigma]])})
    items[0]["z"][0] += fault
    return items


def fde_calls(args, res):
    fde = {"chi2": capi.fde_thresholds(0.01), "max_exclude": 2}
    for nm in args.members:
        row = {}
        for fault in (0.0, 1.0):
            fs, es = members(nm)
            stacks = [stack_of(e, 0.01, fault) for e in es]
            b = capi.Batch(es) if nm > 1 else None
            call = (lambda **k: b.aid_stack_update(stacks, **k)) if b else (lambda **k: es[0].aid_stack_update(stacks[0], **k))
            key = "one_fault" if fault else "no_fault"
            row[key] = {"plain": median_ms(call, args.reps), "fde": median_ms(lambda: call(fde=fde), args.reps)}
            last = call(fde=fde)
            row[key]["outcome"] = (last[0] if b else last)["outcome"]
            if b:
                b.close()
            for f in fs:
                f.close()
        res["calls_ms"][str(nm)] = row


def iterated_calls(args, res):
    for nm in args.members:
        row = {}
        for K in args.iterations:
            fs, es = members(nm)
            stacks = [stack_of(e, 0.01, offset=0.3) for e in es]
            b = capi.Batch(es) if nm > 1 else None
            call = (lambda: b.aid_stack_update(stacks, max_iter=K, tol=0.0)) if b else \
                (lambda: [es[0].aid_stack_update(stacks[0], max_iter=K, tol=0.0)])
            row[str(K)] = {"ms": median_ms(call, args.reps), "iterations": float(np.mean([o["iterations"] for o in call()]))}
            if b:
                b.close()
            for f in fs:
                f.close()
        res["calls_ms"][str(nm)] = row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--members", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--fde", action="store_true", help="plain stack against fault detection and exclusion")
    ap.add_argument("--iterations", type=int, nargs="*", default=None, help="time the iterated stack at these max_iter")
    args = ap.parse_args()
    res = {"gpu": gpu_line(), "clones": 30, "rows": 5, "reps": args.reps, "calls_ms": {}}
    if args.iterations:
        iterated_calls(args, res)
        print(json.dumps(res), flush=True)
        return
    if args.fde:
        fde_calls(args, res)
        print(json.dumps(res), flush=True)
        return
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
