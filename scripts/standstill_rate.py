#!/usr/bin/env python
"""scripts/standstill_rate.py -- wall time of one standstill update (msckf_b200_standstill_update for one filter,
msckf_b200_batch_standstill_update for more) against the plain 9-row stacked update of the same three items
(msckf_b200_aid_stack_update / _batch_aid_stack_update with VELOCITY, GYRO_AT_REST and ACCEL_AT_REST, z and R formed in numpy
from the same readings): the difference is the host's statistics of the window.  fp64 filters at 30 clones (n = 195), --k
readings at rest per window (default 10: one 50 ms frame interval at 200 Hz) at each filter's estimate plus white noise of the
filter's Q_imu.  Host time around each synchronising call, median of --reps after a warm-up, at 1 / 8 / 32 members, the method
of scripts/odometry_rate.py.  Prints one JSON line with the card's name, power limit and max SM clock."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
from msckf_mono_b200 import capi, montecarlo as mc, synth  # noqa: E402
from odometry_rate import gpu_line, median_ms, members  # noqa: E402

CFG = {"noise_scale": 1.0, "sigma_v": 0.01, "scatter_max": 4.0, "chi2_max": 1e9}


def window(e, k, Q, rng):
    """k readings at rest at e's estimate: omega = b_g + n_g, a = b_a - C(q_IG) g + n_a, n ~ N(0, Q / dT), dT = 5 ms"""
    imu, _ = e.state()
    imu = imu.astype(np.float64)
    h = np.r_[imu[6:9], imu[9:12] - mc.quat_to_rot(imu[15:19]) @ imu[12:15]]
    r = np.zeros((k, 7))
    r[:, 6] = 0.005
    r[:, 0:3] = h[0:3] + rng.normal(size=(k, 3)) * np.sqrt(np.diag(Q)[0:3] / 0.005)
    r[:, 3:6] = h[3:6] + rng.normal(size=(k, 3)) * np.sqrt(np.diag(Q)[6:9] / 0.005)
    return r


def items_of(r, Q, cfg):
    """the three items msckf_b200_standstill_update forms from readings r (dT-weighted means, R = s^2 R0 / T)"""
    T = float(np.sum(r[:, 6]))
    w, a = (r[:, 6] @ r[:, 0:3]) / T, (r[:, 6] @ r[:, 3:6]) / T
    s2 = cfg["noise_scale"] ** 2
    return [{"model": capi.AID_VELOCITY, "z": np.zeros(3), "R": cfg["sigma_v"] ** 2 * np.eye(3)},
            {"model": capi.AID_GYRO_AT_REST, "z": w, "R": s2 * Q[0:3, 0:3] / T},
            {"model": capi.AID_ACCEL_AT_REST, "z": a, "R": s2 * Q[6:9, 6:9] / T}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--members", type=int, nargs="+", default=[1, 8, 32])
    args = ap.parse_args()
    Q = np.asarray(synth.make_window_workload(n_features=4, n_clones=2, seq=3)["noise"]["Q_imu"], dtype=np.float64)
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_line(), "clones": 30, "rows": 9, "readings": args.k, "reps": args.reps, "calls_ms": {}}
    for nm in args.members:
        fs, es = members(nm)
        rs = [window(e, args.k, Q, rng) for e in es]
        its = [items_of(r, Q, CFG) for r in rs]
        if nm == 1:
            standstill = lambda: es[0].standstill_update(rs[0], CFG)  # noqa: E731
            stack = lambda: es[0].aid_stack_update(its[0], chi2_max=CFG["chi2_max"])  # noqa: E731
        else:
            b = capi.Batch(es)
            standstill = lambda: b.standstill_update(rs, CFG)  # noqa: E731
            stack = lambda: b.aid_stack_update(its, chi2_max=CFG["chi2_max"])  # noqa: E731
        res["calls_ms"][str(nm)] = {"standstill": median_ms(standstill, args.reps), "aid_stack_9_rows": median_ms(stack, args.reps)}
        if nm > 1:
            b.close()
        for f in fs:
            f.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
