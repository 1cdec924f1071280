#!/usr/bin/env python
"""scripts/mc_consistency.py -- Monte-Carlo consistency of the filter on the synthetic stream (msckf_mono_b200/montecarlo.py):
`--trials` trials of the noise model the filter is given, run as one fully batched MSCKFBatch stream per process, NEES on the
device after every frame's prune.  Prints one JSON summary: per component (orientation, position, IMU pose, IMU state, whole
state) the run's mean ANEES, the fraction of frames inside the two-sided 95 % chi^2 bounds and the position RMSE.

Under torchrun the trials are sharded with shard.sequences_of_rank; the per-trial records (a few KB) are merged with
shard.gather_summaries -- NCCL carries nothing else.

With --position-fix-every K, every K frames each trial also fuses a noisy position fix (standard deviation
--position-fix-sigma, metres) after the prune, and the summary adds the fixes' ANIS against its 95 % chi^2 bounds.

With --map-every K, every K frames each trial also observes the map (every --map-stride-th landmark of the truth stream) from
its newest clone and fuses the observations as mapped landmarks (after the prune and after a position fix), and the summary adds
the map updates' ANIS against its 95 % chi^2 bounds and the fraction of observations gated out.  --map-start F observes the map
only from frame F on (relocalisation after drift), --map-iterations K iterates each map update (at most K linearisations), and
the summary then adds the first map update: the position RMSE before and after it, its ANIS and the IMU-state ANEES after it.
--map-sigma S gives each trial a map with N(0, S^2 I) errors per landmark, --map-uncertain fuses it with Sigma = S^2 I (map
error marginalised per landmark) instead of as exact, and --map-clones K observes the map from the K newest clones.

With --odometry-every K, every K frames each trial also fuses one stacked odometry update (the truth body velocity, and the
truth relative pose of its two newest clones, each plus noise of --odometry-sigma-v m/s and --odometry-sigma-rel m / rad;
--nhc keeps only the body velocity's y and z rows), and the summary adds the stacks' ANIS against its 95 % chi^2 bounds.

With --gnss-every K, every K frames each trial also fuses the truth GNSS antenna position (lever arm --gnss-lever X Y Z in the
IMU frame) plus noise of --gnss-sigma m as ANTENNA_POSITION; --heading-every K adds the truth heading of the IMU's x axis plus
noise of --heading-sigma rad.  --gnss-delay D fuses the epoch of frame f - D at frame f, at that epoch's clone;
--gnss-as-position fuses the antenna position as a plain POSITION fix (the lever-arm bias).  The summary adds the GNSS stacks'
ANIS against its 95 % chi^2 bounds.

With --range-every K, every K frames each trial also fuses the truth ranges from an antenna at --range-lever X Y Z (IMU frame) to
the four surveyed anchors of montecarlo.ANCHORS plus noise of --range-sigma m as RANGE; --plane-every K adds the truth distance
along --plane-axis X Y Z from --plane-lever X Y Z (both in the IMU frame) to the level plane z = --plane-height plus noise of
--plane-sigma m as PLANE_RANGE; a frame's ranges and plane range go in one stacked update.  --range-delay D fuses the epoch of
frame f - D at frame f, at that epoch's clone.  The summary adds the ranging stacks' ANIS against its 95 % chi^2 bounds.

--range-outlier-rate P --range-outlier-bias B makes each anchor range B m long (NLOS) with probability P; --gnss-outlier-rate P
--gnss-outlier-jump D moves each antenna fix D m horizontally in a random direction with probability P.  --fde-alpha A > 0 sends
the GNSS and ranging stacks through fault detection and exclusion (thresholds: the chi^2 quantiles 1 - A) with at most
--fde-max-exclude K items excluded (K = 0: the stack gate only); A = 0 fuses them ungated.  The GNSS and ranging summaries add
the injected faults, faults excluded, clean items excluded, faults missed and stacks rejected; their ANIS is over the stacks
applied.

--range-start F / --gnss-start F fuse no ranging / GNSS epoch before frame F (the first stack after an outage, when the filter has
drifted), and --aid-iterations K iterates the GNSS, ranging and odometry stacks (at most K linearisations, converged at a step
<= --aid-tol); the summary then adds the first ranging / GNSS stack: the position RMSE before and after it, its ANIS, the
IMU-state ANEES after it, the mean linearisations and the share converged.

With --stop-every F --stop-frames K --stop-ramp R the trajectory stops for K frames every F frames, entered and left through
quintic ramps of R frames (synth.StopProfile), and the summary adds the mean growth of the position error over a stop.
--standstill tests every frame interval's IMU readings for rest (msckf_b200_standstill_update with --standstill-noise-scale,
--standstill-sigma-v, --standstill-scatter-max and --standstill-chi2) and skips the vision work of the frames found at rest; the
summary adds the fraction of frames detected per class (stationary: at rest all through the interval; ramp; cruise) and the
applied stacks' ANIS against its 9-dof run bounds.

It also times the batched NEES call (msckf_b200_batch_nees) against the host path (get_covariance + get_state per filter and
a numpy Cholesky solve) for 8 and 32 config-B members (30 clones: n = 195), and reads the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from msckf_mono_b200 import capi, montecarlo as mc, shard, synth  # noqa: E402

FAULTS = ("injected", "faults_excluded", "clean_excluded", "faults_missed", "stacks_rejected")


def gpu_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def host_nees(e, truth_imu, truth_poses):
    """the host path: copy P and the state back, error state and Cholesky solve in numpy"""
    P = e.covariance().astype(np.float64)
    imu, poses = e.state()
    est = {"imu": np.concatenate([imu[0:15], imu[15:19]]).astype(np.float64), "poses": poses.astype(np.float64)}
    err = mc.error_state({"imu": truth_imu, "poses": truth_poses}, est)
    L = np.linalg.cholesky(P)
    y = np.linalg.solve(L, err)  # (a full-state solve: the host path's cost, not its block bookkeeping)
    return float(y @ y)


def time_nees(n_members, reps=20):
    wl = synth.make_window_workload(n_features=4, n_clones=2, seq=3)
    from msckf_mono_b200 import engine_filter
    rng = np.random.default_rng(5)
    fs, es, truth = [], [], []
    for i in range(n_members):
        f = engine_filter(np.float64, max_clones=38)
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        e = capi.Engine(np.float64, borrowed=f.engineHandle())
        for _ in range(30):
            r = np.zeros((2, 7)); r[:, 3:6] = [0, 0, 9.81]; r[:, 6] = 0.005
            e.propagate_n(r)
            e.augment()
        n = 15 + 6 * 30
        A = rng.normal(size=(n, n))
        e.set_covariance(A @ A.T / n + np.eye(n))
        imu, poses = e.state()
        t_imu = np.concatenate([imu[0:15], imu[15:19]]) + 1e-3
        t_imu[15:19] /= np.linalg.norm(t_imu[15:19])
        fs.append(f); es.append(e); truth.append((t_imu, poses.astype(np.float64) + 1e-3))
    b = capi.Batch(es)
    out = {}
    for name, fn in (("device_batched_nees_ms", lambda: b.nees([t[0] for t in truth], [t[1] for t in truth])),
                     ("host_covariance_numpy_ms", lambda: [host_nees(e, *t) for e, t in zip(es, truth)])):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            ts.append(1e3 * (time.perf_counter() - t0))
        out[name] = float(np.median(ts))
    b.close()
    for f in fs:
        f.close()
    return out


def time_aid(n_members, reps=20):
    """wall time of one aided call (a position fix) on n_members fp64 filters at 30 clones: msckf_b200_aid_update for one
    filter, msckf_b200_batch_aid_update for more"""
    wl = synth.make_window_workload(n_features=4, n_clones=2, seq=3)
    from msckf_mono_b200 import engine_filter
    fs, es = [], []
    for i in range(n_members):
        f = engine_filter(np.float64, max_clones=38)
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        e = capi.Engine(np.float64, borrowed=f.engineHandle())
        for _ in range(30):
            r = np.zeros((2, 7)); r[:, 3:6] = [0, 0, 9.81]; r[:, 6] = 0.005
            e.propagate_n(r)
            e.augment()
        fs.append(f); es.append(e)
    specs = [{"model": capi.AID_POSITION, "z": e.state()[0][0:3] + 0.01, "R": 1e6 * np.eye(3)} for e in es]  # (barely moves P)
    b = capi.Batch(es) if n_members > 1 else None
    fn = (lambda: b.aid_update(specs)) if b else (lambda: es[0].aid_update(**specs[0]))
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    if b:
        b.close()
    for f in fs:
        f.close()
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=32)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--dtype", choices=("f32", "f64"), default="f64")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--seq", type=int, default=8)
    ap.add_argument("--position-fix-every", type=int, default=0)
    ap.add_argument("--position-fix-sigma", type=float, default=0.1)
    ap.add_argument("--map-every", type=int, default=0)
    ap.add_argument("--map-stride", type=int, default=20)
    ap.add_argument("--map-start", type=int, default=0)
    ap.add_argument("--map-iterations", type=int, default=1)
    ap.add_argument("--map-sigma", type=float, default=0.0, help="each trial's map = the truth map + N(0, s^2 I) per landmark")
    ap.add_argument("--map-uncertain", action="store_true", help="fuse the map with Sigma = s^2 I (else it is taken as exact)")
    ap.add_argument("--map-clones", type=int, default=1, help="observe the map from the K newest clones (K <= --map-every)")
    ap.add_argument("--map-chi2", type=float, default=0.0, help="> 0: gate each map observation on its own at this chi^2")
    ap.add_argument("--map-outlier-rate", type=float, default=0.0, help="each map observation a wrong match with this probability")
    ap.add_argument("--map-consensus", type=int, default=0, help="> 0: select map inliers by a consensus of this many hypotheses")
    ap.add_argument("--map-consensus-thresh", type=float, default=13.8)
    ap.add_argument("--map-min-inliers", type=int, default=6)
    ap.add_argument("--odometry-every", type=int, default=0)
    ap.add_argument("--odometry-sigma-v", type=float, default=0.05)
    ap.add_argument("--odometry-sigma-rel", type=float, default=0.01)
    ap.add_argument("--nhc", action="store_true")
    ap.add_argument("--gnss-every", type=int, default=0)
    ap.add_argument("--gnss-sigma", type=float, default=0.1)
    ap.add_argument("--gnss-lever", type=float, nargs=3, default=[0.0, 0.0, 0.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--gnss-delay", type=int, default=0, help="fuse the epoch of frame f - d at its clone (frames)")
    ap.add_argument("--gnss-as-position", action="store_true", help="fuse the antenna position as a plain POSITION fix")
    ap.add_argument("--heading-every", type=int, default=0)
    ap.add_argument("--heading-sigma", type=float, default=0.01)
    ap.add_argument("--range-every", type=int, default=0)
    ap.add_argument("--range-sigma", type=float, default=0.1)
    ap.add_argument("--range-lever", type=float, nargs=3, default=[0.0, 0.0, 0.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--range-delay", type=int, default=0, help="fuse the ranges of frame f - d at its clone (frames)")
    ap.add_argument("--plane-every", type=int, default=0)
    ap.add_argument("--plane-sigma", type=float, default=0.02)
    ap.add_argument("--plane-height", type=float, default=mc.PLANE_HEIGHT)
    ap.add_argument("--plane-axis", type=float, nargs=3, default=list(mc.PLANE_AXIS), metavar=("X", "Y", "Z"))
    ap.add_argument("--plane-lever", type=float, nargs=3, default=[0.0, 0.0, 0.0], metavar=("X", "Y", "Z"))
    ap.add_argument("--range-outlier-rate", type=float, default=0.0)
    ap.add_argument("--range-outlier-bias", type=float, default=1.0)
    ap.add_argument("--gnss-outlier-rate", type=float, default=0.0)
    ap.add_argument("--gnss-outlier-jump", type=float, default=5.0)
    ap.add_argument("--fde-alpha", type=float, default=0.0, help="> 0: fault detection and exclusion in the GNSS and ranging stacks")
    ap.add_argument("--fde-max-exclude", type=int, default=2)
    ap.add_argument("--range-start", type=int, default=0, help="fuse no ranging epoch before this frame")
    ap.add_argument("--gnss-start", type=int, default=0, help="fuse no GNSS epoch before this frame")
    ap.add_argument("--aid-iterations", type=int, default=1, help="iterate the GNSS, ranging and odometry stacks (linearisations)")
    ap.add_argument("--aid-tol", type=float, default=1e-10)
    ap.add_argument("--stop-every", type=int, default=0, help="> 0: the trajectory stops every F frames")
    ap.add_argument("--stop-frames", type=int, default=40)
    ap.add_argument("--stop-ramp", type=int, default=5)
    ap.add_argument("--standstill", action="store_true", help="detect standstills and fuse the zero-motion update")
    ap.add_argument("--standstill-noise-scale", type=float, default=1.0)
    ap.add_argument("--standstill-sigma-v", type=float, default=0.01)
    ap.add_argument("--standstill-scatter-max", type=float, default=2.0)
    ap.add_argument("--standstill-chi2", type=float, default=27.9, help="the 9-row stack's gate (27.9: chi^2_9 at 0.999)")
    ap.add_argument("--no-timing", action="store_true")
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    dtype = np.float32 if args.dtype == "f32" else np.float64
    stop = {"every": args.stop_every, "frames": args.stop_frames, "ramp": args.stop_ramp} if args.stop_every > 0 else None
    standstill = {"noise_scale": args.standstill_noise_scale, "sigma_v": args.standstill_sigma_v,
                  "scatter_max": args.standstill_scatter_max, "chi2_max": args.standstill_chi2} if args.standstill else None
    truth = mc.make_truth(n_frames=args.frames, seq=args.seq, stop=stop)
    t0 = time.perf_counter()
    records, _ = mc.run(shard.sequences_of_rank(args.trials, rank, world), truth, dtype=dtype, seed=args.seed,
                        fix_every=args.position_fix_every, fix_sigma=args.position_fix_sigma, map_every=args.map_every,
                        map_stride=args.map_stride, odo_every=args.odometry_every, odo_sigma_v=args.odometry_sigma_v,
                        odo_sigma_rel=args.odometry_sigma_rel, nhc=args.nhc, map_start=args.map_start,
                        map_iterations=args.map_iterations, map_sigma=args.map_sigma, map_uncertain=args.map_uncertain,
                        map_clones=args.map_clones, gnss_every=args.gnss_every, gnss_sigma=args.gnss_sigma,
                        gnss_lever=args.gnss_lever, gnss_delay=args.gnss_delay, gnss_as_position=args.gnss_as_position,
                        heading_every=args.heading_every, heading_sigma=args.heading_sigma, range_every=args.range_every,
                        range_sigma=args.range_sigma, range_lever=args.range_lever, range_delay=args.range_delay,
                        plane_every=args.plane_every, plane_sigma=args.plane_sigma, plane_height=args.plane_height,
                        plane_axis=args.plane_axis, plane_lever=args.plane_lever, range_outlier_rate=args.range_outlier_rate,
                        range_outlier_bias=args.range_outlier_bias, gnss_outlier_rate=args.gnss_outlier_rate,
                        gnss_outlier_jump=args.gnss_outlier_jump, fde_alpha=args.fde_alpha, fde_max_exclude=args.fde_max_exclude,
                        range_start=args.range_start, gnss_start=args.gnss_start, aid_iterations=args.aid_iterations,
                        aid_tol=args.aid_tol, map_chi2=args.map_chi2, map_outlier_rate=args.map_outlier_rate,
                        map_consensus=args.map_consensus, map_consensus_thresh=args.map_consensus_thresh,
                        map_min_inliers=args.map_min_inliers, standstill=standstill)
    wall = time.perf_counter() - t0
    merged = shard.gather_summaries(records)
    s = mc.summarize(merged)
    res = {"gpu": gpu_line(), "trials": args.trials, "frames": args.frames, "dtype": args.dtype, "seq": args.seq, "seed": args.seed,
           "world": world, "wall_s_rank0": wall, "pos_rmse_run_m": s["pos_rmse_run"],
           "components": {c: {k: v[k] for k in ("mean_anees", "mean_dof", "frames_inside", "frames_finite")} for c, v in s["components"].items()}}
    if "fixes" in s:
        res["position_fixes"] = {"every": args.position_fix_every, "sigma_m": args.position_fix_sigma,
                                 **{k: s["fixes"][k] for k in ("mean_anis", "lower", "upper", "fixes_inside", "dof")}}
    if "map" in s:
        res["map"] = {"every": args.map_every, "stride": args.map_stride,
                      **{k: s["map"][k] for k in ("mean_anis", "mean_dof", "run_bounds", "updates_inside", "applied", "observations", "gated")}}
        res["map"].update(sigma_m=args.map_sigma, uncertain=args.map_uncertain, clones=args.map_clones)
        res["map"].update(chi2=args.map_chi2)
        if args.map_outlier_rate > 0 or args.map_consensus > 0:
            tot = {k: sum(sum(r["map"][k]) for r in merged.values()) for k in ("wrong", "wrong_excluded", "right", "right_kept")}
            st = [x for r in merged.values() for x in r["map"]["cons_status"]]
            res["map"].update(outlier_rate=args.map_outlier_rate, consensus=args.map_consensus,
                              consensus_thresh=args.map_consensus_thresh, min_inliers=args.map_min_inliers, **tot,
                              wrong_excluded_share=tot["wrong_excluded"] / max(tot["wrong"], 1),
                              right_kept_share=tot["right_kept"] / max(tot["right"], 1),
                              consensus_status={str(v): st.count(v) for v in sorted(set(st))})
        if args.map_start or args.map_iterations != 1:
            res["map"].update(start=args.map_start, iterations=args.map_iterations, first_update=s["map_first"])
    if "odometry" in s:
        res["odometry"] = {"every": args.odometry_every, "sigma_v": args.odometry_sigma_v, "sigma_rel": args.odometry_sigma_rel,
                           "nhc": args.nhc, **{k: s["odometry"][k] for k in ("mean_anis", "mean_dof", "run_bounds", "updates_inside", "applied")}}
    if "gnss" in s:
        res["gnss"] = {"every": args.gnss_every, "sigma_m": args.gnss_sigma, "lever_m": args.gnss_lever, "delay": args.gnss_delay,
                       "as_position": args.gnss_as_position, "heading_every": args.heading_every, "heading_sigma": args.heading_sigma,
                       **{k: s["gnss"][k] for k in ("mean_anis", "mean_dof", "run_bounds", "updates_inside", "applied", "degenerate") + FAULTS}}
    if "range" in s:
        res["range"] = {"every": args.range_every, "sigma_m": args.range_sigma, "lever_m": args.range_lever, "delay": args.range_delay,
                        "plane_every": args.plane_every, "plane_sigma_m": args.plane_sigma, "plane_height_m": args.plane_height,
                        "plane_axis": args.plane_axis, "plane_lever_m": args.plane_lever,
                        **{k: s["range"][k] for k in ("mean_anis", "mean_dof", "run_bounds", "updates_inside", "applied", "degenerate") + FAULTS}}
    for key, start in (("range", args.range_start), ("gnss", args.gnss_start)):
        if key in res and (start or args.aid_iterations != 1):
            res[key].update(start=start, iterations=args.aid_iterations, tol=args.aid_tol)
            if key + "_first" in s:
                res[key]["first_stack"] = s[key + "_first"]
    if args.fde_alpha > 0 or args.range_outlier_rate > 0 or args.gnss_outlier_rate > 0:
        res["faults"] = {"range_outlier_rate": args.range_outlier_rate, "range_outlier_bias_m": args.range_outlier_bias,
                         "gnss_outlier_rate": args.gnss_outlier_rate, "gnss_outlier_jump_m": args.gnss_outlier_jump,
                         "fde_alpha": args.fde_alpha, "fde_max_exclude": args.fde_max_exclude}
    if "stops" in s:
        res["stops"] = dict(s["stops"], every=args.stop_every, frames_per_stop=args.stop_frames, ramp=args.stop_ramp,
                            standstill=standstill)
        res["stops"].pop("stops")
    for c, v in s["components"].items():  # the per-frame bounds of the first frame (the same for every frame of a fixed dimension)
        res["components"][c]["bounds_frame0"] = [v["lower"][0], v["upper"][0]]
    if not args.no_timing and rank == 0:
        res["nees_timing"] = {str(n): time_nees(n) for n in (8, 32)}
        res["aid_call_ms"] = {str(n): time_aid(n) for n in (1, 8, 32)}
    if rank == 0:
        print(json.dumps(res), flush=True)
        if args.out:
            args.out.parent.mkdir(parents=True, exist_ok=True)
            args.out.write_text(json.dumps({"result": res, "summary": s}, indent=1))
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
