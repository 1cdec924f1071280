#!/usr/bin/env python
"""scripts/landmark_rate.py -- call time of the mapped-landmark update (msckf_b200_landmark_update / _batch_landmark_update) in
fp64 at 30 clones, for 1 / 8 / 32 filters and 25 / 100 / 400 observations spread over the newest 1 / 5 / 30 clones: host wall
clock around the synchronising call, median of 20 after a warm-up.  For <= 16 observations on one filter it also times the path
available without it: get_state, the projection linearised in numpy, then one aid_update(LINEAR).  Per-kernel device times
(k_lmk_clone, k_lmk_gain, k_lmk_downdate) come from torch.profiler over repeated calls.  With --iterations K ..., it times the
iterated update instead: 25 observations over the newest clone and 100 over the newest 5, seen from poses 0.3 m away, at each
max_iter K with tol 0 (so every call makes its K linearisations unless a step is exactly zero), for 1 / 8 / 32 filters, with the
linearisations the calls reported and the per-kernel split (k_lmk_step too) for 100 over 5.  Reads the card's name and power
limit in the same process.  With --map-sigma S, it times the update with map uncertainty instead: 25 and 100 landmarks, each
seen from the newest 1 and 5 clones, with Sigma = S^2 I (msckf_b200_map_landmark_update) against the same observations with
Sigma NULL, for 1 / 8 / 32 filters.  With --consensus H ..., it times the update with a consensus of H hypotheses
(msckf_b200_landmark_update_consensus) against the plain call on the same 100 observations over the newest 5 clones, 30 % of
them wrong matches, for 1 / 8 / 32 filters, with the per-kernel split (k_lmk_hyp, k_lmk_cons too) at 1 and 32 filters.
Prints one JSON line."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from msckf_mono_b200 import capi, synth  # noqa: E402

M = 30
R_PIX = np.diag([2.0e-5, 2.0e-5])


def gpu_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def filters(n):
    from msckf_mono_b200 import engine_filter
    wl = synth.make_window_workload(n_features=4, n_clones=2, seq=3)
    rng = np.random.default_rng(7)
    fs, es = [], []
    for _ in range(n):
        f = engine_filter(np.float64, max_clones=M + 8)
        f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        e = capi.Engine(np.float64, borrowed=f.engineHandle())
        for _ in range(M):
            r = np.zeros((2, 7)); r[:, 0:3] = rng.normal(0, 0.3, (2, 3)); r[:, 3:6] = [0, 0, 9.81]; r[:, 6] = 0.005
            e.propagate_n(r)
            e.augment()
        nn = 15 + 6 * M
        A = rng.normal(size=(nn, nn))
        e.set_covariance(1e-4 * (A @ A.T / nn + np.eye(nn)))
        fs.append(f); es.append(e)
    return fs, es


def observations(rng, e, n_obs, n_clones, offset=None):
    """n_obs observations spread evenly over the newest n_clones clones, landmarks 2 .. 8 m in front, measured exactly (from
    clone positions moved by `offset`, when given)"""
    _, poses = e.state()
    poses = poses.astype(np.float64)
    if offset is not None:
        poses[:, 0:3] += offset
    clone = np.array([M - 1 - (i % n_clones) for i in range(n_obs)], dtype=np.int32)
    d = rng.uniform(2.0, 8.0, n_obs)
    pc = np.stack([rng.uniform(-0.4, 0.4, n_obs) * d, rng.uniform(-0.3, 0.3, n_obs) * d, d], axis=1)
    p_L = np.array([rot(poses[k, 3:7]).T @ v + poses[k, 0:3] for k, v in zip(clone, pc)])
    return {"clone": clone, "z": pc[:, 0:2] / pc[:, 2:3], "p_L": p_L, "R": R_PIX}


def timed(fn, reps=20):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def host_linear(e, spec):
    """the path without the feature: get_state, numpy linearisation, one aid_update(LINEAR)"""
    _, poses = e.state()
    poses = poses.astype(np.float64)
    n = 15 + 6 * M
    m = 2 * len(spec["clone"])
    H, r = np.zeros((m, n)), np.zeros(m)
    for i, (k, zi, pl) in enumerate(zip(spec["clone"], spec["z"], spec["p_L"])):
        C = rot(poses[k, 3:7])
        X, Y, Z = C @ (pl - poses[k, 0:3])
        J = np.array([[1, 0, -X / Z], [0, 1, -Y / Z]]) / Z
        sk = np.array([[0, -Z, Y], [Z, 0, -X], [-Y, X, 0]])
        H[2 * i:2 * i + 2, 15 + 6 * k:21 + 6 * k] = np.hstack([J @ sk, -J @ C])
        r[2 * i:2 * i + 2] = zi - np.array([X, Y]) / Z
    return e.aid_update(capi.AID_LINEAR, r, np.kron(np.eye(m // 2), spec["R"]), H=H)


def kernel_times(fn, reps=50):
    """mean device time per call of each landmark kernel, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("k_lmk_hyp", "k_lmk_cons", "k_lmk_clone", "k_lmk_set", "k_lmk_gain", "k_lmk_step", "k_lmk_downdate"):
            if name in ev.key:
                out[name] = out.get(name, 0.0) + ev.device_time_total / 1e3 / reps  # ms per call
    return out


def iterated(ks):
    rng = np.random.default_rng(5)
    res = {"gpu": gpu_line(), "dtype": "f64", "clones": M, "offset_m": 0.3, "tol": 0.0, "call_ms": {}, "iterations": {},
           "kernel_ms": {}}
    for nf in (1, 8, 32):
        fs, es = filters(nf)
        b = capi.Batch(es) if nf > 1 else None
        for n_obs, nc in ((25, 1), (100, 5)):
            specs = [observations(rng, e, n_obs, nc, offset=np.array([0.3, 0.0, 0.0])) for e in es]
            for k in ks:
                key = f"{nf}x{n_obs}obs/{nc}clones/max_iter{k}"
                its = []
                sp = [dict(s, max_iter=k, tol=0.0) for s in specs]

                def fn():
                    out = b.landmark_update(sp) if b else [es[0].landmark_update(**sp[0])]
                    its.append(np.mean([o["iterations"] for o in out]))
                res["call_ms"][key] = timed(fn)
                res["iterations"][key] = float(np.mean(its))
                if nf in (1, 32) and n_obs == 100:
                    try:
                        res["kernel_ms"][key] = kernel_times(fn)
                    except Exception as ex:  # (the profiler is an extra; the call times above stand on their own)
                        res["kernel_ms"][key] = f"not measured: {ex}"
        if b:
            b.close()
        for f in fs:
            f.close()
    print(json.dumps(res), flush=True)


def map_spec(rng, e, n_lm, n_clones, sigma):
    """n_lm landmarks in front of the newest clone, each observed exactly from n_clones consecutive clones (the newest ones, or
    for odd landmarks with n_clones > 1 the ones before the newest, so no clone set holds more than 256 observations), with
    Sigma = sigma^2 I (the exact-map call when sigma is None)"""
    _, poses = e.state()
    poses = poses.astype(np.float64)
    p = observations(rng, e, n_lm, 1)["p_L"]
    clone, z, p_L, lm = [], [], [], []
    for l in range(n_lm):
        last = M - (l % 2 if n_clones > 1 else 0)
        for k in range(last - n_clones, last):
            pc = rot(poses[k, 3:7]) @ (p[l] - poses[k, 0:3])
            clone.append(k); z.append(pc[0:2] / pc[2]); p_L.append(p[l]); lm.append(l)
    spec = {"clone": np.array(clone, np.int32), "z": np.array(z), "p_L": np.array(p_L), "R": R_PIX}
    if sigma is not None:
        spec.update(landmark=np.array(lm, np.int32), Sigma_L=np.tile([sigma ** 2, 0, sigma ** 2, 0, 0, sigma ** 2], (n_lm, 1)))
    return spec


def uncertain(sigma):
    res = {"gpu": gpu_line(), "dtype": "f64", "clones": M, "map_sigma_m": sigma, "call_ms": {}, "kernel_ms": {}}
    for nf in (1, 8, 32):
        fs, es = filters(nf)
        b = capi.Batch(es) if nf > 1 else None
        for n_lm in (25, 100):
            for nc in (1, 5):
                for tag, s in (("NULL", None), ("Sigma", sigma)):
                    specs = [map_spec(np.random.default_rng([n_lm, nc, i]), e, n_lm, nc, s) for i, e in enumerate(es)]
                    fn = (lambda: b.landmark_update(specs)) if b else (lambda: es[0].landmark_update(**specs[0]))
                    key = f"{nf}x{n_lm}landmarks/{nc}clones/{tag}"
                    res["call_ms"][key] = timed(fn)
                    if nf in (1, 32) and n_lm == 100 and nc == 5:
                        try:
                            res["kernel_ms"][key] = kernel_times(fn)
                        except Exception as ex:  # (the profiler is an extra; the call times above stand on their own)
                            res["kernel_ms"][key] = f"not measured: {ex}"
        if b:
            b.close()
        for f in fs:
            f.close()
    print(json.dumps(res), flush=True)


def consensus(hs):
    res = {"gpu": gpu_line(), "dtype": "f64", "clones": M, "obs": 100, "wrong": 0.3, "call_ms": {}, "kernel_ms": {}, "inliers": {}}
    for nf in (1, 8, 32):
        for h in [0] + list(hs):  # fresh filters for each setting: the timed calls apply their updates
            fs, es = filters(nf)
            b = capi.Batch(es) if nf > 1 else None
            specs = []
            for i, e in enumerate(es):
                rng = np.random.default_rng([nf, i])
                sp = observations(rng, e, 100, 5)
                wrong = np.flatnonzero(rng.uniform(size=100) < 0.3)
                sp["p_L"][wrong] = sp["p_L"][(wrong + 1 + rng.integers(99, size=len(wrong))) % 100]
                specs.append(sp)
            cs = None if h == 0 else {"hypotheses": h, "thresh": 13.8, "min_inliers": 10, "seed": 1}
            key = f"{nf}x100obs/5clones/" + ("plain" if h == 0 else f"consensus{h}")
            out = []
            fn = (lambda: out.append(b.landmark_update(specs, consensus=cs))) if b else \
                (lambda: out.append([es[0].landmark_update(**specs[0], consensus=cs)]))
            res["call_ms"][key] = timed(fn)
            if h:
                res["inliers"][key] = float(np.mean([o["consensus"]["inliers"] for o in out[0]]))  # the first call, on the unchanged filters
            if nf in (1, 32):
                try:
                    res["kernel_ms"][key] = kernel_times(fn)
                except Exception as ex:  # (the profiler is an extra; the call times above stand on their own)
                    res["kernel_ms"][key] = f"not measured: {ex}"
            if b:
                b.close()
            for f in fs:
                f.close()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--consensus", type=int, nargs="*", default=None, help="time consensus calls of these hypothesis counts")
    ap.add_argument("--iterations", type=int, nargs="*", default=None)
    ap.add_argument("--map-sigma", type=float, default=None, help="time Sigma = s^2 I against Sigma NULL")
    args = ap.parse_args()
    if args.consensus:
        return consensus(args.consensus)
    if args.iterations:
        return iterated(args.iterations)
    if args.map_sigma is not None:
        return uncertain(args.map_sigma)
    rng = np.random.default_rng(3)
    res = {"gpu": gpu_line(), "dtype": "f64", "clones": M, "call_ms": {}, "host_linear_ms": {}, "kernel_ms": {}}
    for nf in (1, 8, 32):
        fs, es = filters(nf)
        b = capi.Batch(es) if nf > 1 else None
        for n_obs in (25, 100, 400):
            for nc in (1, 5, 30):
                key = f"{nf}x{n_obs}obs/{nc}clones"
                if n_obs > 256 * nc:
                    res["call_ms"][key] = "over the 256-per-clone cap"
                    continue
                specs = [observations(rng, e, n_obs, nc) for e in es]
                fn = (lambda: b.landmark_update(specs)) if b else (lambda: es[0].landmark_update(**specs[0]))
                res["call_ms"][key] = timed(fn)
                if nf in (1, 32) and n_obs == 100 and nc == 5:
                    try:
                        res["kernel_ms"][key] = kernel_times(fn)
                    except Exception as ex:  # (the profiler is an extra; the call times above stand on their own)
                        res["kernel_ms"][key] = f"not measured: {ex}"
        if nf == 1:
            for n_obs in (4, 16):
                spec = observations(rng, es[0], n_obs, 1)
                res["host_linear_ms"][f"1x{n_obs}obs/1clone"] = timed(lambda: host_linear(es[0], spec))
                res["call_ms"][f"1x{n_obs}obs/1clone"] = timed(lambda: es[0].landmark_update(**spec))
        if b:
            b.close()
        for f in fs:
            f.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
