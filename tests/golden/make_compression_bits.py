"""Generates tests/golden/compression_bits.npz: the exact bits one MARGINALIZE leaves on the device (covariance, delta-x, IMU
state, clone poses, accept flags, m and rank) at shapes that reach every tiling of the compression stage's Gram products and
their split-K sum (k_gram_mma, k_gram, k_assemble).  The rank decision of a long fp32 window looks at pivots that are rounding
noise, so a change in the last bit of T'', R'' or r'' can move it: these vectors pin the bits, not a tolerance.

Run on the GPU:  python tests/golden/make_compression_bits.py [out.npz]
Inputs are regenerated deterministically by msckf_mono_b200.synth (seeded); only outputs are stored.
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

# name: members of one device batch, each (n_features, n_clones, seq, dtype).  c = 6 * n_clones is the Gram products' order,
# K = 3 * n_features their depth (nsplit = K // 96 split-K chunks, at most 16); >= 200 tracks run them on the FP64 tensor cores
CASES = {
    # the benchmark's batch: 8 config-B filters (c = 180: six 32-tiles, the last one 20 columns wide; nsplit = 9)
    "bench": [(300, 30, s, "float32") for s in range(8)],
    "c192": [(250, 32, 40, "float32")],            # whole 32-tiles only
    "c30": [(250, 5, 41, "float32")],              # one partial 32-tile
    "c66": [(250, 11, 42, "float32")],             # three 32-tiles, the last one 2 columns wide
    "nsplit1": [(20, 10, 43, "float32")],          # SIMT Gram tiles, one split
    "nsplit16_f64": [(512, 12, 44, "float64")],    # K = 1536: sixteen splits, fp64
    "m_le_n": [(2, 10, 45, "float32")],            # m = 34 <= n = 75: every row explicit, no Gram part
    "mixed": [(250, 11, 46, "float32"), (120, 20, 47, "float32"), (300, 30, 48, "float32"), (40, 6, 49, "float32")],
}


def members(case):
    """(template engine, its queued tracks, the class filter that owns it) per member, driven up to the MARGINALIZE"""
    from msckf_mono_b200 import capi, engine_filter, synth
    out = []
    for nf, nc, seq, dt in CASES[case]:
        wl = synth.make_window_workload(n_features=nf, n_clones=nc, seq=seq)
        f = engine_filter(np.dtype(dt).type, max_clones=nc + 8, max_tracks=max(512, nf + 48), max_obs=max(512, nf + 48) * nc)
        synth.drive(f, wl, marginalize_last=False)
        off, obs, idx = f.packQueued()
        out.append((capi.Engine(np.dtype(dt).type, borrowed=f.engineHandle()), capi.TrackBatch(off, obs, idx, np.dtype(dt).type), f))
    return out


def outputs(e, rep):
    """what the update leaves, the covariance as its upper triangle (the engine keeps P bitwise symmetric: asserted)"""
    imu, poses = e.state()
    P = e.covariance()
    assert np.array_equal(P, P.T)
    return {"covariance": P[np.triu_indices(P.shape[0])], "delta_x": e.delta_x(), "imu_state": imu, "clone_poses": poses,
            "accepted": rep["accepted"].astype(np.int32), "m_rank": np.array([rep["m"], rep["rank"]], np.int64)}


def run(case, batched):
    """the outputs of each member after one MARGINALIZE, as one device batch or filter by filter"""
    from msckf_mono_b200 import capi
    mem = members(case)
    work = []
    for tmpl, b, _ in mem:
        w = capi.Engine(tmpl.dtype, max_clones=tmpl.num_clones() + 8, max_tracks=max(512, b.n_tracks + 48),
                        max_obs=max(512, b.n_tracks + 48) * tmpl.num_clones())
        w.copy_state_from(tmpl)
        work.append(w)
    batches = [b for _, b, _ in mem]
    if batched:
        grp = capi.Batch(work)
        reps = grp.update(capi.MARGINALIZE, batches)
        res = [outputs(w, r) for w, r in zip(work, reps)]
        grp.close()
    else:
        res = [outputs(w, w.update(capi.MARGINALIZE, b)) for w, b in zip(work, batches)]
    for w in work:
        w.close()
    return res


def key(case, i, name):
    return f"{case}/{i}/{name}"


def main(path):
    arrays = {}
    for case in CASES:
        for i, out in enumerate(run(case, batched=len(CASES[case]) > 1)):
            for name, a in out.items():
                arrays[key(case, i, name)] = a
            print(case, i, "m", out["m_rank"][0], "rank", out["m_rank"][1], "accepted", int(out["accepted"].sum()), flush=True)
    np.savez_compressed(path, **arrays)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else str(Path(__file__).with_name("compression_bits.npz")))
