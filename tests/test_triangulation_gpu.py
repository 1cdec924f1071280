"""k_tri (checkMotion + LM triangulation, TRIANGULATE) against the plain fp64 reference of tests/triangulation_reference.py
computed from the engine's own fetched poses, inputs rounded to the filter's type: the flags exactly, p_f_G relative to the
landmark's distance from the track's first clone.
  (a) the designed tracks: every rejection kind, both exits of the LM's loops, the damping's floor, the Huber branch and all
      six elimination orders of the 3 x 3 solve (what they take is asserted in tests/test_triangulation_reference_cpu.py);
  (b) track lengths on and around the 32-stride of the lane loops, four clone-subset styles each;
  (c) track counts around the four tracks of a CTA and the 16 the grid is rounded to, with rejections at CTA edges, growing the
      track buffers from a small capacity;
  (d) windows of 2 .. 192 clones (the engine's hard limit; TRIANGULATE is not bound by the update's 136): P, the state and
      the counters are left alone;
  (e) one device batch whose members differ in window, longest track and track count, so that each carves the launch's
      shared memory its own way: bit-identical to single filters and right, launched, captured and replayed;
  (f) single observations among other tracks of a CTA: rejected with p_f_G = 0, the neighbours untouched."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import triangulation_reference as tr
from tests import vision_reference as vr
from tests.parity_cases import make_engine
from tests.test_update_shapes_gpu import counters, engine, state64, twin

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
# worst |p_f_G - reference| / |reference - first clone| over each dtype's cases, measured on an H100 80GB HBM3 (700 W power
# limit); asserted at 10 x these and under vr.CONTRACT
MEASURED = {"float64": 4.6e-8, "float32": 2.9e-4}
PARAMS = vr.setup()[2]


def engine_at(dtype, M, threshold):
    """an engine with the builder's M clones whose translation_threshold is `threshold` (tests.test_update_shapes_gpu.engine
    fixes the parameters)"""
    f = make_engine(dtype, max_clones=min(M + 1, 192), max_tracks=8, max_obs=64)
    cam, noise, params, imu = vr.setup()
    f.initialize(cam, noise, dict(params, translation_threshold=threshold), imu)
    e = capi.Engine(dtype, borrowed=f.engineHandle())
    e.filt = f
    for k in range(M):
        if k:
            e.propagate_n(vr.readings(k))
        e.augment()
    return e


def tri_batch(tracks, dtype):
    return capi.TrackBatch(*vr.pack([dict(t, pfg=np.zeros(3)) for t in tracks], dtype)[:3], dtype)


def reference(e, tracks, dtype, params=PARAMS):
    poses = e.state()[1].astype(np.float64)
    return poses, tr.triangulate(poses, [dict(t, obs=t["obs"].astype(dtype).astype(np.float64)) for t in tracks], params)


def compare(rep, ref, poses, tracks, dtype, label, skip_pfg=()):
    """flags exactly; p_f_G of the tracks the reference accepts (a rejected track's LM may legitimately take another path after a
    cost comparison that rounding decides) except those of a kind in skip_pfg; returns the worst relative difference"""
    name = np.dtype(dtype).name
    L = np.array([len(t["idx"]) for t in tracks])
    assert np.array_equal(rep["cm_ok"].astype(bool), ref["cm"]), (label, np.flatnonzero(rep["cm_ok"].astype(bool) != ref["cm"]))
    assert np.array_equal(rep["tri_ok"].astype(bool), ref["ok"]), (label, np.flatnonzero(rep["tri_ok"].astype(bool) != ref["ok"]))
    assert not rep["p_f_G"][L < 2].any(), label
    assert np.isfinite(rep["p_f_G"]).all(), label
    worst = 0.0
    for j, t in enumerate(tracks):
        # fp32: a depth from a baseline below 1/50 of it amplifies the rounding of 30 m positions past any useful bound
        far = name == "float32" and 50 * np.linalg.norm(poses[t["idx"][-1], 0:3] - poses[t["idx"][0], 0:3]) < np.linalg.norm(ref["pfg"][j] - poses[t["idx"][0], 0:3])
        if ref["ok"][j] and t.get("kind") not in skip_pfg and not far:
            d = np.abs(rep["p_f_G"][j].astype(np.float64) - ref["pfg"][j]).max() / np.linalg.norm(ref["pfg"][j] - poses[t["idx"][0], 0:3])
            assert d <= vr.CONTRACT[name]["p_f_G"] and d <= 10 * MEASURED[name], (label, j, t.get("name"), d)
            worst = max(worst, float(d))
    print(f"{label}: {len(tracks)} tracks, {int(ref['cm'].sum())} pass checkMotion, {int(ref['ok'].sum())} triangulate, p_f_G {worst:.2e}")
    return worst


def run(e, tracks, dtype, label, params=PARAMS, skip_pfg=()):
    poses, ref = reference(e, tracks, dtype, params)
    rep = e.update(capi.TRIANGULATE, tri_batch(tracks, dtype))
    compare(rep, ref, poses, tracks, dtype, label, skip_pfg)
    return rep, ref


def rejected_tracks(poses, rng):
    """one track per rejection kind on any window of 4 or more clones: checkMotion (a single observation), cost (gross outliers)"""
    M = len(poses)
    if M < 3:
        return [{"idx": np.zeros(1, np.int32), "obs": np.zeros((1, 2))}]
    idx = np.sort(rng.choice(M, 3, replace=False))
    obs, _ = tr._observe(poses, idx, tr._ahead(poses, idx[1], 0.2, 5.0))
    obs[1] += 0.3
    return [{"idx": idx[:1].astype(np.int32), "obs": obs[:1]}, {"idx": idx.astype(np.int32), "obs": obs}]


# --------------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_branch(dtype):
    e = engine_at(dtype, 70, tr.DESIGN_THRESHOLD)
    poses = e.state()[1].astype(np.float64)
    tracks = tr.designed_tracks(poses, tr.DESIGN_THRESHOLD)
    params = dict(PARAMS, translation_threshold=float(dtype(tr.DESIGN_THRESHOLD)))
    if dtype == np.float32:  # the flags an fp32 run of the reference decides otherwise are legitimately either way: left out
        out = set(tr.fp32_excluded(poses, tracks, params))
        print("fp32 exclusions:", sorted(out))
        assert out <= set(tr.FP32_EXCLUDED) | {t["name"] for t in tracks if t["kind"] == "noisy"}
        tracks = [t for t in tracks if t["name"] not in out]
    rep, ref = run(e, tracks, dtype, f"{np.dtype(dtype).name} designed", params, skip_pfg=("noisy", "behind"))
    kinds = {t["kind"] for t, c, o in zip(tracks, ref["cm"], ref["ok"]) if not (c and o)}
    assert {"motion-", "behind", "cost"} <= kinds
    assert {t["orders"][0] for t in ref["tri_trace"]} == set(tr.ORDERS)


# --------------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("dtype", DTYPES)
def test_track_lengths(dtype):
    e = twin(dtype, 98)
    poses = state64(e)[2]
    lengths = [L for L in (1, 2, 3, 31, 32, 33, 63, 64, 65, 95, 96, 97, 98) for _ in range(4)]
    tracks = vr.make_tracks(np.random.default_rng(11), poses, lengths)
    # make_tracks takes its style from the track's position: four in a row are the four styles
    rep, ref = run(e, tracks, dtype, f"{np.dtype(dtype).name} lengths")
    assert ref["ok"].sum() == len(lengths) - 4


# --------------------------------------------------------------------------------------------------------------------- (c)
@pytest.mark.parametrize("dtype,N", [(dt, N) for N in (1, 3, 4, 5, 15, 16, 17, 511, 512, 513, 4096) for dt in DTYPES
                                     if dt == np.float64 or N in (5, 17, 513)])
def test_track_counts(dtype, N):
    e = twin(dtype, 12)  # created for 64 tracks: the larger counts grow its buffers
    poses = state64(e)[2]
    rng = np.random.default_rng(N)
    tracks = vr.make_tracks(rng, poses, [(2, 3, 12, 7, 5)[j % 5] for j in range(N)])
    bad = rejected_tracks(poses, rng)
    for k, j in enumerate(sorted({j for j in (3, 4, 7, 8, N - 1) if 0 <= j < N})):  # the last and first track of a CTA, the last of all
        tracks[j] = bad[k % 2]
    rep, ref = run(e, tracks, dtype, f"{np.dtype(dtype).name} N={N}")
    assert not ref["ok"][N - 1]


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("dtype,M", [(dt, M) for M in (2, 98, 136, 137, 191, 192) for dt in DTYPES if dt == np.float64 or M in (2, 192)])
def test_windows(dtype, M):
    e = twin(dtype, M) if M < 192 else engine_at(dtype, M, PARAMS["translation_threshold"])  # (twin allocates M + 1 clones)
    poses = state64(e)[2]
    before = state64(e) + (counters(e), e.rank_pivots())
    rng = np.random.default_rng(M)
    lengths = [min(L, M) for L in (2, 3, 33, 64, 98, 98, 17, 5)]
    tracks = vr.make_tracks(rng, poses, lengths) + rejected_tracks(poses, rng)
    # styles 3 and 1 start at clone 0 and end at clone M - 1
    assert any(t["idx"][0] == 0 for t in tracks) and any(t["idx"][-1] == M - 1 for t in tracks)
    run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M}")
    for x, y in zip(before, state64(e) + (counters(e), e.rank_pivots())):
        assert np.array_equal(x, y), M


# --------------------------------------------------------------------------------------------------------------------- (e)
# (window, track lengths): a long window with short tracks next to a short window with its longest, so that no member's carve of
# the shared memory is the launch's; no tracks, one track, 600 tracks
MEMBERS = [(191, [2, 3, 2, 5, 4]), (98, [98, 97, 33, 2, 64]), (2, [2]), (40, []), (12, [(2, 3, 12, 7)[j % 4] for j in range(600)]),
           (136, [17, 65, 3]), (33, [33, 32, 31, 1, 2])]


@pytest.mark.parametrize("dtype", DTYPES)
def test_device_batch_is_bit_identical_and_right(dtype):
    mem = [twin(dtype, M) for M, _ in MEMBERS]
    solo = [engine(dtype, M, src=m) for m, (M, _) in zip(mem, MEMBERS)]
    batch = capi.Batch(mem)
    for it in range(3):  # the same launch shape three times: launched directly, captured as a graph, replayed
        tracks = []
        for i, (m, (M, lengths)) in enumerate(zip(mem, MEMBERS)):
            rng = np.random.default_rng(100 * it + i)
            poses = state64(m)[2]
            t = vr.make_tracks(rng, poses, lengths)
            if len(t) >= 5:
                t[3] = dict(t[3], obs=t[3]["obs"] + 0.3 * (np.arange(len(t[3]["obs"]))[:, None] % 2))  # a cost rejection
            tracks.append(t)
        reps = batch.update(capi.TRIANGULATE, [tri_batch(t, dtype) for t in tracks], full=True)
        for i, (m, s, t, rep) in enumerate(zip(mem, solo, tracks, reps)):
            if not t:
                continue
            label = f"{np.dtype(dtype).name} member {i} run {it}"
            r1 = s.update(capi.TRIANGULATE, tri_batch(t, dtype))
            for k in ("cm_ok", "tri_ok", "p_f_G"):
                assert np.array_equal(rep[k], r1[k]), (label, k)
            poses, ref = reference(m, t, dtype)
            compare(rep, ref, poses, t, dtype, label)
    batch.close()


# --------------------------------------------------------------------------------------------------------------------- (f)
def test_single_observation_tracks_between_others():
    e = twin(np.float64, 12)
    poses = state64(e)[2]
    base = vr.make_tracks(np.random.default_rng(1), poses, [5, 12, 3, 7, 2, 9, 4, 6])
    rep0 = e.update(capi.TRIANGULATE, tri_batch(base, np.float64))
    for w in range(4):  # a single observation in warp w of the first CTA and in warp 3 - w of the second
        tracks = list(base)
        for j in (w, 7 - w):
            tracks[j] = {"idx": base[j]["idx"][:1], "obs": base[j]["obs"][:1]}
        rep = e.update(capi.TRIANGULATE, tri_batch(tracks, np.float64))
        for j in range(8):
            if j in (w, 7 - w):
                assert rep["cm_ok"][j] == 0 and rep["tri_ok"][j] == 0 and not rep["p_f_G"][j].any(), (w, j)
            else:
                assert all(np.array_equal(rep[k][j], rep0[k][j]) for k in ("cm_ok", "tri_ok", "p_f_G")), (w, j)
