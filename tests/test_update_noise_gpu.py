"""The vision update (RESIDUALIZE) under anisotropic pixel noise (u_var != v_var) against the reference of
tests/vision_reference.py, with the shape sweep's builders (tests/test_update_shapes_gpu.py).  Isotropic noise leaves most of
the terms that carry it at exactly zero or at a multiple of another term (the head rows' -(A_h^T D U) Z correction, the
asymmetry of Z^T Yq, the u / v parity of Yq, D2 and the explicit rows' noise, the gate's u_var): at v_var = 4 u_var a slip in
any of them moves dx by 7e-4 .. 5 (tests/test_update_noise_cpu.py), far past the bounds below.
  (a) windows of 1 .. 136 clones (every tail boundary) at v_var = 4 u_var, and at v_var = u_var / 4 on either side of them;
  (b) 1 .. 512 tracks at 12 and 33 clones: every stacked row explicit (m <= n, m = n), the first compressed system, the
      split-K chunks and the DMMA boundary;
  (c) the first 15 stacked rows (explicit when m > n) on a track edge, across a track, inside one track, one row per track,
      with a gated-out track among them;
  (d) the Gram products on SIMT and DMMA tiles, each against the reference and against each other;
  (e) one device batch whose members hold different pixel noise (isotropic, EuRoC, 4, 1/4) over the tail kinds, each member
      against its own reference and its single-filter twin bit for bit, launched directly, captured as a graph and replayed;
  (f) the mapped-landmark update with the filter's own noise (R omitted) equals the call given R = diag(u_var, v_var), bit
      for bit: single, iterated, with map uncertainty, and in a device batch of members of different noise."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import test_update_shapes_gpu as shp
from tests import vision_reference as vr
from tests.parity_cases import measured as parity_measured
from tests.test_landmark_map_gpu import CHI2, scene, sets_for

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
# worst differences to the reference over this file's cases (same measures as tests/test_update_shapes_gpu.py), measured on an
# H100 80GB HBM3 (700 W power limit); every case is asserted at 10 x these and at most at CONTRACT, the isotropic sweep's
# ceilings.  fp32: the cases whose rank equals the reference's.
MEASURED = {"float64": {"dx": 7.66e-06, "P": 5.46e-08, "state": 7.66e-06, "gamma": 4.04e-13},
            "float32": {"dx": 3.02e-03, "P": 8.75e-07, "state": 1.82e-02, "gamma": 1.21e-04}}
CONTRACT = vr.CONTRACT
# fp32 cases whose rank is above the reference's (DESIGN.md 4.4, "fp32 filters under anisotropic noise"): the rank decision of
# an fp32 filter has no gap between rounding noise and the weakest real pivots and keeps some Gamma directions on noise.  Under
# isotropic noise such a direction changes nothing; under anisotropic noise it adds a residual component whose noise is
# correlated with the other rows, and that moves dx (12 % of max |dx| at M = 32, v_var = 4 u_var).  Only these cases are held
# to the wider dx and state ceiling; the same card, measured over them.
EXTRA_RANK_F32 = ({"dx": 0.5, "P": 1e-3, "state": 0.5, "gamma": 1e-2},
                  {"dx": 1.22e-01, "P": 4.62e-04, "state": 1.22e-01, "gamma": 1.00e-04})


def bounds(name, extra_rank):
    """(contract, measured) of a case of dtype `name` whose rank is `extra_rank` above the reference's"""
    return EXTRA_RANK_F32 if name == "float32" and extra_rank > 0 else (CONTRACT[name], MEASURED[name])


def nz(ratio, dtype):
    return vr.pixel_noise(ratio, dtype)


def run(e, tracks, dtype, label, noise):
    return shp.run(e, tracks, dtype, label, noise=noise, bounds=bounds)


# --------------------------------------------------------------------------------------------------------------------- (a)
WINDOW_CASES = [(dt, M, 4.0) for M in shp.WINDOWS for dt in DTYPES] + [(dt, M, 0.25) for M in (32, 33, 63, 64, 136) for dt in DTYPES]


@pytest.mark.parametrize("dtype,M,ratio", WINDOW_CASES)
def test_window_sweep_at_anisotropic_noise(dtype, M, ratio):
    noise = nz(ratio, dtype)
    e = shp.twin(dtype, M, noise)
    _, _, poses = shp.state64(e)
    tracks = shp.sweep_tracks(np.random.default_rng(M), poses, shp.window_lengths(M), unseen=shp.unseen_of(M), outliers=(5, 16))
    rep, ref, _ = run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} v/u={ratio:g}", noise)
    if M == 1:
        assert rep["m"] == 0 and not rep["accepted"].any()
    else:
        assert ref["accepted"].sum() >= len(tracks) // 2


# --------------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("dtype,M,N", shp.N_CASES)
def test_track_count_sweep_at_anisotropic_noise(dtype, M, N):
    noise = nz(4.0, dtype)
    e = shp.twin(dtype, M, noise)
    n = 15 + 6 * M
    _, _, poses = shp.state64(e)
    lengths = shp.n_sweep_lengths(M, N)
    outl = () if isinstance(N, str) else tuple(j for j in range(7, len(lengths), 50))
    tracks = shp.sweep_tracks(np.random.default_rng(1000 + M), poses, lengths, outliers=outl)
    rep, ref, _ = run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} N={N} v/u=4", noise)
    if N == "m=n":
        assert ref["m"] == n and rep["rank"] == n
    if N == "m=n+1":
        assert ref["m"] == n + 1 and ref["sv"] is not None


# --------------------------------------------------------------------------------------------------------------------- (c)
HEAD = [(dt, 12, h) for h in vr.HEAD_CASES for dt in DTYPES] + [(np.float64, 40, "straddle"), (np.float64, 70, "gated")]


@pytest.mark.parametrize("dtype,M,case", HEAD)
def test_head_rows_at_anisotropic_noise(dtype, M, case):
    noise = nz(4.0, dtype)
    e = shp.twin(dtype, M, noise)
    _, _, poses = shp.state64(e)
    lengths, outl = vr.head_lengths(case, M)
    tracks = shp.sweep_tracks(np.random.default_rng(M), poses, lengths, outliers=outl)
    rep, ref, _ = run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} head {case} v/u=4", noise)
    assert ref["m"] > 15 + 6 * M and ref["accepted"][list(outl)].sum() == 0 and ref["accepted"].sum() == len(tracks) - len(outl)


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("N", [200, 512])
def test_gram_tiles_simt_and_dmma_at_anisotropic_noise(N):
    """option 5 = 0 forces the SIMT Gram tiles where the engine would take DMMA (200 tracks and more): both against the
    reference, and against each other at the level of test_gram_on_fp64_tensor_cores_matches_simt_tiles"""
    noise = nz(4.0, np.float64)
    out = []
    for opt in ({}, {5: 0.0}):
        e = shp.twin(np.float64, 12, noise)
        for k, v in opt.items():
            e.set_option(k, v)
        _, _, poses = shp.state64(e)
        tracks = shp.sweep_tracks(np.random.default_rng(N), poses, shp.n_sweep_lengths(12, N), outliers=(7,))
        rep, _, _ = run(e, tracks, np.float64, f"float64 M=12 N={N} options {opt} v/u=4", noise)
        out.append((rep, e.covariance(), e.delta_x()))
    (ra, Pa, dxa), (rb, Pb, dxb) = out
    assert ra["rank"] == rb["rank"] and np.array_equal(ra["accepted"], rb["accepted"])
    lim = parity_measured()["gram_mma_vs_simt_300x30"]
    d = {"dx": float(np.abs(dxa - dxb).max() / np.abs(dxa).max()), "P": float(np.abs(Pa - Pb).max() / np.abs(Pa).max())}
    print(f"DMMA vs SIMT N={N}: " + " ".join(f"{k} {v:.2e}" for k, v in d.items()))
    assert 0 < d["dx"] <= 10 * lim["dx"] and d["P"] <= 10 * lim["P"], d


# --------------------------------------------------------------------------------------------------------------------- (e)
# (M, track lengths, unseen, outliers, noise): four members alike but for their noise (fused tail); k_tail<32> with DMMA
# (200 tracks); k_tail<16>; m <= n; no tracks
RATIOS = [1.0, "euroc", 4.0, 0.25]
MEMBERS = ([(20, shp.window_lengths(20), (1, 10), (5, 16), r) for r in RATIOS]
           + [(40, shp.n_sweep_lengths(40, 200), (), (7,), 4.0), (70, [70, 65, 33, 18, 3, 2, 1] * 3, (1, 35), (2,), 0.25),
              (8, [8, 3, 2, 1], (), (), "euroc"), (6, [], (), (), 4.0)])


@pytest.mark.parametrize("dtype", DTYPES)
def test_device_batch_of_members_with_different_noise(dtype):
    noises = [nz(r, dtype) for *_, r in MEMBERS]
    mem = [shp.twin(dtype, M, noise) for (M, *_), noise in zip(MEMBERS, noises)]
    solo = [shp.engine(dtype, M, src=m, noise=noise) for m, (M, *_), noise in zip(mem, MEMBERS, noises)]
    batch = capi.Batch(mem)
    name = np.dtype(dtype).name
    for it in range(3):  # launched directly, captured as a graph, replayed
        tracks, refs, before = [], [], []
        for i, (m, (M, lengths, unseen, outl, _), noise) in enumerate(zip(mem, MEMBERS, noises)):
            before.append(shp.state64(m))
            seed = 100 * it + (0 if i < 4 else i)  # the first four members see the same tracks
            tr = shp.sweep_tracks(np.random.default_rng(seed), before[-1][2], lengths, unseen=unseen, outliers=outl)
            tracks.append(tr)
            refs.append(shp.expect(m, tr, dtype, noise) if tr else None)
        reps = batch.update(capi.RESIDUALIZE, [shp.batch_of(t, dtype) for t in tracks], full=True)
        for i, (m, s, tr, ref, rep) in enumerate(zip(mem, solo, tracks, refs, reps)):
            label = f"{name} batch member {i} (v/u {MEMBERS[i][4]}) run {it}"
            if not tr:
                assert rep["m"] == 0 and all(np.array_equal(x, y) for x, y in zip(shp.state64(m), before[i])), label
                continue
            r1 = s.update(capi.RESIDUALIZE, shp.batch_of(tr, dtype))
            for k in ("m", "rank"):
                assert rep[k] == r1[k], (label, k, rep[k], r1[k])
            for k in ("accepted", "gamma", "valid"):
                assert np.array_equal(rep[k], r1[k]), (label, k)
            for x, y in zip(shp.state64(m) + (m.delta_x(),), shp.state64(s) + (s.delta_x(),)):
                assert np.array_equal(x, y), label
            shp.compare(m, rep, ref, tr, dtype, label, bounds)
        if it == 0:  # the same window and tracks: only the noise tells the first four members apart
            assert all(np.array_equal(a, b) for a, b in zip(before[0], before[1]))
            Ps = [shp.state64(m)[0] for m in mem[:4]]
            assert all(not np.array_equal(Ps[a], Ps[b]) for a in range(4) for b in range(a))
        assert refs[4]["m"] > 15 + 6 * 40 and refs[6]["m"] <= 15 + 6 * 8
    batch.close()


# --------------------------------------------------------------------------------------------------------------------- (f)
def landmark_scene(e, seed):
    """clone, z, p_L, landmark, Sigma_L of sets_for / scene of tests/test_landmark_map_gpu.py on the engine's window"""
    rng = np.random.default_rng(seed)
    _, _, poses = shp.state64(e)
    sets, bad = sets_for(rng, len(poses))
    return scene(rng, poses, sets, bad=bad)


def landmark_result_equal(a, b, label):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), (label, k, a[k], b[k])


def same_filter(a, b, label):
    for x, y in zip(a.state() + (a.covariance(),), b.state() + (b.covariance(),)):
        assert np.array_equal(x, y), label


@pytest.mark.parametrize("form", ["single", "iterated", "map"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_landmark_update_defaults_to_the_filters_pixel_noise(dtype, form):
    noise = nz(4.0, dtype)
    a, b = shp.twin(dtype, 12, noise), shp.twin(dtype, 12, noise)
    clone, z, p_L, lm, Sig = landmark_scene(a, 3)
    kw = {"chi2_obs": CHI2}
    if form == "iterated":
        kw.update(max_iter=4, tol=1e-12)
    if form == "map":
        kw.update(landmark=lm, Sigma_L=Sig)
    ra = a.landmark_update(clone, z, p_L, **kw)
    rb = b.landmark_update(clone, z, p_L, R=np.diag(noise), **kw)
    assert ra["applied"] == 1 and 0 < ra["used"] < len(clone), ra
    landmark_result_equal(ra, rb, form)
    same_filter(a, b, form)


@pytest.mark.parametrize("dtype", DTYPES)
def test_landmark_device_batch_reads_each_members_noise(dtype):
    """members of different pixel noise, R omitted, in one device batch: each equals its single-filter twin given its own
    R = diag(u_var, v_var)"""
    noises = [nz(r, dtype) for r in RATIOS]
    mem = [shp.twin(dtype, 12, noise) for noise in noises]
    twins = [shp.twin(dtype, 12, noise) for noise in noises]
    specs = []
    for i, m in enumerate(mem):
        clone, z, p_L, lm, Sig = landmark_scene(m, 3)  # the same observations for every member
        s = {"clone": clone, "z": z, "p_L": p_L, "chi2_obs": CHI2, "max_iter": [0, 4, 0, 4][i], "tol": 1e-12}
        if i >= 2:
            s.update(landmark=lm, Sigma_L=Sig)
        specs.append(s)
    single = [t.landmark_update(s["clone"], s["z"], s["p_L"], R=np.diag(noise), chi2_obs=s["chi2_obs"], max_iter=s["max_iter"],
                                tol=s["tol"], landmark=s.get("landmark"), Sigma_L=s.get("Sigma_L"))
              for t, s, noise in zip(twins, specs, noises)]
    batch = capi.Batch(mem)
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t) in enumerate(zip(mem, twins)):
        landmark_result_equal(got[i], single[i], f"member {i}")
        same_filter(m, t, f"member {i}")
    # members 0 and 1 (isotropic, EuRoC) saw the same observations with different noise
    assert not np.array_equal(mem[0].covariance(), mem[1].covariance())
