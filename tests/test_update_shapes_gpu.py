"""The vision update (RESIDUALIZE: k_jac onward at caller-given p_f_G) at every window, track and batch shape its kernels dispatch
on, against the dense fp64 reference of tests/vision_reference.py computed from the engine's own fetched state:
  (a) windows of 1 .. 136 clones: each tail kernel's boundary from both sides (fused <= 32 < k_tail<32> <= 63 < k_tail<16> <= 136),
      the exact and +-1 residues of the 32-tiles of c = 6M and n = 15 + 6M, tracks of 1 .. 98 observations over clone subsets;
  (b) 1 .. 512 tracks at fixed windows: every stacked row explicit (m <= n, m = n) or compressed (m = n + 1), the split-K
      chunks of the Gram products (one, a ragged last one, sixteen) and the DMMA boundary at 200 tracks;
  (c) options that act on one side of a rule only are bit-neutral on the other side: the rule sits where (a) and (b) think;
  (d) k_jac's groups of 32 / 64 / 128 threads per track are bit-identical at every track length of (a);
  (e) one device batch of members of every kind above equals its single-filter twins bit for bit and the reference, launched
      directly, captured as a graph and replayed;
  (f) 137 clones: the update fails with ERR_CAPACITY and writes nothing; pruned back to 136 it is right;
  (g) triangulation (TRIANGULATE) at the sweep's track lengths against msckf_numpy's checkMotion / initializePosition."""
import ctypes as C

import numpy as np
import pytest

from msckf_mono_b200 import capi
from oracle.msckf_numpy import MSCKF as NumpyMSCKF, CamState
from tests import vision_reference as vr
from tests.parity_cases import make_engine

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
WINDOWS = [1, 2, 3, 8, 16, 31, 32, 33, 35, 63, 64, 98, 128, 131, 136]
LENGTHS = [1, 2, 3, 17, 18, 33, 34, 65, 66, 97, 98]
# worst differences to the reference over each test's cases, measured on an H100 80GB HBM3 (700 W power limit); every case is
# asserted at 10 x these.  dx, P: max |difference| / max |reference|; state: max |difference| of the injected IMU state and clone
# poses / max |dx| (or 8 ulps of the state, where larger); gamma: max |difference| / (1 + gamma); p_f_G: max
# |difference| / |p_f_G|.
MEASURED = {"float64": {"dx": 1.24e-05, "P": 7.13e-09, "state": 1.24e-05, "gamma": 9.54e-13, "p_f_G": 3.41e-09},
            "float32": {"dx": 7.20e-04, "P": 3.83e-07, "state": 2.00e-02, "gamma": 1.21e-04, "p_f_G": 5.30e-05}}
# ceilings that separate rounding from a wrong result, whatever was measured
CONTRACT = vr.CONTRACT

_bases = {}


def engine(dtype, M, src=None, noise=None):
    """an engine (owned by a class filter it keeps alive) with the builder's M clones and pixel noise (u_var, v_var) (default
    isotropic, vr.SIGMA2), or a twin of `src` (whose state, pixel noise included, it copies)"""
    f = make_engine(dtype, max_clones=M + 1, max_tracks=64, max_obs=2048)
    f.initialize(*vr.setup(noise))
    e = capi.Engine(dtype, borrowed=f.engineHandle())
    e.filt = f
    if src is not None:
        e.copy_state_from(src)
        return e
    for k in range(M):
        if k:
            e.propagate_n(vr.readings(k))
        e.augment()
    return e


def twin(dtype, M, noise=None):
    """a fresh copy of the (cached) engine with M clones and pixel noise `noise`"""
    key = (np.dtype(dtype).name, M, noise)
    if key not in _bases:
        _bases[key] = engine(dtype, M, noise=noise)
    return engine(dtype, M, src=_bases[key], noise=noise)


def state64(e):
    imu, poses = e.state()
    return e.covariance().astype(np.float64), imu.astype(np.float64), poses.astype(np.float64)


def batch_of(tracks, dtype):
    return capi.TrackBatch(*vr.pack(tracks, dtype)[:3], dtype, vr.pack(tracks, dtype)[3])


def unseen_of(M):
    """clones no track sees: none in the small windows and at 98 (whose 98-observation track needs every clone)"""
    return () if M < 8 or M == 98 else (1, M // 2)


def sweep_tracks(rng, poses, lengths, unseen=(), outliers=()):
    """tracks of the given lengths (clamped to the clones seen); outliers only on tracks of 3 or more observations"""
    nvis = len(poses) - len(unseen)
    return vr.make_tracks(rng, poses, lengths, unseen=unseen, outliers=[j for j in outliers if min(lengths[j], nvis) >= 3])


def worst_tile(D):
    """(row, column) of the 32 x 32 tile of |D| with the largest entry"""
    i, j = np.unravel_index(np.argmax(np.abs(D)), D.shape)
    return int(i) // 32, int(j) // 32


def expect(e, tracks, dtype, noise=None):
    """the reference of an update of `e` (pixel noise `noise`, as the engine holds it) by `tracks` (as the engine receives
    them), asserting that no accept flag is within 10 % of its threshold"""
    P, imu, poses = state64(e)
    tr = vr.rounded(tracks, dtype)
    ref = vr.reference(P, imu, poses, tr, noise=noise)
    assert vr.gate_margin(ref, tr) > 0.1
    return ref


def compare(e, rep, ref, tracks, dtype, label, bounds=None, noise_floor=0.0):
    """the update's report and the engine's state after it against the reference: flags, m and rank exactly (and the rank
    pivots' gap), the numbers against CONTRACT and 10 x MEASURED (or against the (contract, measured) pair of one dtype that
    bounds(dtype name, rank above the reference's) gives); returns the numbers.  noise_floor: the rank decision's largest
    noise pivot in a plain fp64 evaluation of the same Gram form (vision_reference.gram_noise), where the model below
    underestimates it; the engine's is held to 10 x that there, and a noise pivot that lands above the threshold inside
    that band may be kept or dropped, as in fp32"""
    name = np.dtype(dtype).name
    lengths = np.array([len(t["idx"]) for t in tracks])
    assert np.array_equal(rep["accepted"].astype(bool), ref["accepted"]), (label, rep["accepted"], ref["accepted"])
    assert not rep["accepted"][lengths == 1].any(), label
    assert rep["m"] == ref["m"], (label, rep["m"], ref["m"])
    P1, imu1, poses1 = state64(e)
    got = {}
    if ref["m"] == 0:
        assert np.array_equal(P1, ref["P"]) and np.array_equal(imu1, ref["imu"]) and np.array_equal(poses1, ref["poses"]), label
        return got
    n = P1.shape[0]
    if ref["sv"] is not None:
        s = ref["sv"]
        assert np.all((s < vr.NULL_SV) | (s > vr.REAL_SV)), (label, s[(s >= vr.NULL_SV) & (s <= vr.REAL_SV)])
    # the rank decision (Gamma's relative pivots against the threshold 1e-9): the reference's rank directions are kept with
    # pivots at least two decades above everything else (fp64).  The rest is rounding noise, bounded below by a model of it;
    # the engine keeps exactly those of its noise pivots that land above the threshold (long fp64 windows: the noise of a gauge
    # direction reaches 1e-9 .. 3e-8 there, and its sign decides; fp32 filters: up to 4e-6, as large as the weakest real pivots
    # of the longest windows)
    pv = e.rank_pivots()
    assert pv.size == n, label
    pv = np.sort(pv)[::-1]
    real, null = pv[: ref["rank"]], pv[ref["rank"]:]
    noise = float(np.abs(null).max()) if null.size else 0.0
    assert real.min() > 1e-9 and (name == "float32" or real.min() > 100 * noise), (label, real.min(), noise)  # fp32: no gap
    # where the noise comes from: Gamma is a Gram matrix (the Gram form squares the conditioning of H_c), and its skip-Cholesky
    # leaves a null direction a pivot of about eps * n * cond(Gamma), cond(Gamma) ~ 1 / (smallest real pivot).  A kernel that
    # made it larger than that model allows would otherwise hide in the count of noise pivots kept below
    eps = np.finfo(np.float64 if name == "float64" else np.float32).eps  # the Jacobians are formed in the filter's type
    assert noise <= max(100 * eps * n / real.min(), 10 * noise_floor), (label, noise, real.min(), noise_floor)
    extra = int(np.sum(null > 1e-9))
    if name == "float64" and not noise_floor:
        assert rep["rank"] == ref["rank"] + extra, (label, rep["rank"], ref["rank"], noise)
    else:  # a Gamma direction kept on noise may still be dropped by its S'' pivot (fp64: within the Gram form's noise floor)
        assert ref["rank"] <= rep["rank"] <= ref["rank"] + extra, (label, rep["rank"], ref["rank"], noise)
    contract, measured = (CONTRACT[name], MEASURED[name]) if bounds is None else bounds(name, rep["rank"] - ref["rank"])
    fin = lengths >= 2
    g = rep["gamma"].astype(np.float64)[fin]
    # gamma relative where it is large, absolute where it is below 1 (a clean 2-observation track's single row can be ~1e-6:
    # fp32 cancellation there says nothing about the gate)
    got["gamma"] = float(np.max(np.abs(g - ref["gamma"][fin]) / (1 + ref["gamma"][fin]))) if fin.any() else 0.0
    dx = e.delta_x()
    assert dx.size == n, label
    scale = np.abs(ref["dx"]).max()
    got["dx"] = float(np.abs(dx - ref["dx"]).max() / scale)
    D = P1 - ref["P"]
    got["P"] = float(np.abs(D).max() / np.abs(ref["P"]).max())
    # the injected state against |dx|, or against a few ulps of the state where that is larger: an fp32 filter rounds the
    # injected p, v and q to fp32 (half an ulp of a 30 m position is 1e-6 m, more than a small update's dx)
    unit = max(scale, 8 * np.finfo(dtype).eps * max(np.abs(ref["imu"][0:19]).max(), np.abs(ref["poses"]).max()))
    got["state"] = float(max(np.abs(imu1[0:19] - ref["imu"][0:19]).max(), np.abs(poses1 - ref["poses"]).max()) / unit)
    assert np.array_equal(imu1[19:29], ref["imu"][19:29]), label  # the observability copies are not touched
    print(f"{label}: m {ref['m']} rank {rep['rank']} (reference {ref['rank']}, smallest real pivot {real.min():.1e}, "
          f"largest noise pivot {noise:.1e}) " + " ".join(f"{k} {v:.2e}" for k, v in got.items()))
    for k, v in got.items():
        where = f" worst P tile (row, column) {worst_tile(D)}" if k == "P" else ""
        assert v <= contract[k], (label, k, v, where)
        assert v <= 10 * measured[k], (label, k, v, where)
    return got


def run(e, tracks, dtype, label, noise=None, bounds=None):
    ref = expect(e, tracks, dtype, noise)
    rep = e.update(capi.RESIDUALIZE, batch_of(tracks, dtype))
    return rep, ref, compare(e, rep, ref, tracks, dtype, label, bounds)


def window_lengths(M):
    return [min(L, M) for L in LENGTHS] * 2


# --------------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", WINDOWS)
def test_window_sweep_against_the_reference(dtype, M):
    e = twin(dtype, M)
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(M), poses, window_lengths(M), unseen=unseen_of(M), outliers=(5, 16))
    rep, ref, _ = run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M}")
    if M == 1:
        assert rep["m"] == 0 and not rep["accepted"].any()
    else:
        assert ref["accepted"].sum() >= len(tracks) // 2


# --------------------------------------------------------------------------------------------------------------------- (b)
def n_sweep_lengths(M, N):
    """N track lengths at window M; "m=n" / "m=n+1": a few tracks whose rows add up to n = 15 + 6M or n + 1"""
    if N == "m=n":
        return {12: [12, 12, 12, 12, 3], 33: [33, 33, 33, 12, 3]}[M]
    if N == "m=n+1":
        return {12: [12, 12, 12, 10, 4, 3], 33: [33, 33, 33, 12, 3, 2]}[M]
    cyc = [M, M - 1, 3, 2, M // 2, M]
    return [cyc[j % len(cyc)] for j in range(N)]


N_CASES = [(dt, M, N) for M in (12, 33) for N in (1, 2, 31, 32, 63, 64, 65, 199, 200, 511, 512, "m=n", "m=n+1") for dt in DTYPES
           if dt == np.float64 or N in (199, 200, 512)]


@pytest.mark.parametrize("dtype,M,N", N_CASES)
def test_track_count_sweep_against_the_reference(dtype, M, N):
    e = twin(dtype, M)
    n = 15 + 6 * M
    _, _, poses = state64(e)
    lengths = n_sweep_lengths(M, N)
    outl = () if isinstance(N, str) else tuple(j for j in range(7, len(lengths), 50))
    tracks = sweep_tracks(np.random.default_rng(1000 + M), poses, lengths, outliers=outl)
    rep, ref, _ = run(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} N={N}")
    if N == "m=n":
        assert ref["m"] == n and rep["rank"] == n  # every stacked row explicit: the square Q of the reference
    if N == "m=n+1":
        assert ref["m"] == n + 1 and ref["sv"] is not None  # the first compressed system


# --------------------------------------------------------------------------------------------------------------------- (c)
def option_twins(M, lengths, options, seed):
    """(per option setting: report, P, dx, state) of twins updated by the same tracks, the reference and the tracks"""
    out = []
    for opt in options:
        e = twin(np.float64, M)
        for k, v in opt.items():
            e.set_option(k, v)
        _, _, poses = state64(e)
        tracks = sweep_tracks(np.random.default_rng(seed), poses, lengths, outliers=(5,))
        rep, ref, _ = run(e, tracks, np.float64, f"M={M} N={len(lengths)} options {opt}")
        out.append((rep, e.covariance(), e.delta_x(), e.state()))
    return out


def same_bits(a, b):
    (ra, Pa, dxa, sa), (rb, Pb, dxb, sb) = a, b
    return (np.array_equal(ra["gamma"], rb["gamma"]) and np.array_equal(Pa, Pb) and np.array_equal(dxa, dxb)
            and all(np.array_equal(x, y) for x, y in zip(sa, sb)))


@pytest.mark.parametrize("M", [32, 33, 63, 64, 136])
def test_tail_options_act_on_fused_windows_only(M):
    """option 3 = 0 (separate substitution) and option 7 = 1 (one chain CTA) change only the fused tail (M <= 32)"""
    out = option_twins(M, [min(L, M) for L in LENGTHS] * 2, [{}, {3: 0.0}, {7: 1.0}], seed=M)
    for o in out[1:]:
        assert same_bits(out[0], o) == (M > 32), M


@pytest.mark.parametrize("N", [199, 200])
def test_simt_gram_option_acts_from_200_tracks_only(N):
    """option 5 = 0 (SIMT Gram tiles) changes nothing below 200 tracks, where the Gram products run on SIMT anyway"""
    out = option_twins(12, n_sweep_lengths(12, N), [{}, {5: 0.0}], seed=N)
    assert same_bits(out[0], out[1]) == (N < 200)


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [40, 70, 98])
def test_jac_group_sizes_are_bit_identical_at_every_track_length(dtype, M):
    """k_jac with 32, 64 and 128 threads per track (option 6) at every track length of the sweep: M = 40 (lengths up to 34) and
    M = 70 (up to 66) run the requested group in both dtypes; M = 98 adds the 97- and 98-observation tracks, whose groups do
    not fit twice in a CTA's shared memory in fp64, so the engine widens the group there (asserted: the widened launch is the
    one compared)"""
    lengths = [L for L in LENGTHS if L <= M] * 2
    out = []
    for g in (128, 64, 32):
        e = twin(dtype, M)
        e.set_option(6, float(g))
        _, _, poses = state64(e)
        tracks = sweep_tracks(np.random.default_rng(M), poses, lengths, outliers=(5,))
        rep = e.update(capi.RESIDUALIZE, batch_of(tracks, dtype))
        used = e.jac_group()
        if M < 98:
            assert used == g, (M, g, used)
        else:
            assert used >= g and (used == 128 or dtype == np.float32), (M, g, used)
        out.append((rep, e.covariance(), e.delta_x(), e.state()))
    assert out[0][0]["accepted"].sum() > len(lengths) // 2
    for o in out[1:]:
        assert np.array_equal(out[0][0]["accepted"], o[0]["accepted"]) and same_bits(out[0], o)


# --------------------------------------------------------------------------------------------------------------------- (e)
# (M, track lengths, unseen, outliers): fused with 199 tracks (SIMT Gram, 6 splits); k_tail<32> with 200 (DMMA); k_tail<16>
# with 20 tracks (one split); 512 tracks (16 splits); m <= n; no tracks; every track gated out; a 98-observation track (k_jac's
# group widened for every member)
MEMBERS = [(12, n_sweep_lengths(12, 199), (), (7, 57)), (40, n_sweep_lengths(40, 200), (), (7,)),
           (70, [70, 65, 33, 18, 3, 2, 1] * 3, (1, 35), (2,)), (12, n_sweep_lengths(12, 512), (), (7,)),
           (8, [8, 3, 2, 1], (), ()), (6, [], (), ()), (16, [16, 9, 5], (), (0, 1, 2)), (98, [98, 97, 66, 34, 3, 2], (), ())]


@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_shape_device_batch(dtype):
    mem = [twin(dtype, M) for M, *_ in MEMBERS]
    solo = [engine(dtype, M, src=m) for m, (M, *_) in zip(mem, MEMBERS)]
    batch = capi.Batch(mem)
    name = np.dtype(dtype).name
    for it in range(3):  # the same launch shape three times: launched directly, captured as a graph, replayed
        tracks, refs, before = [], [], []
        for i, (m, (M, lengths, unseen, outl)) in enumerate(zip(mem, MEMBERS)):
            before.append(state64(m))
            tr = sweep_tracks(np.random.default_rng(100 * it + i), before[-1][2], lengths, unseen=unseen, outliers=outl)
            tracks.append(tr)
            refs.append(expect(m, tr, dtype) if tr else None)
        bs = [batch_of(t, dtype) for t in tracks]
        reps = batch.update(capi.RESIDUALIZE, bs, full=True)
        for i, (m, s, tr, ref, rep) in enumerate(zip(mem, solo, tracks, refs, reps)):
            label = f"{name} batch member {i} run {it}"
            if not tr:
                assert rep["m"] == 0 and all(np.array_equal(x, y) for x, y in zip(state64(m), before[i])), label
                continue
            r1 = s.update(capi.RESIDUALIZE, batch_of(tr, dtype))
            for k in ("m", "rank"):
                assert rep[k] == r1[k], (label, k, rep[k], r1[k])
            for k in ("accepted", "gamma", "valid"):
                assert np.array_equal(rep[k], r1[k]), (label, k)
            for x, y in zip(state64(m) + (m.delta_x(),), state64(s) + (s.delta_x(),)):
                assert np.array_equal(x, y), label
            compare(m, rep, ref, tr, dtype, label)
        assert refs[6]["m"] == 0 and not reps[6]["accepted"].any()
    batch.close()


# --------------------------------------------------------------------------------------------------------------------- (f)
def counters(e):
    c = (C.c_longlong * 8)()
    capi.check(capi.lib().msckf_b200_get_counters(e.h, c), "msckf_b200_get_counters")
    return list(c)


def test_window_of_137_clones_fails_and_writes_nothing():
    e = twin(np.float64, 137)
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(137), poses, window_lengths(137), unseen=unseen_of(137))
    before = state64(e) + (counters(e), e.launch_count(), e.rank_pivots())
    with pytest.raises(RuntimeError, match="rc=-2"):
        e.update(capi.RESIDUALIZE, batch_of(tracks, np.float64))
    after = state64(e) + (counters(e), e.launch_count(), e.rank_pivots())
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    e.prune(np.arange(1, 137))
    assert e.num_clones() == 136
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(136), poses, window_lengths(136), unseen=unseen_of(136), outliers=(5, 16))
    run(e, tracks, np.float64, "float64 M=137 pruned to 136")


# --------------------------------------------------------------------------------------------------------------------- (g)
@pytest.mark.parametrize("dtype", DTYPES)
def test_triangulation_at_the_sweep_track_lengths(dtype):
    """k_tri (4 tracks per CTA; 23 tracks: a ragged last CTA) against msckf_numpy's checkMotion / initializePosition on the
    same poses and observations, in the same precision"""
    M = 98
    e = twin(dtype, M)
    P0, imu, poses = state64(e)
    lengths = [LENGTHS[j % len(LENGTHS)] for j in range(23)]
    tracks = vr.make_tracks(np.random.default_rng(5), poses, lengths, offset=0.0)
    rep = e.update(capi.TRIANGULATE, capi.TrackBatch(*vr.pack(tracks, dtype)[:3], dtype))
    assert np.array_equal(state64(e)[0], P0)
    f = NumpyMSCKF(dtype)
    S = f.S
    params = vr.setup()[2]
    f.params = {"translation_threshold": S(params["translation_threshold"]), "max_gn_cost_norm": S(params["max_gn_cost_norm"])}
    raw = e.state()[1]
    cams = [CamState(p[0:3].copy(), p[3:7].copy(), 0.0, k) for k, p in enumerate(raw)]
    name = np.dtype(dtype).name
    worst = 0.0
    for j, t in enumerate(tracks):
        if len(t["idx"]) < 2:
            assert rep["cm_ok"][j] == 0 and rep["tri_ok"][j] == 0, j
            continue
        cs = [cams[k] for k in t["idx"]]
        obs = [o for o in t["obs"].astype(dtype)]
        assert rep["cm_ok"][j] == int(f._check_motion(obs[0], cs)), j
        ok, p = f._initialize_position(cs, obs)
        assert rep["tri_ok"][j] == int(ok) and ok, j
        worst = max(worst, float(np.abs(rep["p_f_G"][j].astype(np.float64) - p).max() / np.linalg.norm(p)))
    print(f"{name} triangulation: p_f_G {worst:.2e}")
    assert worst <= CONTRACT[name]["p_f_G"] and worst <= 10 * MEASURED[name]["p_f_G"]
