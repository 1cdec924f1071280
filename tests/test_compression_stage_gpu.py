"""The compression stage on its own (k_blockdiag, k_gram / k_gram_mma, k_assemble, k_rows; DESIGN.md 4.4): every update here
runs RESIDUALIZE at caller-given p_f_G with option 8 set, so it stops once T'', R'', r'' are written, and reads them and the
stage's inputs back (msckf_b200_stage_buffer).  Every case checks
  * that every entry of T'', R'', r'' is finite: option 8 fills the stage's workspaces with NaN first, so an element a kernel
    reads without any kernel having written it shows up;
  * the Gram block (Lambda, Psi), beta and the explicit rows against tests/compression_reference.same_operation, entry by
    entry: |engine - reference| <= gamma_k * scale (k: the entry's summation depth), and kappa = max |engine - reference| /
    (u * scale) within 10 x the value measured (MEASURED_KAPPA); where the scale is 0 (a structural zero the code writes) the
    entry is exactly 0;
  * the whole n x n result against tests/compression_reference.basis_free (from tests/vision_reference.py's per-track
    H_o,j, r_o,j, A_j): max |engine - reference| / max |reference| within 10 x MEASURED_BASIS_FREE and below
    BASIS_FREE_CEILING, and exactly 0 at the structural zeros;
  * P, the state and delta-x unchanged, bit for bit, and the report's rank 0.
Grid: (a) windows of 2 .. 16 clones (c = 6M: every even width of the last 32-tile), 31 .. 33, 64, 98, 133, 136, each with ~30
tracks (SIMT Gram tiles), 200 tracks (DMMA) and 200 tracks with option 5 = 0 (SIMT); (b) 1 .. 600 tracks at M = 12 and 33 (one
split, a ragged last chunk, nsplit recomputed below the cap, 16 splits), each plan asserted through the host's mirror; (c) the
row cases: m = 0 with tracks, m < n, m = n, m = n + 1, and every explicit-row layout of vision_reference.HEAD_CASES at isotropic
and anisotropic pixel noise; (d) the symmetries the code guarantees bit for bit; (e) one device batch of every kind above,
launched, captured and replayed, member by member equal to its single-filter twin."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import compression_reference as cr
from tests import vision_reference as vr
from tests.test_update_shapes_gpu import engine, n_sweep_lengths, state64, sweep_tracks, twin

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
STOP = 8  # option 8: stop after the compression
# worst values over the grid, measured on an H100 80GB HBM3 (700 W power limit); each case is asserted at 10 x these.
# kappa: max |engine - same-operation reference| / (u scale), u = 2^-53, in the Gram block and beta ("gram") and in the explicit
# rows and their R'' coupling ("head"); the same in both filter precisions (every sum of the stage is fp64)
MEASURED_KAPPA = {"gram": 9.17, "head": 19.8}
# max |engine - basis-free reference| / max |reference| of T'', R'', r'', over their explicit rows and over the others apart, per
# filter precision (the Jacobians are formed in it)
MEASURED_BASIS_FREE = {"float64": 3.45e-13, "float32": 4.76e-4}
# ceilings that separate rounding from a wrong result, whatever was measured
BASIS_FREE_CEILING = {"float64": 1e-8, "float32": 1e-2}
NAMES = ("T2", "R2", "r2", "Z", "Yq", "ur", "D1", "D2", "bb", "Xg", "rg", "Vg", "taug", "accept", "row_off")


def batch_of(tracks, dtype):
    off, obs, idx, pfg = vr.pack(tracks, dtype)
    return capi.TrackBatch(off, obs, idx, dtype, pfg)


def buffers(e):
    return {k: e.stage_buffer(k) for k in NAMES}


def check_stage(e, tracks, dtype, label, noise=None):
    """the stage's outputs of e after an update by `tracks` (option 8 set) against both references; returns the buffers"""
    name = np.dtype(dtype).name
    u_var, v_var = noise if noise is not None else vr.pixel_noise(1.0, dtype)
    b = buffers(e)
    M = (b["T2"].shape[0] - 15) // 6
    n = 15 + 6 * M
    for k in ("T2", "R2", "r2"):
        assert np.isfinite(b[k]).all(), (label, k, np.argwhere(~np.isfinite(b[k]))[:5])
    off, _, idx, _ = vr.pack(tracks, dtype)
    nsplit = cr.split_plan(len(tracks))[0]
    so = cr.same_operation(b, off, idx, u_var, v_var, M, nsplit)
    kap = {}
    for k, s, d in (("T2", "sT", "kT"), ("R2", "sR", "kR"), ("r2", "sr", "kr")):
        bad = cr.within_gamma(b[k], so[k], so[s], so[d])
        assert bad.size == 0, (label, k, "outside gamma_k * scale at", bad[:5].tolist())
    # (a scale of 0 makes the bound above an exact zero: T'' columns < 15 below the head, rows >= m when m <= n, clones no
    # accepted track sees, ...)
    for region in ("gram", "head"):
        vals = [cr.kappa(b["T2"], so["T2"], so["sT"], so[region]), cr.kappa(b["R2"], so["R2"], so["sR"], so[region]),
                cr.kappa(b["r2"], so["r2"], so["sr"], so[region + "_rows"])]
        kap[region] = max(vals)
    # basis-free
    P, imu, poses = state64(e)
    tr = vr.rounded(tracks, dtype)
    blocks = vr.project_tracks(imu, poses, tr)
    gam, acc = vr.gate(P, blocks, tr, u_var)
    assert np.array_equal(acc, b["accept"].astype(bool)), (label, acc, b["accept"])
    assert vr.gate_margin({"gamma": gam}, tr) > 0.1, label
    bf = cr.basis_free(blocks, acc, u_var, v_var, n, head_bases={j: Q[:, 3:] for j, Q in so["Q"].items()})
    worst = 0.0
    for got, ref, s in zip((b["T2"], b["R2"], b["r2"]), bf[:3], bf[3:]):
        assert np.all(got[s == 0] == 0), (label, "structural zero", np.argwhere((s == 0) & (got != 0))[:5].tolist())
        for rows in (so["head_rows"], ~so["head_rows"]):  # the explicit rows (~|X|) and the Gram rows (~|X|^2) apart
            if np.abs(ref[rows]).max(initial=0) > 0:
                worst = max(worst, float(np.abs(got[rows] - ref[rows]).max() / np.abs(ref[rows]).max()))
    print(f"{label}: m {so['m']} n {n} nsplit {nsplit} kappa gram {kap['gram']:.1f} head {kap['head']:.1f} basis-free {worst:.2e}")
    assert worst <= BASIS_FREE_CEILING[name], (label, worst)
    assert worst <= 10 * MEASURED_BASIS_FREE[name], (label, worst)
    for region, v in kap.items():
        assert v <= 10 * MEASURED_KAPPA[region], (label, region, v)
    return b, so


def stage_update(e, tracks, dtype, label, noise=None):
    """one update with option 8: P, the state and delta-x are left as they were, the rank is 0; then check_stage"""
    e.set_option(STOP, 1.0)
    before = state64(e) + (e.delta_x(),)
    rep = e.update(capi.RESIDUALIZE, batch_of(tracks, dtype))
    after = state64(e) + (e.delta_x(),)
    for x, y in zip(before, after):
        assert np.array_equal(x, y), label
    assert rep["rank"] == 0, label
    b, so = check_stage(e, tracks, dtype, label, noise)
    assert rep["m"] == so["m"] and np.array_equal(rep["accepted"], b["accept"]), label
    return rep, b, so


def cyc_lengths(M, N):
    cyc = [M, M - 1, 3, 2, M // 2, M]
    return [max(1, min(cyc[j % len(cyc)], M, 98)) for j in range(N)]  # (98: the longest track)


# --------------------------------------------------------------------------------------------------------------------- (a)
WINDOWS = list(range(2, 17)) + [31, 32, 33, 64, 98, 133, 136]
KINDS = {"simt30": (30, True), "dmma200": (200, True), "simt200": (200, False)}


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", WINDOWS)
def test_windows(M, dtype, kind):
    N, opt5 = KINDS[kind]
    e = twin(dtype, M)
    e.set_option(5, 1.0 if opt5 else 0.0)
    _, _, poses = state64(e)
    unseen = () if M < 8 or M == 98 else (1, M // 2)
    tracks = sweep_tracks(np.random.default_rng(M), poses, cyc_lengths(M, N), unseen=unseen, outliers=(5,))
    _, b, so = stage_update(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} {kind}")
    assert (so["m"] > 15 + 6 * M or M == 2) and cr.dmma(N, opt5) == (kind == "dmma200")


# --------------------------------------------------------------------------------------------------------------------- (b)
# N -> its split-K plan (nsplit, kchunk, depth of the last chunk), as the host picks it: one chunk shorter than a k-slab (1, 2),
# one chunk of 93 .. 99 rows (31 .. 33: a ragged last k-slab), two splits (64, 65), the DMMA edge (199, 200), nsplit recomputed
# below the cap (511: 14, 530: 15), sixteen splits (512), and a last chunk shorter than one k-slab (600)
PLANS = {1: (1, 16, 3), 2: (1, 16, 6), 31: (1, 96, 93), 32: (1, 96, 96), 33: (1, 112, 99), 64: (2, 96, 96), 65: (2, 112, 83),
         199: (6, 112, 37), 200: (6, 112, 40), 511: (14, 112, 77), 512: (16, 96, 96), 530: (15, 112, 22), 600: (15, 128, 8)}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [12, 33])
@pytest.mark.parametrize("N", list(PLANS))
def test_track_counts(N, M, dtype):
    plan = cr.split_plan(N)
    assert plan == PLANS[N], (N, plan)
    e = twin(dtype, M)
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(1000 + M + N), poses, n_sweep_lengths(M, N),
                          outliers=tuple(range(7, N, 50)))
    stage_update(e, tracks, dtype, f"{np.dtype(dtype).name} M={M} N={N} plan {plan}")


# --------------------------------------------------------------------------------------------------------------------- (c)
ROWS = {"m=0 (one observation each)": (1, [1] * 5, ()), "m=0 (every track gated)": (16, [16, 9, 5], (0, 1, 2)),
        "m<n": (8, [8, 3, 2, 1], ()), "m=n": (12, n_sweep_lengths(12, "m=n"), ()), "m=n+1": (12, n_sweep_lengths(12, "m=n+1"), ())}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(ROWS))
def test_row_cases(case, dtype):
    M, lengths, outl = ROWS[case]
    e = twin(dtype, M)
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(7), poses, lengths, outliers=outl)
    rep, b, so = stage_update(e, tracks, dtype, f"{np.dtype(dtype).name} {case}")
    n = 15 + 6 * M
    want = {"m=n": n, "m=n+1": n + 1}.get(case)
    if case.startswith("m=0"):
        assert rep["m"] == 0 and not b["T2"].any() and not b["R2"].any() and not b["r2"].any()
    elif case == "m<n":
        assert 0 < rep["m"] < n
    else:
        assert rep["m"] == want


@pytest.mark.parametrize("ratio", [1.0, 4.0, "euroc"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", vr.HEAD_CASES)
def test_head_rows(case, dtype, ratio):
    """the explicit rows' layouts across track edges; anisotropic noise (isotropic noise hides a swapped u_var / v_var)"""
    M = 20
    noise = vr.pixel_noise(ratio, dtype)
    e = engine(dtype, M, noise=noise)
    _, _, poses = state64(e)
    lengths, outl = vr.head_lengths(case, M)
    tracks = vr.make_tracks(np.random.default_rng(11), poses, lengths, outliers=outl)
    rep, b, so = stage_update(e, tracks, dtype, f"{np.dtype(dtype).name} {case} ratio {ratio}", noise=noise)
    assert rep["m"] > 15 + 6 * M and (case != "gated" or not b["accept"][1])


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("opt5", [1.0, 0.0])
@pytest.mark.parametrize("M", [12, 33, 136])
def test_symmetry_the_code_guarantees(M, opt5):
    """Bit for bit, as the sources guarantee it:
      * R'''s coupling: k_rows writes R''(h, 15 + col) and R''(15 + col, h) from one value;
      * a mirror entry (tile ta < tb) takes the same split sums as its entry (k_assemble), and sum X^T X per clone is bitwise
        symmetric (k_blockdiag adds x_p x_q and x_q x_p, the same products): T''(a, b) == T''(b, a) in every off-diagonal tile
        pair, R''(a, b) == R''(b, a) there where a and b belong to different clones (sum X^T D X multiplies by d first, so its
        (p, q) and (q, p) may differ in the last bit);
      * the SIMT Gram tiles (option 5 = 0) form Z^T Z's (i, j) and (j, i) of a diagonal tile from the same products in the same
        order: T'' is bitwise symmetric there too.  The DMMA form and G2 (Z^T Yq + Yq^T Z, added in opposite orders) carry no
        such guarantee: there only the rounding bound of check_stage holds"""
    e = twin(np.float64, M)
    e.set_option(5, opt5)
    _, _, poses = state64(e)
    tracks = sweep_tracks(np.random.default_rng(3), poses, cyc_lengths(M, 200), unseen=(1, M // 2), outliers=(5,))
    _, b, so = stage_update(e, tracks, np.float64, f"symmetry M={M} option 5 = {opt5}")
    T2, R2 = b["T2"], b["R2"]
    assert np.array_equal(R2[:15, 15:], R2[15:, :15].T)
    c = 6 * M
    a = np.arange(c)
    tile, clone = a // cr.K["GT"], a // 6
    off_tile = tile[:, None] != tile[None, :]
    G, H = T2[15:, 15:], R2[15:, 15:]
    assert np.array_equal(G[off_tile], G.T[off_tile])
    other = off_tile & (clone[:, None] != clone[None, :])
    assert np.array_equal(H[other], H.T[other])
    if opt5 == 0.0:
        assert np.array_equal(G, G.T)
    # the straddling clone blocks exist at this window (6 x 6 blocks across a 32-tile edge), or the test says nothing of them
    assert (off_tile & (clone[:, None] == clone[None, :])).any() == (c > cr.K["GT"])


# --------------------------------------------------------------------------------------------------------------------- (e)
# (M, track lengths, option 5): 1 tile / 1 split (SIMT); 26 tiles, DMMA; 16 splits, DMMA; 15 splits with a last chunk 8 deep,
# SIMT; m <= n; no tracks
MEMBERS = [(2, cyc_lengths(2, 30), 1.0), (136, cyc_lengths(136, 200), 1.0), (12, n_sweep_lengths(12, 512), 1.0),
           (33, n_sweep_lengths(33, 600), 0.0), (8, [8, 3, 2, 1], 1.0), (6, [], 1.0)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_device_batch(dtype):
    name = np.dtype(dtype).name
    mem = [twin(dtype, M) for M, *_ in MEMBERS]
    solo = [engine(dtype, M, src=m) for m, (M, *_) in zip(mem, MEMBERS)]
    for m, s, (_, _, o5) in zip(mem, solo, MEMBERS):
        for x in (m, s):
            x.set_option(5, o5)
            x.set_option(STOP, 1.0)
    batch = capi.Batch(mem)
    for it in range(3):  # the same launch shape three times: launched directly, captured as a graph, replayed
        tracks = [sweep_tracks(np.random.default_rng(100 * it + i), state64(m)[2], L, outliers=(5,) if len(L) > 5 else ())
                  for i, (m, (M, L, _)) in enumerate(zip(mem, MEMBERS))]
        before = [state64(m) + (m.delta_x(),) for m in mem]
        reps = batch.update(capi.RESIDUALIZE, [batch_of(t, dtype) for t in tracks])
        for i, (m, s, tr, rep) in enumerate(zip(mem, solo, tracks, reps)):
            label = f"{name} batch member {i} run {it}"
            for x, y in zip(before[i], state64(m) + (m.delta_x(),)):
                assert np.array_equal(x, y), label
            assert rep["rank"] == 0, label
            if not tr:  # the stage wrote nothing for it
                assert rep["m"] == 0 and m.stage_buffer("T2") is None, label
                continue
            s.update(capi.RESIDUALIZE, batch_of(tr, dtype))
            bm, bs = buffers(m), buffers(s)
            # (k_jac writes no Jacobian, residual or reflector for a track of one observation: those entries are left over)
            L = np.array([len(t["idx"]) for t in tr])
            valid = {"Xg": np.repeat(L >= 2, L), "rg": np.repeat(L >= 2, L), "Vg": np.repeat(L >= 2, 2 * L), "taug": L >= 2}
            for k in NAMES:
                x, y = (bm[k][valid[k]], bs[k][valid[k]]) if k in valid else (bm[k], bs[k])
                assert np.array_equal(x, y), (label, k)
            check_stage(m, tr, dtype, label)
    assert reps[4]["m"] <= 15 + 6 * 8
    batch.close()


def test_batch_members_must_agree_on_the_stop():
    """a batch whose members disagree on option 8 is refused at stage time, and nothing is written"""
    a, b = twin(np.float64, 12), twin(np.float64, 12)
    a.set_option(STOP, 1.0)
    batch = capi.Batch([a, b])
    tracks = [sweep_tracks(np.random.default_rng(i), state64(x)[2], cyc_lengths(12, 20)) for i, x in enumerate((a, b))]
    before = [state64(x) + (x.delta_x(), x.launch_count()) for x in (a, b)]
    with pytest.raises(RuntimeError, match="rc=-3"):
        batch.update(capi.RESIDUALIZE, [batch_of(t, np.float64) for t in tracks])
    for x, bf in zip((a, b), before):
        for p, q in zip(bf, state64(x) + (x.delta_x(), x.launch_count())):
            assert np.array_equal(p, q)
    b.set_option(STOP, 1.0)
    batch.update(capi.RESIDUALIZE, [batch_of(t, np.float64) for t in tracks])
    batch.close()


def test_the_stop_never_leaks_into_a_full_update():
    """a graph captured with option 8 never replays without it, nor the reverse: after three stopped updates (launched,
    captured, replayed), which change nothing, three full ones launch what a twin that never set the option launches and end
    where it ends, bit for bit"""
    M = 12
    ref, e = twin(np.float64, M), twin(np.float64, M)
    tracks = sweep_tracks(np.random.default_rng(5), state64(ref)[2], cyc_lengths(M, 40), outliers=(5,))
    n0 = ref.launch_count()
    for _ in range(3):
        ref.update(capi.RESIDUALIZE, batch_of(tracks, np.float64))
    e.set_option(STOP, 1.0)
    for _ in range(3):
        stage_update(e, tracks, np.float64, "stopped")
    e.set_option(STOP, 0.0)
    n1 = e.launch_count()
    for _ in range(3):
        e.update(capi.RESIDUALIZE, batch_of(tracks, np.float64))
    assert e.launch_count() - n1 == ref.launch_count() - n0
    for x, y in zip(state64(e) + (e.delta_x(),), state64(ref) + (ref.delta_x(),)):
        assert np.array_equal(x, y)

