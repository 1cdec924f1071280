"""The vision update's chi-square gate in k_jac (RESIDUALIZE at caller-given p_f_G) on both sides of its threshold, and when its
Cholesky fails, against the dense fp64 reference of tests/vision_reference.py:
  (a) every track length 2 .. 98, one track just below and one just above CHI2[L] (vision_reference.threshold_tracks: 1e-9 of
      the threshold in fp64, 0.4 x the gap to the neighbouring entry in fp32), k_jac's groups of 32 / 64 / 128 threads per track
      (option 6) bit-identical: a gate reading a neighbouring entry, a mis-rounded entry or another table flips a flag;
  (b) one device batch of members carrying (a)'s tracks equals its single-filter twins bit for bit and gates as designed,
      launched directly, captured as a graph and replayed;
  (c) a clone block of P made strongly negative: the tracks that see it (first, or from the second panel of the gate Cholesky
      on, up to the last observation of a 98-observation track) report gamma = 1e30 and are rejected, their CTA neighbours and
      every other track are unaffected, in a filter and as the broken member of a device batch.  This is the non-positive
      pivot of M = Y + u_var I; the other branch of the same failure path, a non-positive pivot of B^T B (the gate's 3 x 3
      factor, feature_kernels.cuh), is not covered: no track with a positive definite M makes B^T B singular;
  (d) a track's observations in any order gate and update like the ascending ones;
  (e) a track that names one clone twice is refused before anything runs (MSCKF sees a feature once per image);
  (f) a track of 99 observations is refused before anything runs.
Accepted and rejected tracks alternate, pairs in both orders, so that at 32 and 64 threads per track (two tracks per CTA) each
CTA holds one of each.

compare()'s model of the rank decision's noise pivots (100 eps n / smallest real pivot) underestimates the noise of the Gram
form itself on some of these windows: a plain fp64 evaluation of the same formula (vision_reference.gram_noise) reaches 3e-9
where the model allows 6.6e-10 (130 tracks over 70 clones, smallest real pivot 1.45e-2; the engine 4.8e-9 on the same
tracks).  In fp64 the engine's noise pivots are held to 10 x that evaluation where it is the larger, and a noise pivot in
that band above the rank threshold (1.45e-9 on a device-batch member of (b)) is kept as rank or dropped by its S'' pivot,
as compare() allows in fp32: the rank is then between the reference's and the reference's plus those pivots."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import vision_reference as vr
from tests.test_update_shapes_gpu import batch_of, compare, counters, engine, same_bits, state64, twin

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
GROUPS = (128, 64, 32)
# (window, track lengths): every group runs as requested on 70 clones; the longest tracks need 98
WINDOWS = [(70, list(range(2, 67))), (98, list(range(67, 99)))]
# worst differences to the reference over (a) .. (d), measured on an H100 80GB HBM3 (700 W power limit); asserted at 10 x these
# and at vision_reference.CONTRACT.  Measures as in tests/test_update_shapes_gpu.py
MEASURED = {"float64": {"dx": 3.61e-07, "P": 7.48e-10, "state": 3.61e-07, "gamma": 1.06e-13},
            "float32": {"dx": 9.94e-05, "P": 2.55e-07, "state": 1.72e-04, "gamma": 3.71e-05}}
CONTRACT = vr.CONTRACT


def bounds(name, extra):
    return CONTRACT[name], MEASURED[name]


def threshold_pairs(e, lengths, dtype, seed):
    """(tracks, design flags) of vision_reference.threshold_pairs at e's state"""
    P, imu, poses = state64(e)
    tracks, _, _, sides = vr.threshold_pairs(np.random.default_rng(seed), P, imu, poses, lengths, dtype)
    return tracks, sides < 0


def checked(e, rep, ref, tracks, dtype, label, imu, poses, floor=None):
    """compare() with the fp64 Gram form's own noise floor (module docstring); returns the floor"""
    if floor is None:
        floor = vr.gram_noise(imu, poses, tracks, ref) if dtype == np.float64 else 0.0
    compare(e, rep, ref, tracks, dtype, label, bounds, noise_floor=floor)
    return floor


def check_group(e, M, g, dtype):
    used = e.jac_group()
    if M <= 70:
        assert used == g, (M, g, used)
    else:  # the longest tracks' groups do not fit twice in a CTA's shared memory in fp64: the engine widens them
        assert used >= g and (used == 128 or dtype == np.float32), (M, g, used)


def outcome(e, rep):
    return rep, e.covariance(), e.delta_x(), e.state()


# --------------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("M,lengths", WINDOWS, ids=["M70", "M98"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_gate_on_both_sides_of_every_threshold(dtype, M, lengths):
    tracks = want = ref = floor = None
    out = []
    for g in GROUPS:
        e = twin(dtype, M)
        e.set_option(6, float(g))
        if tracks is None:
            tracks, want = threshold_pairs(e, lengths, dtype, M)
            _, imu, poses = st = state64(e)
            ref = vr.reference(*st, tracks)
            assert np.array_equal(ref["accepted"], want)
        rep = e.update(capi.RESIDUALIZE, batch_of(tracks, dtype))
        check_group(e, M, g, dtype)
        label = f"{np.dtype(dtype).name} M={M} group {g}"
        assert np.array_equal(rep["accepted"].astype(bool), want), (label, np.flatnonzero(rep["accepted"].astype(bool) != want))
        floor = checked(e, rep, ref, tracks, dtype, label, imu, poses, floor)
        out.append(outcome(e, rep))
    for o in out[1:]:
        assert same_bits(out[0], o)


# --------------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("windows", [(70, 98), (70, 70)], ids=["70+98", "70+70"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_threshold_device_batch(dtype, windows):
    """(70, 98): the 98-observation tracks widen the batch's groups in fp64; (70, 70): two tracks per CTA"""
    lens = dict(WINDOWS)
    mem = [twin(dtype, M) for M in windows]
    solo = [engine(dtype, M, src=m) for m, M in zip(mem, windows)]
    batch = capi.Batch(mem)
    name = np.dtype(dtype).name
    for it in range(3):  # the same launch shape three times: launched directly, captured as a graph, replayed
        tracks, wants, before = [], [], []
        for i, (m, M) in enumerate(zip(mem, windows)):
            tr, want = threshold_pairs(m, lens[M], dtype, 10 * it + i)
            tracks.append(tr); wants.append(want); before.append(state64(m))
        reps = batch.update(capi.RESIDUALIZE, [batch_of(t, dtype) for t in tracks], full=True)
        for i, (m, s, tr, want, rep, st) in enumerate(zip(mem, solo, tracks, wants, reps, before)):
            label = f"{name} batch member {i} (M={windows[i]}) run {it}"
            r1 = s.update(capi.RESIDUALIZE, batch_of(tr, dtype))
            for k in ("m", "rank"):
                assert rep[k] == r1[k], (label, k, rep[k], r1[k])
            for k in ("accepted", "gamma", "valid"):
                assert np.array_equal(rep[k], r1[k]), (label, k)
            for x, y in zip(state64(m) + (m.delta_x(),), state64(s) + (s.delta_x(),)):
                assert np.array_equal(x, y), label
            assert np.array_equal(rep["accepted"].astype(bool), want), label
            ref = vr.reference(*st, tr)
            assert np.array_equal(ref["accepted"], want), label
            checked(m, rep, ref, tr, dtype, label, *st[1:])
    batch.close()


# --------------------------------------------------------------------------------------------------------------------- (c)
def track_on(rng, poses, idx):
    """a clean track over the clones idx (in this order), its landmark in front of the middle one"""
    idx = np.asarray(idx, dtype=np.int32)
    p = vr.landmark(rng, poses[idx[len(idx) // 2]])
    obs = np.array([vr.project(poses[k], p)[1] for k in idx]) + np.sqrt(vr.SIGMA2) / 10 * rng.normal(size=(len(idx), 2))
    return {"idx": idx, "obs": obs, "pfg": p}


# (window, broken clone, clone lists of the tracks that see it): at 70 clones the broken clone first (the bad pivot in the
# gate Cholesky's first panel of 8 rows) or at observation 4, 7, 8, 20, 40 (a later panel; 40: the last one of its track);
# at 98 clones at observation 4 of 5 and 47 of 48, and last of the 98-observation track
BROKEN = {70: (40, [np.arange(40, 40 + L) for L in (2, 3, 8, 17, 30)]
                   + [np.arange(40 - p, 40 - p + L) for p, L in ((4, 5), (4, 12), (7, 20), (8, 9), (20, 33), (40, 41))]),
          98: (97, [np.arange(93, 98), np.arange(50, 98), np.arange(98)])}


def broken_case(e, M, dtype, seed):
    """breaks e's clone block (P_kk = -1e3 I); (tracks, which see the broken clone): each one that does paired in a CTA with
    one that does not (pairs in both orders)"""
    k, seen = BROKEN[M]
    P = e.covariance().astype(np.float64)
    P[15 + 6 * k:21 + 6 * k, 15 + 6 * k:21 + 6 * k] = -1e3 * np.eye(6)
    e.set_covariance(P)
    rng = np.random.default_rng(seed)
    _, _, poses = state64(e)
    bad = [track_on(rng, poses, idx) for idx in seen]
    good = vr.make_tracks(rng, poses, [len(t["idx"]) for t in bad] if M == 70 else [97, 66, 34], unseen=(k,))
    tracks, broken = [], []
    for j, (b, o) in enumerate(zip(bad, good)):
        pair = (b, o) if j % 2 == 0 else (o, b)
        tracks += pair
        broken += [p is b for p in pair]
    return vr.rounded(tracks, dtype), np.array(broken), k


def check_broken(e, before, rep, tracks, broken, k, dtype, label):
    """the broken tracks: gamma 1e30, rejected; the others: the reference computed at the state `before` on them alone"""
    S = np.dtype(dtype).type
    assert np.all(rep["gamma"][broken] == S(1e30)), (label, rep["gamma"][broken])
    assert not rep["accepted"][broken].any(), label
    ok = np.flatnonzero(~broken)
    kept = [tracks[j] for j in ok]
    P, imu, poses = before
    ref = vr.reference(P, imu, poses, kept)
    assert ref["accepted"].all(), label
    sub = {"accepted": rep["accepted"][ok], "gamma": rep["gamma"][ok], "m": rep["m"], "rank": rep["rank"]}
    checked(e, sub, ref, kept, dtype, label, imu, poses)
    # compare() measures P against its largest entry, the broken block's 1e3: the rest of P against its own
    keep = np.r_[0:15 + 6 * k, 21 + 6 * k:P.shape[0]]
    D = state64(e)[0][np.ix_(keep, keep)] - ref["P"][np.ix_(keep, keep)]
    rel = float(np.abs(D).max() / np.abs(ref["P"][np.ix_(keep, keep)]).max())
    name = np.dtype(dtype).name
    print(f"{label}: P outside the broken clone {rel:.2e}")
    assert rel <= CONTRACT[name]["P"] and rel <= 10 * MEASURED[name]["P"], (label, rel)


@pytest.mark.parametrize("M", [70, 98])
@pytest.mark.parametrize("dtype", DTYPES)
def test_gate_factor_failure_rejects_only_its_track(dtype, M):
    out = []
    for g in GROUPS:
        e = twin(dtype, M)
        e.set_option(6, float(g))
        tracks, broken, k = broken_case(e, M, dtype, M)
        before = state64(e)
        rep = e.update(capi.RESIDUALIZE, batch_of(tracks, dtype))
        check_group(e, M, g, dtype)
        check_broken(e, before, rep, tracks, broken, k, dtype, f"{np.dtype(dtype).name} M={M} group {g} broken clone {k}")
        out.append(outcome(e, rep))
    for o in out[1:]:
        assert same_bits(out[0], o)


@pytest.mark.parametrize("dtype", DTYPES)
def test_gate_factor_failure_in_a_device_batch(dtype):
    """members: threshold pairs, the broken window of 70 clones, clean sweep-like tracks; each equals its single call"""
    M = 70
    mem = [twin(dtype, M) for _ in range(3)]
    tracks, want = threshold_pairs(mem[0], WINDOWS[0][1], dtype, 7)
    broken_tracks, broken, k = broken_case(mem[1], M, dtype, 8)
    before = state64(mem[1])
    _, _, poses = state64(mem[2])
    clean = vr.rounded(vr.make_tracks(np.random.default_rng(9), poses, [70, 66, 33, 17, 3, 2] * 3), dtype)
    trs = [tracks, broken_tracks, clean]
    solo = [engine(dtype, M, src=m) for m in mem]
    batch = capi.Batch(mem)
    reps = batch.update(capi.RESIDUALIZE, [batch_of(t, dtype) for t in trs], full=True)
    batch.close()
    for i, (m, s, tr, rep) in enumerate(zip(mem, solo, trs, reps)):
        label = f"{np.dtype(dtype).name} broken batch member {i}"
        r1 = s.update(capi.RESIDUALIZE, batch_of(tr, dtype))
        for key in ("m", "rank"):
            assert rep[key] == r1[key], (label, key)
        for key in ("accepted", "gamma", "valid"):
            assert np.array_equal(rep[key], r1[key]), (label, key)
        for x, y in zip(state64(m) + (m.delta_x(),), state64(s) + (s.delta_x(),)):
            assert np.array_equal(x, y), label
    assert np.array_equal(reps[0]["accepted"].astype(bool), want)
    assert reps[2]["accepted"].all()
    check_broken(mem[1], before, reps[1], broken_tracks, broken, k, dtype, f"{np.dtype(dtype).name} broken batch member")


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("M,lengths", WINDOWS, ids=["M70", "M98"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_observation_order_does_not_matter(dtype, M, lengths):
    """each track's observations reversed and randomly permuted: the same flags and m as in ascending order, the numbers within
    compare()'s bounds of the ascending tracks' reference, and in fp64 the same rank (an fp32 filter keeps a rounding-noise
    pivot of Gamma or not by its rounding, which the order changes: compare() bounds that rank)"""
    base = twin(dtype, M)
    tracks, want = threshold_pairs(base, lengths, dtype, 100 + M)
    _, imu, poses = st = state64(base)
    ref = vr.reference(*st, tracks)
    floor = None
    rng = np.random.default_rng(M)
    orders = {"ascending": lambda L: np.arange(L), "reversed": lambda L: np.arange(L)[::-1], "permuted": rng.permutation}
    first = None
    for name, order in orders.items():
        e = twin(dtype, M)
        tr = []
        for t in tracks:
            p = order(len(t["idx"]))
            tr.append(dict(t, idx=t["idx"][p], obs=t["obs"][p]))
        rep = e.update(capi.RESIDUALIZE, batch_of(tr, dtype))
        label = f"{np.dtype(dtype).name} M={M} {name}"
        assert np.array_equal(rep["accepted"].astype(bool), want), label
        floor = checked(e, rep, ref, tracks, dtype, label, imu, poses, floor)
        first = first or rep
        assert rep["m"] == first["m"] and (dtype == np.float32 or rep["rank"] == first["rank"]), (label, rep["m"], rep["rank"],
                                                                                                  first["m"], first["rank"])


# ----------------------------------------------------------------------------------------------------------------- (e), (f)
def snapshot(e):
    return state64(e) + (counters(e), e.launch_count(), e.delta_x())


def assert_refused(call, engines, mode, why):
    before = [snapshot(e) for e in engines]
    with pytest.raises(RuntimeError, match="rc=-3.*" + why):
        call()
    for b, e in zip(before, engines):
        for x, y in zip(b, snapshot(e)):
            assert np.array_equal(x, y), mode


def refused_everywhere(dtype, M, bad_tracks, why):
    """bad_tracks refused (for the reason `why`, matched against the error message) by a filter and by a device batch whose
    other member is fine, in both update modes that take tracks through k_jac; the filter then updates by the good tracks as
    usual in both modes"""
    e, other = twin(dtype, M), twin(dtype, M)
    _, _, poses = state64(e)
    good = vr.rounded(vr.make_tracks(np.random.default_rng(3), poses, [min(M, 98), M // 2, 3]), dtype)
    batch = capi.Batch([other, e])
    for mode in (capi.RESIDUALIZE, capi.MARGINALIZE):
        b = batch_of(good + bad_tracks, dtype)
        assert_refused(lambda: e.update(mode, b), [e], mode, why)
        assert_refused(lambda: batch.update(mode, [batch_of(good, dtype), b]), [other, e], mode, why)
    batch.close()
    for mode in (capi.MARGINALIZE, capi.RESIDUALIZE):
        rep = twin(dtype, M).update(mode, batch_of(good, dtype))
        assert rep["accepted"][:2].all() and rep["m"] > 0, (mode, rep["accepted"])


@pytest.mark.parametrize("dtype", DTYPES)
def test_track_naming_a_clone_twice_is_refused(dtype):
    rng = np.random.default_rng(11)
    _, _, poses = state64(twin(dtype, 70))
    bad = [track_on(rng, poses, idx) for idx in ([3, 5, 5, 9], [20, 21, 22, 23, 24, 25, 26, 20], [69, 69])]
    refused_everywhere(dtype, 70, vr.rounded(bad, dtype), "names one clone twice")


@pytest.mark.parametrize("dtype", DTYPES)
def test_track_of_99_observations_is_refused(dtype):
    _, _, poses = state64(twin(dtype, 100))
    bad = vr.make_tracks(np.random.default_rng(12), poses, [99])
    assert len(bad[0]["idx"]) == 99
    refused_everywhere(dtype, 100, vr.rounded(bad, dtype), "track length must be in")
