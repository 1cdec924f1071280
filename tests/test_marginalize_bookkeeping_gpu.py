"""MARGINALIZE end to end on tracks with designed checkMotion / triangulation outcomes, staged so that a failure names its stage:
  1. the report's tri_ok equals the plain reference's (tests/triangulation_reference.py) and its cm_ok the reference's
     checkMotion where marginalize() consults it (passed where it does not: counter <= 3);
  2. the report's valid flags and the filter's num_residualized / pfg_shifted / pfg_oob counters equal loop_ab on those flags
     (msckf.h:352-399, :419: the bookkeeping k_jac's prologue restates as a strided scan with group reductions);
  3. the update equals the dense reference of tests/vision_reference.py on the valid tracks, each at the position the engine
     triangulated for the track loop_ab says loop B reads (p_f_G_vec[iter]: a neighbour's after a checkMotion rejection).
Patterns: no rejection, one checkMotion rejection at chosen tracks (every later track shifted), triangulation rejections only
(pushed: no shift), so many checkMotion rejections that late tracks read out of bounds, everything rejected, rejections among the
first tracks while the counter is <= 3; at track counts that make the scan stride once and several times for each group size
(128, 64, 32 threads per track, bit-identical), from counters of 0, 2 and 6 (reached by a preceding update), and in a device batch launched, captured and replayed with new
patterns."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests import triangulation_reference as tr
from tests import vision_reference as vr
from tests.test_triangulation_gpu import engine_at
from tests.test_update_shapes_gpu import compare, counters, state64

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
THRESHOLD = tr.DESIGN_THRESHOLD
PARAMS = dict(vr.setup()[2], translation_threshold=THRESHOLD)


def fresh(dtype, M, counter0):
    """an engine of M clones at THRESHOLD whose counter is counter0, reached by a MARGINALIZE of counter0 clean tracks.  Built
    anew each time (identically driven engines are bit-identical): a twin made by msckf_b200_copy_state inherits the counter
    but triangulates at its own filter's translation_threshold"""
    e = engine_at(dtype, M, THRESHOLD)
    if counter0:
        e.update(capi.MARGINALIZE, batch(make(np.random.default_rng(0), state64(e)[2], "v" * counter0), dtype))
    assert counters(e)[0] == counter0
    return e


def batch(tracks, dtype):
    return capi.TrackBatch(*vr.pack([dict(t, pfg=np.zeros(3)) for t in tracks], dtype)[:3], dtype)


def make(rng, poses, pattern):
    """tracks with the outcomes of `pattern`: "v" valid (3 .. 6 observations of a landmark ahead), "m" fails checkMotion (two
    observations, 20 % below the threshold; it triangulates), "t" fails triangulation (gross outliers), "b" fails both"""
    M = len(poses)
    out = []
    for ch in pattern:
        if ch in "mb":
            k = int(rng.integers(0, M - 2))
            idx = np.array([k, k + 2])
            obs = tr.motion_track(poses, idx, 0.8, THRESHOLD)
            if ch == "b":
                obs = obs + [[0.0, 0.0], [0.3, -0.3]]
        else:
            L = int(rng.integers(3, 7))
            idx = np.sort(rng.choice(M, L, replace=False))
            obs, _ = tr._observe(poses, idx, tr._ahead(poses, idx[L // 2], rng.uniform(-0.3, 0.3), rng.uniform(3, 8)))
            obs += 3e-4 * rng.normal(size=obs.shape)
            if ch == "t":
                obs[1::2] += 0.3 * rng.choice([-1.0, 1.0], size=obs[1::2].shape)
        out.append({"idx": idx.astype(np.int32), "obs": obs})
    return out


def pattern(kind, N, rng):
    if kind == "none":
        return "v" * N
    if kind.startswith("m@"):
        j = min(int(kind[2:]), N - 1)
        return "v" * j + "m" + "v" * (N - 1 - j)
    if kind == "last":
        return "v" * (N - 1) + "m"
    if kind == "tri":
        return "".join("t" if j % 3 == 1 else "v" for j in range(N))
    if kind == "oob":
        return "".join("m" if j % 4 else "v" for j in range(N))
    if kind == "all":
        return "".join("mtb"[j % 3] for j in range(N))
    if kind == "early":
        return "mtvb" + "".join(rng.choice(list("vvvmt"), N - 4))
    return "".join(rng.choice(list("vvvmtb"), N))


_refs = {}


def staged(e, tracks, dtype, label, counter0, key=None):
    """one MARGINALIZE of e, stages 1 - 3; returns (report, counters, P, dx, state, loop_ab's result) for bit comparisons.  Calls
    with the same key are on the same poses and tracks: the triangulation reference is computed once"""
    name = np.dtype(dtype).name
    P0, imu, poses = state64(e)
    c0 = counters(e)
    assert c0[0] == counter0, label
    tracks = vr.rounded([dict(t, pfg=np.zeros(3)) for t in tracks], dtype)
    if key is None or key not in _refs:
        _refs[key] = tr.triangulate(poses, tracks, dict(PARAMS, translation_threshold=float(dtype(THRESHOLD))))
    ref = _refs[key]
    rep = e.update(capi.MARGINALIZE, batch(tracks, dtype))
    c1 = counters(e)
    ab = tr.loop_ab(ref["cm"], ref["ok"], counter0)
    # stage 1 (MARGINALIZE reports checkMotion as marginalize() saw it: passed where it was not consulted, counter <= 3)
    assert np.array_equal(rep["cm_ok"].astype(bool), ab["pushed"]), (label, "stage 1 cm_ok", np.flatnonzero(rep["cm_ok"].astype(bool) != ab["pushed"]))
    assert np.array_equal(rep["tri_ok"].astype(bool), ref["ok"]), (label, "stage 1 tri_ok", np.flatnonzero(rep["tri_ok"].astype(bool) != ref["ok"]))
    # stage 2
    assert np.array_equal(rep["valid"].astype(bool), ab["valid"]), (label, "stage 2 valid", np.flatnonzero(rep["valid"].astype(bool) != ab["valid"]))
    assert (c1[0], c1[1] - c0[1], c1[2] - c0[2]) == (ab["counter"], ab["pfg_shifted"], ab["pfg_oob"]), (label, "stage 2 counters", c0, c1, ab)
    # stage 3
    used = [dict(tracks[j], pfg=rep["p_f_G"][ab["src"][j]].astype(np.float64)) for j in np.flatnonzero(ab["valid"])]
    upd = vr.reference(P0, imu, poses, used)
    # a checkMotion-failing track that is valid all the same (not consulted: counter <= 3) has its landmark along the direction
    # of travel: an update through it amplifies the rounding of p_f_G past any bound, so stage 3 leaves those cases to 1 and 2
    if vr.gate_margin(upd, used) > 0.1 and not any(len(tracks[j]["idx"]) == 2 for j in np.flatnonzero(ab["valid"])):
        got = dict(rep, accepted=rep["accepted"][ab["valid"]], gamma=rep["gamma"][ab["valid"]])
        compare(e, got, upd, used, dtype, label + " stage 3")
        assert not rep["accepted"][~ab["valid"]].any(), (label, "stage 3")
    else:
        print(label, "stage 3 skipped: a gate within 10 % of its threshold, or a valid track without parallax")
    return rep, c1, e.covariance(), e.delta_x(), e.state(), ab


KINDS = ["none", "m@0", "m@1", "m@31", "m@32", "m@63", "m@64", "m@127", "m@128", "m@129", "last", "tri", "oob", "all", "early", "mixed"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [5, 120, 129, 300])
def test_patterns_against_the_reference_at_every_group_size(dtype, N):
    """every pattern at N tracks, from counters 0, 2 and 6 in turn, with 128, 64 and 32 threads per track: stages 1 - 3 and the
    three group sizes bit-identical"""
    M = 12 if N < 300 else 40
    seen = {"shifted": 0, "oob": 0, "he_mid": 0}
    for i, kind in enumerate(KINDS if dtype == np.float64 else KINDS[::3]):
        counter0 = (0, 2, 6)[i % 3] if kind != "early" else (0, 2)[N % 2]
        rng = np.random.default_rng(1000 * N + i)
        pat = pattern(kind, N, rng)
        outs = []
        for g in (128, 64, 32):
            e = fresh(dtype, M, counter0)
            e.set_option(6, float(g))
            tracks = make(np.random.default_rng(7 * N + i), state64(e)[2], pat)
            outs.append(staged(e, tracks, dtype, f"{np.dtype(dtype).name} N={N} {kind} counter {counter0} G={g}", counter0,
                               key=(np.dtype(dtype).name, N, kind)))
            assert e.jac_group() == g
        ab = outs[0][5]
        seen["shifted"] += ab["pfg_shifted"]
        seen["oob"] += ab["pfg_oob"]
        seen["he_mid"] += int(counter0 <= 3 < ab["counter"])
        for o in outs[1:]:
            for k in ("cm_ok", "tri_ok", "valid", "accepted", "gamma", "p_f_G"):
                assert np.array_equal(outs[0][0][k], o[0][k]), (N, kind, k)
            assert outs[0][1] == o[1] and np.array_equal(outs[0][2], o[2]) and np.array_equal(outs[0][3], o[3]), (N, kind)
            assert all(np.array_equal(x, y) for x, y in zip(outs[0][4], o[4])), (N, kind)
    assert (seen["shifted"] > 0 and seen["oob"] > 0 or N == 5) and seen["he_mid"] > 0, seen  # (five tracks cannot run out of positions)


@pytest.mark.parametrize("dtype", DTYPES)
def test_device_batch_with_rejections(dtype):
    """eight members with different patterns, track counts and counters (32 threads per track): each bit-identical to a twin run
    alone and right; launched, captured and replayed, each run with new patterns at the same launch shape"""
    spec = [(12, 0, 5), (12, 2, 120), (12, 6, 129), (40, 0, 300), (12, 6, 33), (40, 2, 64), (12, 0, 130), (12, 6, 300)]
    mem = [fresh(dtype, M, c) for M, c, _ in spec]
    solo = [fresh(dtype, M, c) for M, c, _ in spec]
    b = capi.Batch(mem)
    for it in range(3):
        tracks = []
        for i, (m, (M, _, N)) in enumerate(zip(mem, spec)):
            rng = np.random.default_rng(50 * it + i)
            tracks.append(make(rng, state64(m)[2], pattern(KINDS[(5 * it + 2 * i + 1) % len(KINDS)], N, rng)))
        c0 = [counters(s)[0] for s in solo]
        reps = b.update(capi.MARGINALIZE, [batch(t, dtype) for t in tracks], full=True)
        for i, (m, s, t, rep) in enumerate(zip(mem, solo, tracks, reps)):
            label = f"{np.dtype(dtype).name} member {i} run {it}"
            r1, c1, P1, dx1, st1, ab = staged(s, t, dtype, label, c0[i])
            for k in ("cm_ok", "tri_ok", "valid", "accepted", "gamma", "p_f_G"):
                assert np.array_equal(rep[k], r1[k]), (label, k)
            assert counters(m) == c1 and np.array_equal(m.covariance(), P1), label
            assert all(np.array_equal(x, y) for x, y in zip(m.state(), st1)), label
            if rep["m"]:
                assert np.array_equal(m.delta_x(), dx1), label
    b.close()
