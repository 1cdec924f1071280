"""The chi-square gate's table and the threshold tracks that tests/test_gate_threshold_gpu.py holds the engine's gate to.

  * The engine's own copy of the table (msckf_mono_b200/csrc/chi2_table.inc, the one k_jac reads) is chi2.ppf(0.05, k),
    k = 1 .. 99, and equals the oracle's copy.
  * vision_reference.threshold_tracks places every track length 2 .. 98 on both sides of its threshold CHI2[L], in both
    precisions, within a tenth of the distance it aims for.
  * The pair of one length catches a gate that reads a neighbouring entry (CHI2[L - 1] or CHI2[L + 1]: one flag of the pair
    flips) and does not flip under the rounding of the table to the filter's precision (an fp32 filter holds the table in
    fp32; an fp64 pair sits 1e-9 from its threshold and does flip there, so it catches an fp64 filter holding an fp32 table).
    A track exactly at its threshold cannot be built (gamma is a rounded sum), so `<=` in place of `<` in the gate is out of
    reach of any such test.
  * The rank decision's noise pivots on such a window: a plain fp64 evaluation of the engine's Gram form
    (vision_reference.gram_noise) exceeds the model tests/test_update_shapes_gpu.py's compare() holds the engine to (100 eps n
    / smallest real pivot), while the reference's own Gram matrix H_c^T H_c stays below it.  The excess is the formula's, so
    the GPU tests hold the engine's noise to that evaluation where it is the larger."""
import re
from pathlib import Path

import numpy as np
import pytest
from scipy.stats import chi2

from tests import vision_reference as vr

ROOT = Path(__file__).resolve().parents[1]
LENGTHS = list(range(2, 99))
# (window, lengths) as the GPU sweep runs them: every group runs as requested up to 66 observations on 70 clones
WINDOWS = [(70, [L for L in LENGTHS if L <= 66]), (98, [L for L in LENGTHS if L > 66])]


def table(path):
    vals = [float(x) for x in re.findall(r"[-+0-9.]+e[-+][0-9]+", path.read_text())]
    assert len(vals) == 99, path
    return np.array(vals)


def test_engine_chi2_table_is_the_lower_five_percent_quantile():
    eng = table(ROOT / "msckf_mono_b200" / "csrc" / "chi2_table.inc")
    assert np.allclose(eng, chi2.ppf(0.05, np.arange(1, 100)), rtol=1e-14, atol=0)
    assert np.array_equal(eng, table(ROOT / "oracle" / "chi2_table.inc"))
    assert np.array_equal(eng, vr.CHI2)


_pairs = {}


def pairs(dtype, M, lengths):
    """(tracks, gamma, target) of a pair per length on the msckf_numpy filter's window of M clones (its state as a filter of
    dtype holds it)"""
    key = (np.dtype(dtype).name, M)
    if key not in _pairs:
        P, imu, poses = vr.numpy_state(vr.numpy_filter(M))
        P, imu, poses = (x.astype(dtype).astype(np.float64) for x in (P, imu, poses))
        tracks, gam, target, sides = vr.threshold_pairs(np.random.default_rng(M), P, imu, poses, lengths, dtype)
        ls = np.array(vr.threshold_sides(lengths)[0])
        _pairs[key] = (tracks, gam, target, ls, sides, np.array([vr.gate_delta(L, dtype) for L in ls]))
    return _pairs[key]


def flags(gam, lengths, thresholds):
    return gam < np.array([thresholds[L] for L in lengths])


@pytest.mark.parametrize("M,lengths", WINDOWS, ids=["M70", "M98"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_threshold_tracks_land_on_both_sides_of_every_threshold(dtype, M, lengths):
    tracks, gam, target, ls, sides, delta = pairs(dtype, M, lengths)
    assert [len(t["idx"]) for t in tracks] == list(ls)
    for t in tracks:  # as the engine receives them
        assert np.array_equal(t["obs"], t["obs"].astype(dtype)) and np.array_equal(t["pfg"], t["pfg"].astype(dtype))
    miss = np.abs(gam / target - 1) / delta
    print(f"{np.dtype(dtype).name} M={M}: worst |gamma / target - 1| / delta {miss.max():.1e}")
    assert miss.max() < 0.1, (ls[np.argmax(miss)], miss.max())
    assert np.array_equal(flags(gam, ls, vr.CHI2), sides < 0)


@pytest.mark.parametrize("M,lengths", WINDOWS, ids=["M70", "M98"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_threshold_pairs_catch_a_neighbouring_entry_but_not_rounding(dtype, M, lengths):
    tracks, gam, _, ls, sides, _ = pairs(dtype, M, lengths)
    ext = np.append(vr.CHI2, chi2.ppf(0.05, 100))  # the entry a gate reading past the table's end would want
    good = flags(gam, ls, vr.CHI2)
    for shift in (-1, 1):
        moved = flags(gam, ls, {L: ext[L + shift] for L in ls})
        for L in lengths:  # one flag of every pair flips
            assert np.sum(moved[ls == L] != good[ls == L]) == 1, (shift, L)
    own = vr.CHI2.astype(dtype).astype(np.float64)
    assert np.array_equal(flags(gam, ls, own), good)
    if dtype == np.float64:  # an fp64 filter with its table rounded to fp32 flips flags
        assert np.sum(flags(gam, ls, vr.CHI2.astype(np.float32).astype(np.float64)) != good) > len(lengths) // 2


def test_gram_form_noise_pivots_exceed_the_conditioning_model():
    """130 threshold tracks over 70 clones (the window and seed of one fp64 device-batch member of the GPU tests): the
    rank decision's largest noise pivot is 3e-9 in the Gram form evaluated in fp64, 4.6 x the model's 6.6e-10, and 5e-10
    from the reference's own H_c^T H_c; the real pivots stay far above either"""
    P, imu, poses = vr.numpy_state(vr.numpy_filter(70))
    tracks, _, _, _ = vr.threshold_pairs(np.random.default_rng(1), P, imu, poses, WINDOWS[0][1], np.float64)
    ref = vr.reference(P, imu, poses, tracks)
    n = P.shape[0]
    Hh, Hc = ref["H_o"][:15, 15:], ref["H_o"][:, 15:]
    G = np.block([[np.eye(15), Hh], [Hh.T, Hc.T @ Hc]])
    pv = np.sort(vr.skip_cholesky_pivots(G))[::-1]
    real, direct = pv[ref["rank"] - 1], np.abs(pv[ref["rank"]:]).max()
    model = 100 * np.finfo(np.float64).eps * n / real
    gram = vr.gram_noise(imu, poses, tracks, ref)
    print(f"smallest real pivot {real:.2e}: noise model {model:.2e}, H_c^T H_c {direct:.2e}, Gram form {gram:.2e}")
    assert real > 1e5 * max(gram, direct)
    assert direct < model < gram
