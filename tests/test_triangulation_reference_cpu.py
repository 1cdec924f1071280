"""The plain reference of tests/triangulation_reference.py, which tests/test_triangulation_gpu.py and
tests/test_marginalize_bookkeeping_gpu.py hold the engine to: it must agree with msckf_numpy's restatement of the same text in
fp64, reach the least-squares answer where its trace says the LM converged, restate marginalize()'s bookkeeping as msckf_numpy
does, and its designed tracks must take every branch the GPU tests claim to cover, each decision with a margin."""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.msckf_numpy import MSCKF as NumpyMSCKF, CamState
from tests import triangulation_reference as tr
from tests import vision_reference as vr

M = 70
PARAMS = dict(vr.setup()[2], translation_threshold=tr.DESIGN_THRESHOLD)


@pytest.fixture(scope="module")
def poses():
    return vr.numpy_state(vr.numpy_filter(M))[2]


@pytest.fixture(scope="module")
def designed(poses):
    tracks = tr.designed_tracks(poses, tr.DESIGN_THRESHOLD)
    return tracks, tr.triangulate(poses, tracks, PARAMS)


def random_tracks(poses):
    return vr.make_tracks(np.random.default_rng(3), poses, [2, 3, 5, 17, 32, 33, 64, 65, 70] * 2, outliers=(4, 11))


def test_reference_restates_msckf_numpy(poses, designed):
    f = NumpyMSCKF(np.float64)
    f.params = PARAMS
    cams = [CamState(p[0:3].copy(), p[3:7].copy(), 0.0, k) for k, p in enumerate(poses)]
    rnd = random_tracks(poses)
    tracks = designed[0] + rnd
    ref = tr.triangulate(poses, tracks, PARAMS)
    for j, t in enumerate(tracks):
        cs, obs = [cams[k] for k in t["idx"]], list(t["obs"])
        assert ref["cm"][j] == f._check_motion(obs[0], cs), j
        ok, p = f._initialize_position(cs, obs)
        assert ref["ok"][j] == ok, j
        assert np.abs(ref["pfg"][j] - p).max() <= 1e-10 * np.linalg.norm(p - poses[t["idx"][0], 0:3]), (j, t.get("name"))
    assert ref["ok"][len(designed[0]):].sum() >= len(rnd) - 2


def test_converged_tracks_are_at_the_least_squares_minimum(poses, designed):
    tracks, ref = designed
    n = 0
    for j, t in enumerate(tracks):
        trc = ref["tri_trace"][j]
        if not trc["converged"] or trc["huber"][-1] or t["kind"] == "behind":  # (behind: a depth crosses zero next to the minimum)
            continue
        p = tr.minimiser(poses, list(t["idx"]), t["obs"], trc["sol"])
        assert np.abs(ref["pfg"][j] - p).max() <= 1e-6 * np.linalg.norm(p - poses[t["idx"][0], 0:3]), t["name"]
        n += 1
    assert n >= len(tracks) // 2


@pytest.mark.parametrize("order", tr.ORDERS)
def test_ldlt3_solves_in_every_order_with_ties_and_zero_pivots(order):
    rng = np.random.default_rng(sum(order) + 10 * order[0])
    B = rng.normal(size=(3, 3))
    A = B @ B.T
    d = np.empty(3)
    d[list(order)] = [9.0, 7.0, 5.0]  # order[0] has the largest diagonal entry
    A[np.diag_indices(3)] = d
    b = rng.normal(size=3)
    x, got, tie, zero = tr.ldlt3(A, b)
    assert got == order and not tie and not zero
    assert np.abs(x - np.linalg.solve(A, b)).max() < 1e-12
    A[order[1], order[1]] = A[order[2], order[2]] = 6.0  # a tie in the second search: the entry that sits first wins
    x, got, tie, zero = tr.ldlt3(A, b)
    assert tie and got[0] == order[0]
    assert np.abs(x - np.linalg.solve(A, b)).max() < 1e-12
    x, got, tie, zero = tr.ldlt3(np.diag(np.where(np.arange(3) == order[2], 0.0, d)), b)  # a zero pivot: that unknown is 0
    assert zero and got[2] == order[2] and x[order[2]] == 0 and np.allclose(np.delete(x, order[2]), np.delete(b / d, order[2]))


def test_first_index_wins_a_tie():
    assert tr.ldlt3(np.diag([2.0, 2.0, 2.0]), np.ones(3))[1:3] == ((0, 1, 2), True)
    assert tr.ldlt3(np.diag([1.0, 2.0, 2.0]), np.ones(3))[1:3] == ((1, 2, 0), True)
    assert tr.ldlt3(np.diag([2.0, 1.0, 2.0]), np.ones(3))[1:3] == ((0, 2, 1), True)
    # a tie in the second search is between the slots as the first swap left them: (0, 2) after 0 <-> 1, (1, 0) after 0 <-> 2
    assert tr.ldlt3(np.diag([2.0, 3.0, 2.0]), np.ones(3))[1:3] == ((1, 0, 2), True)
    assert tr.ldlt3(np.diag([2.0, 2.0, 3.0]), np.ones(3))[1:3] == ((2, 1, 0), True)


def bookkeeping_filter(cm, tri, counter0):
    """msckf_numpy's marginalize() on tracks whose checkMotion / initializePosition results are cm / tri, the rest stubbed so
    that only the bookkeeping of its two loops runs (the gate rejects everything)"""
    f = vr.numpy_filter(3)
    f.num_feature_tracks_residualized = counter0
    n = 15 + 6 * 3
    f._check_motion = lambda obs0, cs: bool(cm[int(obs0[0])])
    f._initialize_position = lambda cs, obs: (bool(tri[int(obs[0][0])]), np.full(3, float(obs[0][0])))
    f._calc_residual = lambda p, cs, obs: np.zeros(4)
    f._calc_meas_jacobian = lambda p, ci: (np.zeros((1, n)), np.zeros((4, 1)))
    f._gating_test = lambda H, r, dof: (False, 0.0)
    f._measurement_update = lambda H, r, Ro: None
    f.feature_tracks_to_residualize = [
        SimpleNamespace(observations=[np.array([float(k), 0.0])] * 2, cam_states=f.cam_states[0:2], cam_state_indices=[0, 1],
                        initialized=False, p_f_G=None) for k in range(len(cm))]
    f.marginalize()
    return f


@pytest.mark.parametrize("counter0", [0, 2, 3, 4, 100])
def test_loop_ab_restates_msckf_numpy_bookkeeping(counter0):
    rng = np.random.default_rng(counter0)
    seen = {"shifted": 0, "oob": 0}
    for N in (1, 2, 4, 5, 33, 130):
        for p_cm, p_tri in ((1.0, 1.0), (0.9, 0.8), (0.5, 0.5), (0.1, 0.9), (0.0, 1.0), (1.0, 0.0)):
            cm, tri = rng.random(N) < p_cm, rng.random(N) < p_tri
            f = bookkeeping_filter(cm, tri, counter0)
            ab = tr.loop_ab(cm, tri, counter0)
            if f.last_marg is None:
                continue
            assert np.array_equal(ab["valid"], f.last_marg["valid"]), (N, cm, tri)
            if ab["valid"].any():  # (marginalize returns before loop B when no track passed)
                assert (ab["pfg_shifted"], ab["pfg_oob"]) == (f.stats["pfg_shifted"], f.stats["pfg_oob"]), (N, cm, tri)
            assert ab["counter"] == f.num_feature_tracks_residualized
            assert np.array_equal(ab["pushed"], [p is not None for p in f.last_marg["p_f_G"]])
            seen["shifted"] += ab["pfg_shifted"]
            seen["oob"] += ab["pfg_oob"]
    assert seen["shifted"] > 0 and seen["oob"] > 0


def test_designed_tracks_take_every_branch_with_a_margin(poses, designed):
    tracks, ref = designed
    kinds = {k: [j for j, t in enumerate(tracks) if t["kind"] == k] for k in {t["kind"] for t in tracks}}
    cmt, trt = ref["cm_trace"], ref["tri_trace"]
    # every rejection kind occurs where it was designed, and alone
    assert not ref["cm"][kinds["motion-"]].any() and ref["cm"][kinds["motion+"]].all()
    assert all(abs(abs(cmt[j]["margin"]) - 0.2) < 1e-9 for j in kinds["motion-"] + kinds["motion+"])
    assert {cmt[j]["decider"] for j in kinds["motion+"]} == {1, 2, 3} and all(cmt[j]["above"] == 1 for j in kinds["motion+"])
    for j in kinds["behind"]:
        assert not ref["ok"][j] and trt[j]["behind"] == 1 and trt[j]["cost_margin"] < -0.5, tracks[j]["name"]
        assert trt[j]["min_depth_obs"] == int(tracks[j]["name"].split("@")[1])
    assert {(trt[j]["min_depth_obs"] % 32, trt[j]["min_depth_obs"] // 32) for j in kinds["behind"]} == {(1, 0), (0, 0), (0, 1), (31, 0), (8, 1), (11, 0)}
    for j in kinds["cost"]:
        assert not ref["ok"][j] and trt[j]["behind"] == 0 and trt[j]["cost_margin"] >= 1.0, tracks[j]["name"]  # 2 x the threshold
    for j in kinds["huber"]:
        assert ref["ok"][j] and max(trt[j]["huber"]) >= 1, tracks[j]["name"]
    assert ref["ok"][kinds["clean"]].all() and ref["cm"][kinds["clean"]].all() and ref["ok"][kinds["parallax"]].all()
    # no decision within 10 % of its threshold (depth: a millimetre)
    for j, t in enumerate(tracks):
        assert abs(cmt[j]["margin"]) > 0.1 and abs(trt[j]["cost_margin"]) > 0.1 and abs(trt[j]["min_depth"]) > 5e-4, t["name"]
    # the LM's control flow
    assert {trt[j]["exit"] for j in range(len(tracks))} == {"cap", "delta"}
    assert max(max(t["inner"]) for t in trt) == 11
    assert min(min(t["lambdas"]) for t in trt) == 1e-10
    assert any(a and not b for t in trt for b, a in zip(t["accepted"], t["accepted"][1:]))  # refused, then accepted at a larger lambda
    assert any(t["outer"] == 11 for t in trt) and any(t["outer"] == 1 for t in trt)
    # the solve
    assert {t["orders"][0] for t in trt} == set(tr.ORDERS_REACHED) == set(tr.ORDERS)
    assert not any(t["tie"] or t["zero"] for t in trt)


def test_fp32_exclusions_are_listed(poses, designed):
    """the designed tracks whose flags an fp32 run of the reference decides otherwise: the fp32 GPU cases leave them out by name"""
    assert sorted(tr.fp32_excluded(poses, designed[0], PARAMS)) == sorted(tr.FP32_EXCLUDED)
