"""The iterated mapped-landmark update without a GPU: the dense numpy IEKF of tests/landmark_iter_reference.py (one
linearisation is the dense EKF of tests/test_landmark_gpu.py exactly; a converged result satisfies the Gauss-Newton
stationarity condition; on the relocalisation toy the single linearisation is inconsistent after a large drift and the
iterated update is consistent), the class's and the bindings' handling of max_iter / tol over a recording fake of the C-ABI
(tests/stub/stub_landmark_iter.cpp), and the runner's map_start."""
import ctypes as C
import subprocess

import numpy as np
import pytest
from scipy import stats

from msckf_mono_b200 import capi, montecarlo as mc
from msckf_mono_b200.cview import FilterBatch
from tests.common import ROOT
from tests.landmark_iter_reference import boxminus, boxplus, iekf, relocalisation_trial, stationarity
from tests.test_aid_gpu import numpy_update
from tests.test_landmark_cpu import _filters, _obs
from tests.test_landmark_gpu import R_PIX, dense, landmarks_in_front, project

M_CPU = 6


def _state(rng, M):
    """a synthetic prior: P (15 + 6 M, well conditioned), IMU vector [29], clone poses [M, 7] looking along +z"""
    n = 15 + 6 * M
    A = rng.normal(size=(n, n))
    P = 0.05 * (A @ A.T / n) + 0.01 * np.eye(n)
    imu = np.zeros(29)
    imu[15:19] = [0.0, 0.0, 0.0, 1.0]
    imu[0:3] = rng.normal(size=3)
    poses = np.zeros((M, 7))
    for k in range(M):
        q = np.concatenate([rng.normal(size=3) * 0.1, [1.0]])
        poses[k, 3:7] = q / np.linalg.norm(q)
        poses[k, 0:3] = [0.3 * k, 0.0, 0.0]
    return P, imu, poses


def _drifted(rng, poses, per, drift):
    e = np.zeros(15 + 6 * len(poses))
    for k in range(len(poses)):
        e[15 + 6 * k:21 + 6 * k] = np.array([0, 0, drift / 20, drift, -drift / 2, drift / 3]) + rng.normal(size=6) * 1e-3
    truth = boxplus(poses, e)
    clone, z, p_L = [], [], []
    for k in range(len(poses)):
        pl = landmarks_in_front(rng, truth[k], per, depth=(3.0, 15.0))
        clone += [k] * per
        z.append(project(truth[k], pl)[1] + 0.002 * rng.normal(size=(per, 2)))
        p_L.append(pl)
    return np.array(clone), np.vstack(z), np.vstack(p_L)


@pytest.mark.parametrize("gated", [False, True])
def test_one_linearisation_is_the_dense_ekf(gated):
    rng = np.random.default_rng(5)
    P, imu, poses = _state(rng, M_CPU)
    clone, z, p_L = _drifted(rng, poses, 5, 0.3)
    chi2 = float(np.median(dense(P, poses, clone, z, p_L, R_PIX)[3])) if gated else 0.0  # a gate that takes half
    H, r, Rb, gam, flag = dense(P, poses, clone, z, p_L, R_PIX, chi2)
    Pr, imur, posesr, nisr, _ = numpy_update(P, imu, poses, H, r, Rb)
    for max_iter in (0, 1):
        out = iekf(P, imu, poses, clone, z, p_L, R_PIX, chi2, max_iter=max_iter)
        assert out["iterations"] == 1 and out["converged"] == 0 and out["step"] == 0.0
        assert np.array_equal(out["P"], Pr) and np.array_equal(out["imu"], imur) and np.array_equal(out["poses"], posesr)
        assert out["nis"] == pytest.approx(nisr, rel=1e-12) and np.array_equal(out["flag"], flag)
    if gated:
        assert 0 < flag.sum() < len(flag)  # the gate took some and left some


def test_converged_update_is_stationary_and_flags_are_frozen():
    rng = np.random.default_rng(6)
    P, imu, poses = _state(rng, M_CPU)
    clone, z, p_L = _drifted(rng, poses, 5, 1.0)
    one = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=1)
    out = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=16, tol=1e-12)
    assert out["converged"] == 1 and 3 <= out["iterations"] < 16 and out["step"] <= 1e-12
    assert out["nis"] == one["nis"] and out["dof"] == one["dof"] and np.array_equal(out["gamma"], one["gamma"])
    assert stationarity(P, out["H"], out["r"], out["Rb"], out["dx"]) < 1e-9
    # one linearisation is far from stationary at this drift
    assert stationarity(P, one["H"], one["r"], one["Rb"], one["dx"]) > 1e-3
    # the applied delta is the last step's: the state moved to x^ [+] dx
    assert np.abs(boxminus(out["poses"], poses) - out["dx"][15:]).max() < 1e-12


def test_step_after_the_cap_is_not_taken():
    rng = np.random.default_rng(7)
    P, imu, poses = _state(rng, M_CPU)
    clone, z, p_L = _drifted(rng, poses, 5, 1.0)
    steps = [iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=k)["step"] for k in (2, 3, 4)]
    assert steps[0] > steps[1] > steps[2] > 0.0  # the steps shrink: the iteration contracts
    out = iekf(P, imu, poses, clone, z, p_L, R_PIX, max_iter=3)
    assert out["iterations"] == 3 and out["converged"] == 0


@pytest.mark.parametrize("drift_pos,drift_yaw", [(0.3, 0.02), (1.0, 0.05)])
def test_relocalisation_toy(drift_pos, drift_yaw):
    """5 clones with a drift shared by all of them and a small per-clone part, 5 landmarks per clone at 3-15 m, pixel sigma
    1/458, truths drawn from the prior: the ANEES of a consistent filter is 30 (6 M dof)"""
    M, draws = 5, 200
    dof = 6 * M
    lo, hi = stats.chi2.ppf(0.025, draws * dof) / draws, stats.chi2.ppf(0.975, draws * dof) / draws
    res = {}
    for max_iter in (1, 10):
        rng = np.random.default_rng(11)
        nees = [relocalisation_trial(rng, M, 5, drift_pos, drift_yaw, 1.0 / 458.0, max_iter)[0] for _ in range(draws)]
        res[max_iter] = float(np.mean(nees))
    print(f"relocalisation toy at {drift_pos} m / {drift_yaw} rad: ANEES {res[1]:.1f} (one linearisation), {res[10]:.1f} "
          f"(iterated), bounds [{lo:.1f}, {hi:.1f}]")
    assert res[1] > 3 * dof
    assert lo <= res[10] <= hi


@pytest.fixture(scope="module")
def iter_view():
    so = ROOT / "tests" / "stub" / "libmsckf_landmark_iter_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / "stub_engine.cpp", ROOT / "tests" / "stub" / "stub_batch_state.cpp",
           ROOT / "tests" / "stub" / "stub_landmark_iter.cpp", csrc / "filter_capi.cpp", csrc / "batch_capi.cpp",
           csrc / "landmark_capi.cpp"]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", *map(str, src), "-o", str(so)])
    return so


def _iter_of(f):
    m, t = C.c_int(), C.c_double()
    f.lib.msckf_b200_stub_landmark_iter(C.c_void_p(f.engineHandle()), C.byref(m), C.byref(t))
    return m.value, t.value


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_class_passes_max_iter_and_tol(iter_view, dtype):
    (f,), _ = _filters(iter_view, 1, dtype, frames=4)
    z, p = _obs(3)
    r = f.landmark_update([2, 0, 2], z, p)
    assert _iter_of(f) == (1, 1e-10) and r["iterations"] == 1 and r["converged"] == 0  # the defaults: one linearisation
    r = f.landmark_update([2, 0], z[:2], p[:2], max_iter=8, tol=1e-7)
    assert _iter_of(f) == (8, 1e-7) and r["iterations"] == 8 and r["converged"] == 1 and r["applied"] == 1
    with pytest.raises(RuntimeError):
        f.landmark_update([2], z[:1], p[:1], max_iter=17)
    assert _iter_of(f) == (8, 1e-7)  # refused: nothing recorded
    f.close()


def test_batch_passes_max_iter_and_tol(iter_view):
    fs, _ = _filters(iter_view, 3, np.float64, frames=4)
    fb = FilterBatch(fs)
    z, p = _obs(3)
    res = fb.landmark_update([([0, 1], z[:2], p[:2]), None, ([2], z[:1], p[:1])], max_iter=4, tol=1e-6)
    assert res[1] is None and res[0]["iterations"] == 4 and res[2]["iterations"] == 4
    assert _iter_of(fs[0]) == (4, 1e-6) and _iter_of(fs[2]) == (4, 1e-6) and _iter_of(fs[1]) == (-1, -1.0)
    fb.landmark_update([([1], z[:1], p[:1]), None, None])
    assert _iter_of(fs[0]) == (1, 1e-10)
    assert fs[0].lib.msckf_b200_stub_batch_landmark_calls(C.c_void_p(fb.handle())) == 2
    fb.close()
    for f in fs:
        f.close()


def test_binding_structs_carry_the_iteration():
    a, keep = capi.landmark_struct({"clone": [0, 1], "z": np.zeros((2, 2)), "p_L": np.ones((2, 3)), "max_iter": 6, "tol": 1e-9})
    assert a.max_iter == 6 and a.tol == 1e-9
    a, _ = capi.landmark_struct({"clone": [0], "z": np.zeros((1, 2)), "p_L": np.ones((1, 3))})
    assert a.max_iter == 0 and a.tol == 0.0  # zero-initialised: the single linearisation
    names = [f for f, _ in capi.LandmarkResult._fields_]
    assert names[-3:] == ["iterations", "converged", "step"] and C.sizeof(capi.LandmarkResult) == 56
    assert C.sizeof(capi.Landmarks) == 80 and capi.Landmarks.tol.offset == 72


def test_map_start_keeps_each_frames_map():
    truth = mc.make_truth(n_frames=30, seq=8)
    for k in (0, 2):
        a = mc.make_trial(truth, k, map_every=1, map_stride=20)
        b = mc.make_trial(truth, k, map_every=1, map_stride=20, map_start=17)
        assert len(b["maps"]) == 30 and all(m is None for m in b["maps"][:17])
        for ma, mb in zip(a["maps"][17:], b["maps"][17:]):
            assert all(np.array_equal(x, y) for x, y in zip(ma, mb))
        for fa, fb_ in zip(a["frames"], b["frames"]):
            assert np.array_equal(fa["update"][0], fb_["update"][0])


def test_summary_reports_the_first_map_update():
    rng = np.random.default_rng(3)
    recs = {}
    for k in range(4):
        rows = [{c: 1.0 for c in mc.COMPONENTS} | {"dim_full": 33, "first_bad_pivot": -1} for _ in range(5)]
        first = {"frame": 3, "pos_err2_before": 4.0, "pos_err2_after": 0.01, "nis": float(rng.chisquare(20)), "dof": 20,
                 "iterations": 5, "converged": 1}
        recs[k] = mc.trial_record(rows, [0.0] * 5, map_first=first)
    s = mc.summarize(recs)
    f = s["map_first"]
    assert f["frame"] == 3 and f["pos_rmse_before"] == 2.0 and f["pos_rmse_after"] == pytest.approx(0.1)
    assert f["mean_dof"] == 20 and f["iterations"] == 5 and f["converged"] == 1.0
    assert f["imu_anees"] == s["components"]["imu"]["anees"][3] and f["bounds"][0] < 20 < f["bounds"][1]
    assert "map_first" not in mc.summarize({0: mc.trial_record(rows, [0.0] * 5)})
