"""The dense reference of the mapped-landmark update with map uncertainty (tests/landmark_map_reference.py) checked three ways,
its row count, the Python binding's packing of landmark ids and Sigma_L, and the class and C view over a recording stub of
the C-ABI (tests/stub/stub_landmark_map.cpp).  No GPU."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from msckf_mono_b200 import capi, montecarlo as mc
from msckf_mono_b200.cview import FilterBatch
from oracle.msckf_numpy import quat_normalized
from tests import landmark_map_reference as ref
from tests.common import ROOT
from tests.test_aid_gpu import numpy_update
from tests.test_landmark_cpu import _filters
from tests.test_landmark_gpu import dense as exact_dense

R_PIX = np.array([[2.0e-5, 3.0e-6], [3.0e-6, 1.5e-5]])


def window(rng, M):
    """clone poses along a line, looking forward with small rotations, a dense SPD P and an IMU state"""
    poses = np.zeros((M, 7))
    for k in range(M):
        poses[k, 3:7] = quat_normalized(np.concatenate([rng.normal(size=3) * 0.05, [1.0]]))
        poses[k, 0:3] = [0.0, 0.0, -0.2 * k]
    n = 15 + 6 * M
    A = rng.normal(size=(n, n)) * 0.01
    P = A @ A.T + np.diag(rng.uniform(1e-4, 4e-3, n))
    imu = np.zeros(29)
    imu[18] = 1.0
    return poses, P, imu


def scene(rng, poses, sets, sigma=0.1, noise=0.002):
    """landmarks seen from each clone set in `sets` (lists of clones), a dense random Sigma per landmark; returns
    clone, z, p_L, landmark, Sigma [L, 6] in shuffled observation order"""
    clone, z, p_L, lm, Sig = [], [], [], [], []
    for l, cs in enumerate(sets):
        pl = ref.landmarks_seen_from(rng, poses, cs)
        B = rng.normal(size=(3, 3)) * sigma
        Sig.append(ref.tri(B @ B.T + sigma ** 2 * np.eye(3)))
        for k in cs:
            clone.append(k); lm.append(l); p_L.append(pl)
            z.append(ref.project(poses[k], pl)[1][0] + noise * rng.normal(size=2))
    o = rng.permutation(len(clone))
    return (np.array(clone)[o], np.array(z)[o], np.array(p_L)[o], np.array(lm)[o], np.array(Sig))


def close(a, b, tol):
    for x, y in zip(a, b):
        x, y = np.asarray(x, float), np.asarray(y, float)
        assert np.abs(x - y).max() <= tol * max(1.0, np.abs(y).max()), np.abs(x - y).max()


def test_marginal_equals_schmidt_joint_update():
    rng = np.random.default_rng(1)
    for M, sets in ((1, [[0]] * 3), (3, [[0], [0, 1], [0, 1, 2], [1, 2], [2]]), (9, [[0, 2, 4, 5, 6, 7, 8, 1], [3, 4], [5]] * 2)):
        poses, P, imu = window(rng, M)
        clone, z, p_L, lm, Sig = scene(rng, poses, sets)
        H, r, Rb, F, lmu, _, flag = ref.dense(P, poses, clone, z, p_L, lm, Sig, R_PIX)
        assert np.all(flag == 0)
        marg = numpy_update(P, imu, poses, H, r, Rb)
        joint = ref.schmidt(P, imu, poses, H, r, F, lmu, Sig, R_PIX)
        close(marg, joint, 1e-12)


def test_vanishing_map_error_is_the_exact_map_update():
    rng = np.random.default_rng(2)
    poses, P, imu = window(rng, 5)
    clone, z, p_L, lm, Sig = scene(rng, poses, [[0, 1], [1, 2, 3, 4], [4], [0, 2]])
    He, re, Rbe, _, _ = exact_dense(P, poses, clone, z, p_L, R_PIX)
    exact = numpy_update(P, imu, poses, He, re, Rbe)
    prev = np.inf
    for s in (1e-2, 1e-4, 1e-6, 1e-8):  # the difference falls linearly with Sigma
        H, r, Rb, _, _, _, _ = ref.dense(P, poses, clone, z, p_L, lm, Sig * s, R_PIX)
        got = numpy_update(P, imu, poses, H, r, Rb)
        d = max(np.abs(np.asarray(x, float) - np.asarray(y, float)).max() / max(1.0, np.abs(np.asarray(y, float)).max())
                for x, y in zip(got, exact))
        assert d <= 0.02 * prev
        prev = d
    assert prev <= 1e-6


def test_one_observation_is_the_inflated_noise():
    rng = np.random.default_rng(3)
    poses, P, imu = window(rng, 4)
    clone, z, p_L, lm, Sig = scene(rng, poses, [[2]])
    H, r, Rb, F, _, gam, _ = ref.dense(P, poses, clone, z, p_L, lm, Sig, R_PIX)
    Ri = R_PIX + F @ ref.sym(Sig[0]) @ F.T
    He, re, Rbe, game, _ = exact_dense(P, poses, clone, z, p_L, Ri)
    assert np.array_equal(H, He) and np.array_equal(r, re)
    close([Rb, gam], [Rbe, game], 1e-15)
    close(numpy_update(P, imu, poses, H, r, Rb), numpy_update(P, imu, poses, He, re, Rbe), 1e-14)


def test_row_count():
    # clone 0: one-clone landmarks a, b (4 rows -> 4); set {0, 1}: two landmarks, one gated (3 used -> 6); set {1, 2, 3}: 5
    # landmarks (15 used -> min(30, 18) = 18)
    clone = [0, 0, 0, 1, 0, 1] + [1, 2, 3] * 5
    lm = [0, 1, 2, 2, 3, 3] + [l for l in range(4, 9) for _ in range(3)]
    flag = [0, 0, 0, 0, 0, 1] + [0] * 15
    assert ref.rows(clone, lm, flag) == 4 + 6 + 18
    # a landmark of a two-clone set whose observations are all gated: its group has no rows
    assert ref.rows([0, 1], [0, 0], [1, 1]) == 0
    # only one-clone landmarks: the exact map's count
    assert ref.rows([0, 0, 0, 0, 3], [0, 1, 2, 3, 4], [0] * 5) == 6 + 2


def test_binding_packs_landmarks_and_sigma():
    S = np.array([[[4.0, 1.0, 2.0], [1.0, 5.0, 3.0], [2.0, 3.0, 6.0]]])
    spec = {"clone": [0, 1], "z": np.zeros((2, 2)), "p_L": np.ones((2, 3)), "landmark": [0, 0], "Sigma_L": S}
    a, keep = capi.landmark_map_struct(spec)
    assert a.n_landmarks == 1
    got = np.ctypeslib.as_array(C.cast(a.Sigma_L, C.POINTER(C.c_double)), shape=(6,))
    assert np.array_equal(got, [4.0, 1.0, 5.0, 2.0, 3.0, 6.0])
    assert np.array_equal(np.ctypeslib.as_array(C.cast(a.landmark, C.POINTER(C.c_int)), shape=(2,)), [0, 0])
    b, _ = capi.landmark_map_struct(dict(spec, Sigma_L=got.copy()))
    assert np.array_equal(np.ctypeslib.as_array(C.cast(b.Sigma_L, C.POINTER(C.c_double)), shape=(6,)), got)
    # an exact map (no Sigma_L, or a member left alone): every field zero
    for s in ({"clone": [0], "z": np.zeros((1, 2)), "p_L": np.ones((1, 3))}, None):
        e, _ = capi.landmark_map_struct(s)
        assert e.landmark is None and e.Sigma_L is None and e.n_landmarks == 0
    # the exact-map struct keeps its layout: the map travels beside it
    assert C.sizeof(capi.Landmarks) == 80 and C.sizeof(capi.LandmarkMap) == 24


@pytest.fixture(scope="module")
def map_view():
    so = ROOT / "tests" / "stub" / "libmsckf_landmark_map_view_stub.so"
    csrc = ROOT / "msckf_mono_b200" / "csrc"
    src = [ROOT / "tests" / "stub" / "stub_engine.cpp", ROOT / "tests" / "stub" / "stub_batch_state.cpp",
           ROOT / "tests" / "stub" / "stub_landmark_iter.cpp", ROOT / "tests" / "stub" / "stub_landmark_map.cpp",
           csrc / "filter_capi.cpp", csrc / "batch_capi.cpp", csrc / "landmark_capi.cpp", csrc / "map_capi.cpp"]
    deps = src + [csrc / "filter_view.hpp", ROOT / "include" / "msckf_mono" / "msckf.h", ROOT / "include" / "msckf_mono" / "types.h",
                  ROOT / "include" / "msckf_b200.h", ROOT / "include" / "msckf_mono_c.h"]
    if (not so.exists()) or any(s.stat().st_mtime > so.stat().st_mtime for s in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT / 'include'}", *map(str, src), "-o", str(so)])
    return so


def _map_calls(f):
    out = (C.c_longlong * 3)()
    f.lib.msckf_b200_stub_map_calls(C.c_void_p(f.engineHandle()), out)
    return list(out)


def _map_last(f):
    cl, lm, p, sg, n6 = (C.c_int * 64)(), (C.c_int * 64)(), (C.c_double * 192)(), (C.c_double * 64)(), C.c_int()
    n = f.lib.msckf_b200_stub_map_last(C.c_void_p(f.engineHandle()), cl, lm, p, 64, sg, 64, C.byref(n6))
    return list(cl[:n]), list(lm[:n]), np.array(p[:3 * n]).reshape(-1, 3), np.array(sg[:n6.value])


LMK_P = np.array([[1.0, 2.0, 5.0], [-1.0, 0.5, 7.0]])
LMK_S = np.array([[1e-2, 0.0, 2e-2, 0.0, 0.0, 3e-2], [4e-2, 1e-3, 5e-2, 0.0, 2e-3, 6e-2]])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_class_maps_ids_and_forwards_the_map(map_view, dtype):
    (f,), wl = _filters(map_view, 1, dtype, frames=4)
    z = np.tile([0.01, -0.02], (3, 1))
    cb = _map_calls(f)  # (the stub keys its records by engine address, which an earlier, closed filter may have had)
    r = f.map_update([2, 0, 2], [1, 0, 0], z, LMK_P, LMK_S)
    assert r["applied"] == 1 and list(r["flag"]) == [0, 0, 0]
    c0 = _map_calls(f)
    assert c0[0] - cb[0] == 1 and c0[1] == cb[1]
    clones, lm, p, sg = _map_last(f)
    assert clones == [2, 0, 2] and lm == [1, 0, 0]
    assert np.array_equal(p, LMK_P[[1, 0, 0]]) and np.array_equal(sg, LMK_S.ravel())
    # IMU readings queued before the call are handed over first; one C-ABI call per class call
    for (w, a, dT) in wl["frames"][3]["imu"][:4]:
        f.propagate(w, a, dT)
    f.map_update([1], [0], z[:1], LMK_P, LMK_S)
    c1 = _map_calls(f)
    assert c1[0] - c0[0] == 1 and c1[1] == c0[1] and c1[2] - c0[2] == 4
    # an image outside the window or a landmark outside the map: refused before any C-ABI call
    with pytest.raises(RuntimeError, match="not in the window"):
        f.map_update([9], [0], z[:1], LMK_P, LMK_S)
    with pytest.raises(RuntimeError, match="not in the map"):
        f.map_update([1], [2], z[:1], LMK_P, LMK_S)
    assert _map_calls(f) == c1
    f.close()


def test_batch_maps_ids_and_forwards_the_map(map_view):
    fs, _ = _filters(map_view, 3, np.float64, frames=4)
    fb = FilterBatch(fs)
    z = np.tile([0.01, -0.02], (2, 1))
    S33 = np.stack([ref.sym(s) for s in LMK_S])
    cb = [_map_calls(f)[:2] for f in fs]
    res = fb.map_update([([0, 2], [1, 1], z, LMK_P, LMK_S), None, ([1], [0], z[:1], LMK_P[:1], S33[:1])])
    assert res[1] is None and res[0]["applied"] == 1 and res[2]["applied"] == 1
    calls = [[a - b for a, b in zip(_map_calls(f)[:2], c)] for f, c in zip(fs, cb)]
    assert calls == [[0, 1], [0, 0], [0, 1]]
    cl, lm, p, sg = _map_last(fs[0])
    assert cl == [0, 2] and lm == [1, 1] and np.array_equal(p, LMK_P[[1, 1]]) and np.array_equal(sg, LMK_S.ravel())
    cl, lm, p, sg = _map_last(fs[2])
    assert cl == [1] and lm == [0] and np.array_equal(sg, LMK_S[0])
    with pytest.raises(RuntimeError, match="not in the map"):
        fb.map_update([([0], [1], z[:1], LMK_P[:1], LMK_S[:1]), None, None])
    assert [[a - b for a, b in zip(_map_calls(f)[:2], c)] for f, c in zip(fs, cb)] == calls
    fb.close()
    for f in fs:
        f.close()


def test_runner_inputs_are_unchanged_under_defaults():
    truth = mc.make_truth(n_frames=30, seq=8)
    for k in (0, 3):
        base = mc.make_trial(truth, k, fix_every=3, map_every=2, odo_every=4)
        same = mc.make_trial(truth, k, fix_every=3, map_every=2, odo_every=4, map_sigma=0.0, map_clones=1)
        assert "map_points" not in base and "map_points" not in same
        for key in ("fixes", "odometry"):
            assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(base[key], same[key]))
        for a, b in zip(base["maps"], same["maps"]):
            assert (a is None and b is None) or (len(a) == len(b) == 3 and all(np.array_equal(x, y) for x, y in zip(a, b)))


def test_map_error_stream_is_independent_of_the_others():
    truth = mc.make_truth(n_frames=30, seq=8)
    base = mc.make_trial(truth, 2, seed=5, fix_every=3, map_every=3, odo_every=4)
    noisy = mc.make_trial(truth, 2, seed=5, fix_every=3, map_every=3, odo_every=4, map_sigma=0.1, map_clones=3)
    for fa, fb_ in zip(base["frames"], noisy["frames"]):
        assert np.array_equal(fa["update"][0], fb_["update"][0]) and np.array_equal(fa["add"][0], fb_["add"][0])
    for key in ("fixes", "odometry"):
        assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(base[key], noisy[key]))
    pts = truth["landmarks"][::20]
    err = noisy["map_points"] - pts
    assert np.abs(err - 0.1 * np.random.default_rng([5, 2, 4]).standard_normal(pts.shape)).max() <= 1e-12 * np.abs(pts).max()
    for a, b in zip(base["maps"], noisy["maps"]):
        if a is None:
            assert b is None
            continue
        idx, p, z, ago = b
        new = ago == 0  # the newest frame's observations: the same indices and pixel noise as with one clone
        assert np.array_equal(idx[new], a[0]) and np.array_equal(z[new], a[2]) and np.array_equal(p, noisy["map_points"][idx])
        assert set(ago) <= {0, 1, 2}
