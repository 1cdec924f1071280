"""The dense fp64 reference of the state calls (tests/state_reference.py) that tests/test_state_kernels_gpu.py holds the engine
to: it must reproduce msckf_numpy's propagate, augmentState and covariance slicing in fp64 on windows of 0, 3 and 40 clones at
every Pade branch, Eigen's Pade (msckf_numpy.expm_eigen) must agree with scipy's expm at every branch the GPU tests take, and
the GPU tests' readings must take every branch, each at least 1 % from its threshold, and a pivoting LU in each dtype."""
import numpy as np
import pytest
import scipy.linalg as sla

from oracle.msckf_numpy import MSCKF as NumpyMSCKF, expm_eigen, quat_normalized
from tests import state_reference as sr

DTYPES = [np.float64, np.float32]
# |expm_eigen - scipy expm| / max |expm| over the branch readings below, in the filter's precision: fp64 agrees to rounding, fp32
# to the rounding of its Pade degree 7 and up to four squarings
EXPM_BOUND = {"float64": 1e-13, "float32": 2e-5}


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max())


def all_readings():
    """every reading the GPU tests' branch cases use, of both dtypes' branches"""
    return [r for dt in DTYPES for _, _, r in sr.branch_readings(dt)]


def numpy_filter(M, seed):
    """msckf_numpy in fp64 at sr.setup() with M clones (a few readings apart) and a dense random SPD covariance"""
    f = NumpyMSCKF(np.float64)
    f.initialize(*sr.setup())
    rng = np.random.default_rng(seed)
    for k in range(M):
        for r in sr.readings(rng, 3, 0.01):
            f.propagate(r[0:3], r[3:6], r[6])
        f.augmentState(k, 0.03 * k)
    n = 15 + 6 * M
    B = rng.normal(size=(n, n))
    f._split_P((B @ B.T) / n + 0.1 * np.eye(n))
    return f


def state_of(f):
    """(P, imu [29], poses [M, 7]) of a msckf_numpy filter in the engine's layout"""
    s = f.imu
    imu = np.concatenate([s[k] for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG", "p_I_G_null", "v_I_G_null", "q_IG_null")])
    poses = np.array([np.concatenate([c.p_C_G, c.q_CG]) for c in f.cam_states]).reshape(-1, 7)
    return f._assemble_P(), imu, poses


def move_null_state(f, rng):
    """a null state away from the current one, as an aided fix leaves it"""
    s = f.imu
    s["p_I_G_null"] = s["p_I_G"] + 0.05 * rng.normal(size=3)
    s["v_I_G_null"] = s["v_I_G"] + 0.05 * rng.normal(size=3)
    s["q_IG_null"] = quat_normalized(s["q_IG"] + 0.02 * rng.normal(size=4))


@pytest.mark.parametrize("M", [0, 3, 40])
def test_propagate_matches_msckf_numpy(M):
    for i, r in enumerate(all_readings()):
        f = numpy_filter(M, seed=M)
        if i % 2:
            move_null_state(f, np.random.default_rng(i))
        P, imu, poses = state_of(f)
        P1, imu1 = sr.propagate(P, imu, r, sr.Q_IMU)
        f.propagate(r[0:3], r[3:6], r[6])
        P2, imu2, poses2 = state_of(f)
        assert rel(P1, P2) < 1e-12, (M, i, rel(P1, P2))
        assert np.abs(imu1 - imu2).max() < 1e-12 and np.array_equal(poses2, poses), (M, i)


@pytest.mark.parametrize("M", [0, 3, 40])
def test_propagate_n_is_the_single_steps_in_sequence(M):
    f = numpy_filter(M, seed=10 + M)
    P, imu, _ = state_of(f)
    rs = np.vstack([sr.readings(np.random.default_rng(2), 5), sr.branch_readings(np.float64)[3][2]])
    P1, imu1 = sr.propagate_n(P, imu, rs, sr.Q_IMU)
    for r in rs:
        f.propagate(r[0:3], r[3:6], r[6])
    P2, imu2, _ = state_of(f)
    assert rel(P1, P2) < 1e-12 and np.abs(imu1 - imu2).max() < 1e-12


@pytest.mark.parametrize("M", [0, 3, 40])
def test_augment_matches_msckf_numpy(M):
    f = numpy_filter(M, seed=20 + M)
    P, imu, poses = state_of(f)
    cam = sr.CAMERA
    P1, poses1 = sr.augment(P, imu, poses, cam["q_CI"], cam["p_C_I"])
    f.augmentState(M, 1.0)
    P2, imu2, poses2 = state_of(f)
    assert P1.shape == (P.shape[0] + 6,) * 2
    assert rel(P1, P2) < 1e-12 and np.abs(poses1 - poses2).max() < 1e-12
    assert np.array_equal(P1[:-6, :-6], P)  # the old block is copied, not recomputed
    assert np.array_equal(imu2, imu)


@pytest.mark.parametrize("M", [3, 40])
def test_prune_matches_msckf_numpy_slicing(M):
    rng = np.random.default_rng(30 + M)
    for keep in ([], [M // 2], list(range(1, M)), list(range(M - 1)), list(range(0, M, 2)),
                 sorted(rng.choice(M, M // 2, replace=False).tolist())):
        f = numpy_filter(M, seed=30 + M)
        P, imu, poses = state_of(f)
        P1, poses1 = sr.prune(P, poses, keep)
        f.cam_states = [f.cam_states[k] for k in keep]
        f._gather_cov(keep)
        P2, _, poses2 = state_of(f)
        assert np.array_equal(P1, P2) and np.array_equal(poses1, poses2), keep


@pytest.mark.parametrize("dtype", DTYPES)
def test_expm_eigen_matches_scipy_at_every_branch(dtype):
    """in each dtype's precision, at each of its branch readings: also checks sr.pade_uv (the closed-form coefficients) against
    scipy, since the descriptor's pivoting is read off it"""
    name = np.dtype(dtype).name
    imu = sr.imu_vector()
    for deg, sq, r in sr.branch_readings(dtype):
        F, _ = sr.F_and_G(imu.astype(dtype).astype(np.float64), r[0:3].astype(dtype), r[3:6].astype(dtype))
        A = (F.astype(dtype) * dtype(r[6])).astype(dtype)
        ref = sla.expm(A.astype(np.float64))
        got = expm_eigen(A).astype(np.float64)
        assert rel(got, ref) < EXPM_BOUND[name], (deg, sq, rel(got, ref))
        U, V = sr.pade_uv(A.astype(np.float64) * 2.0 ** -sq, deg)
        E = sla.solve(V - U, V + U)
        for _ in range(sq):
            E = E @ E
        assert rel(E, ref) < EXPM_BOUND["float64"], (deg, sq, rel(E, ref))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gpu_inputs_cover_every_branch(dtype):
    """the readings of tests/test_state_kernels_gpu.py take each Pade branch of their dtype at least 1 % from its threshold
    (fp64: degrees 3, 5, 7, 9 and 13; 13 with 1 and with >= 3 squarings; fp32: degrees 3 and 5, 7 with 0 and >= 2 squarings),
    and one of them pivots, its pivot well clear of the diagonal"""
    name = np.dtype(dtype).name
    imu = sr.imu_vector()
    seen = set()
    swaps = 0
    for deg, sq, r in sr.branch_readings(dtype):
        d = sr.describe(imu, r, dtype)
        assert (d["deg"], d["sq"]) == (deg, sq) and d["margin"] > 0.01, (deg, sq, d)
        assert d["swap"] == (d["gap"] > 1.0), d
        seen.add((deg, min(sq, 3)))
        swaps += d["gap"] > 1.3
    want = {(3, 0), (5, 0), (7, 0), (9, 0), (13, 0), (13, 1), (13, 3)} if name == "float64" else {(3, 0), (5, 0), (7, 0), (7, 2)}
    assert want <= seen, want - seen
    assert swaps >= 1


def test_pick_changes_branch_at_every_threshold():
    """pick() (the descriptor's restatement of ExpmPick) just below and just above each threshold of the margin"""
    for dtype in DTYPES:
        for t in sr.thresholds(dtype, upto=200.0):
            lo, hi = sr.pick(t * (1 - 1e-9), dtype), sr.pick(t * (1 + 1e-9), dtype)
            assert lo != hi, (dtype, t)
    assert sr.pick(30.0, np.float64) == (13, 3) and sr.pick(11.0, np.float32) == (7, 2) and sr.pick(0.01, np.float64) == (3, 0)
