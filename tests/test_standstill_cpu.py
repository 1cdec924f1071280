"""The standstill update without a GPU: the split of the dense NIS into the scatter and the mean term and the equality of the
9-row and the dense 6k + 3-row updates (tests/standstill_reference.py), the at-rest models' Jacobians against central
differences through montecarlo.perturb, and what makes each mutation of the design visible."""
import numpy as np
import pytest

from msckf_mono_b200 import montecarlo as mc
from oracle.msckf_numpy import quat_to_rot
from tests import standstill_reference as ref


def _quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def _state(rng, M):
    """a random imu vector (p, v, b_g, b_a, g, q_IG), clone poses and an SPD P over 15 + 6M"""
    imu = np.zeros(19)
    imu[0:3] = rng.normal(size=3)
    imu[3:6] = 0.02 * rng.normal(size=3)
    imu[6:9] = 0.01 * rng.normal(size=3)
    imu[9:12] = 0.1 * rng.normal(size=3)
    imu[12:15] = [0.0, 0.0, -9.81]
    imu[15:19] = _quat(rng)
    poses = np.zeros((M, 7))
    for k in range(M):
        poses[k, 0:3] = rng.normal(size=3)
        poses[k, 3:7] = _quat(rng)
    n = 15 + 6 * M
    A = rng.normal(size=(n, n))
    P = 1e-3 * (A @ A.T / n + 0.1 * np.eye(n))
    return imu, poses, P


def _Q(rng):
    """a Q_imu whose gyro and accelerometer blocks are full SPD matrices"""
    Q = np.diag(rng.uniform(1e-6, 1e-4, size=12))
    for c0, scale in ((0, 1e-6), (6, 1e-4)):
        B = rng.normal(size=(3, 3))
        Q[c0:c0 + 3, c0:c0 + 3] = scale * (B @ B.T / 3 + 0.5 * np.eye(3))
    return Q


@pytest.mark.parametrize("k", [2, 10, 400])
@pytest.mark.parametrize("noise_scale", [1.0, 2.5])
def test_scatter_and_mean_split_the_dense_update(k, noise_scale):
    rng = np.random.default_rng(100 + k)
    imu, poses, P = _state(rng, 3)
    Q = _Q(rng)
    r = ref.rest_readings(rng, imu, k, Q, noise_scale)
    st = ref.stats(r, Q, noise_scale, sigma_v=0.02)
    dense = ref.dense_update(P, imu, poses, r, Q, noise_scale, sigma_v=0.02)
    mean = ref.mean_update(P, imu, poses, st)
    assert abs(st["sigma"] + mean["nis"] - dense["nis"]) <= 1e-10 * dense["nis"]
    assert np.abs(mean["P"] - dense["P"]).max() <= 1e-10 * np.abs(dense["P"]).max()
    assert np.abs(mean["dx"] - dense["dx"]).max() <= 1e-10 * np.abs(dense["dx"]).max()
    assert abs(st["scatter"] - st["sigma"] / (6 * (k - 1))) <= 1e-15 * st["scatter"]


def test_the_mutations_change_what_the_tests_compare():
    """A count-weighted mean moves z; the scatter divided by 6k moves the reported scatter; the sign of H_theta moves the
    update.  Each is far outside the tolerances the GPU tests apply."""
    rng = np.random.default_rng(7)
    imu, poses, P = _state(rng, 2)
    Q = _Q(rng)
    r = ref.rest_readings(rng, imu, 10, Q)
    st = ref.stats(r, Q)
    cnt = ref.stats(r, Q, weights="count")
    assert np.abs(cnt["w"] - st["w"]).max() > 1e-9 and np.abs(cnt["a"] - st["a"]).max() > 1e-9
    assert abs(st["sigma"] / 60.0 - st["scatter"]) > 1e-3 * st["scatter"]
    good, flipped = ref.mean_update(P, imu, poses, st), ref.mean_update(P, imu, poses, st, theta_sign=-1.0)
    assert np.abs(good["P"] - flipped["P"]).max() > 1e-6 * np.abs(good["P"]).max()


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(23)
    M = 2
    imu, poses, _ = _state(rng, M)
    n = 15 + 6 * M
    est = {"imu": imu, "poses": poses}
    z = ref.predicted(imu) + 1e-3 * rng.normal(size=6)
    eps = 1e-6
    Hcd = np.zeros((6, n))
    for c in range(n):
        e = np.zeros(n); e[c] = eps
        sp, sm = mc.perturb(est, e), mc.perturb(est, -e)
        Hcd[:, c] = -((z - ref.predicted(sp["imu"])) - (z - ref.predicted(sm["imu"]))) / (2 * eps)
    H = ref.rest_jacobian(imu, n)
    assert np.abs(Hcd - H).max() <= 1e-6, np.abs(Hcd - H).max()
    assert np.abs(Hcd - ref.rest_jacobian(imu, n, theta_sign=-1.0)).max() > 1.0
    # the accelerometer rows cannot see yaw: H_theta (C g) = 0
    u = quat_to_rot(imu[15:19]) @ imu[12:15]
    assert np.abs(H[3:6, 0:3] @ u).max() <= 1e-12


def test_stationary_window_has_the_chi_square_scatter():
    """at rest the scatter is chi-square with 6 (k - 1) dof whatever the state: its mean over windows is 1"""
    rng = np.random.default_rng(5)
    Q = _Q(rng)
    vals = []
    for _ in range(400):
        imu, _, _ = _state(rng, 0)
        vals.append(ref.stats(ref.rest_readings(rng, imu, 10, Q), Q)["scatter"])
    assert abs(np.mean(vals) - 1.0) < 0.05


# ---- the stop profile of the synthetic trajectory and the runner's stop summary -------------------------------------------
STOP = {"every": 30, "frames": 8, "ramp": 4}


def test_stop_profile_is_at_rest_on_its_plateaus_and_smooth_across_its_ramps():
    from msckf_mono_b200 import synth
    wl = synth.make_stream_workload(n_frames=70, seq=1, max_features=10, pixel_sigma=0.0, imu_noise_frac=0.0, stop=STOP)
    traj, fr = wl["traj"], wl["frames"]
    classes = [traj.frame_class(fr[k - 1]["time"], fr[k]["time"]) for k in range(1, len(fr))]
    assert "cruise" in classes and "ramp" in classes
    n_still = 0
    for k in range(1, len(fr)):
        if classes[k - 1] != "stationary":
            continue
        n_still += 1
        t = fr[k]["time"]
        assert np.array_equal(traj.vel(t), np.zeros(3)) and np.array_equal(traj.acc(t), np.zeros(3))
        for (w, a, dT), j in zip(fr[k]["imu"], range(100)):
            assert np.array_equal(w, np.zeros(3))
            tm = fr[k - 1]["time"] + (j + 0.5) * dT
            assert np.abs(a - traj.R_GI(tm).T @ -synth.G_VEC).max() == 0.0
    assert n_still >= 2 * (STOP["frames"] - 1)
    # s, s' and s'' are continuous: no jump across a ramp's ends bigger than the step allows
    ts = np.linspace(wl["t0"], wl["t0"] + 2 * traj.P, 40001)
    W = np.array([traj.warp(t) for t in ts])
    h = ts[1] - ts[0]
    assert np.abs(np.diff(W[:, 0])).max() <= 1.0001 * h
    assert np.abs(np.diff(W[:, 1])).max() <= 2.0 * h / traj.D
    assert np.abs(np.diff(W[:, 2])).max() <= 10.0 * h / traj.D ** 2
    assert W[:, 1].min() == 0.0 and W[:, 1].max() == 1.0
    # the vision stream sees no motion over a stop: the camera pose of every frame of a stop is one pose
    cls = [None] + classes
    for k in range(2, len(fr)):
        if cls[k] == "stationary":
            assert np.array_equal(traj.pos(fr[k]["time"]), traj.pos(fr[k - 1]["time"]))


def _digest(wl):
    import hashlib
    h = hashlib.sha256()
    for fr in wl["frames"]:
        for (w, a, dT) in fr["imu"]:
            h.update(np.asarray(w, np.float64).tobytes()); h.update(np.asarray(a, np.float64).tobytes()); h.update(np.float64(dT).tobytes())
        for key in ("update", "add"):
            h.update(np.ascontiguousarray(fr[key][0], np.float64).tobytes()); h.update(np.ascontiguousarray(fr[key][1]).tobytes())
    return h.hexdigest()


# the stream of make_stream_workload(n_frames=12, seq=4, max_features=20) before the stop profile existed
STREAM_DIGEST = "e7db312ad2be893f6230c73c17c0afac83df1318553804b0c68c7f9d635def6c"


def test_no_stop_profile_changes_nothing():
    from msckf_mono_b200 import synth
    a = synth.make_stream_workload(n_frames=12, seq=4, max_features=20)
    assert _digest(a) == STREAM_DIGEST
    b = synth.make_stream_workload(n_frames=12, seq=4, max_features=20, stop=None)
    assert type(a["traj"]) is synth.Trajectory and type(b["traj"]) is synth.Trajectory
    for fa, fb in zip(a["frames"], b["frames"]):
        for (wa, aa, da), (wb, ab, db) in zip(fa["imu"], fb["imu"]):
            assert np.array_equal(wa, wb) and np.array_equal(aa, ab) and da == db
        for key in ("update", "add"):
            assert np.array_equal(fa[key][0], fb[key][0]) and np.array_equal(fa[key][1], fb[key][1])
    t = mc.make_truth(n_frames=12, seq=4)
    assert "frame_class" not in t
    tr = mc.make_trial(t, 0, seed=3)
    t2 = mc.make_truth(n_frames=12, seq=4, stop=None)
    tr2 = mc.make_trial(t2, 0, seed=3)
    for fa, fb in zip(tr["frames"], tr2["frames"]):
        for (wa, aa, _), (wb, ab, _) in zip(fa["imu"], fb["imu"]):
            assert np.array_equal(wa, wb) and np.array_equal(aa, ab)


def test_stop_summary():
    cls = [None, "cruise", "ramp", "stationary", "stationary", "stationary", "ramp", "cruise"]
    e = [0.0, 0.1, 0.2, 0.3, 0.35, 0.5, 0.6, 0.7]
    recs = []
    for k in range(2):
        rec = mc.trial_record([], [x ** 2 for x in e], frame_class=cls,
                              standstill_rows=[{"nis": 9.0 + k, "dof": 9 if o == 0 else 0, "applied": int(o == 0), "outcome": o,
                                                "scatter": 1.0} for o in (1, 1, 0, 0, 2, 1, 1)])
        recs.append(rec)
    s = mc.stop_summary(recs)
    assert s["stops"] == [[3, 5]] and s["frames"] == {"stationary": 3, "ramp": 2, "cruise": 2}
    assert abs(s["pos_err_growth_per_stop"] - (0.5 - 0.2)) < 1e-12
    assert s["detected"] == {"stationary": 2 / 3, "ramp": 0.0, "cruise": 0.0}
    assert s["applied"] == 4 and abs(s["anis"] - 9.5) < 1e-12 and s["dof"] == 9
