"""Synthetic IMU + feature-track workloads for the MSCKF update path.

Nothing here is on the product path: it only manufactures inputs (IMU samples and
normalised-coordinate feature tracks with ids) with the shape the reference front-ends
deliver (datasets/asl_msckf.cpp:233-294: propagate per IMU sample, then per image
augmentState / update / addFeatures / marginalize / prune*), so that the oracle and the
H100 engine can be driven through the same MSCKF<_S> surface on identical inputs.

Calibration and noise parameters are the *effective* EuRoC values of SURVEY.md section 5
(euroc/MH_03_kalibr.yaml:6-13, launch/asl_msckf.launch:15-35, datasets/asl_msckf.cpp:73-134).
Seeds: 20260923 + sequence_index (SURVEY.md section 8d).
"""
from __future__ import annotations

import numpy as np

BASE_SEED = 20260923

# euroc/MH_03_kalibr.yaml:6-9 (T_cam_imu: imu -> cam) and :13 intrinsics
T_CAM_IMU = np.array(
    [
        [0.0148655429818, -0.999880929698, 0.00414029679422, -0.021640145497],
        [0.999557249008, 0.0149672133247, 0.025715529948, -0.064676986768],
        [-0.0257744366974, 0.00375618835797, 0.999660727178, 0.009810730590],
        [0.0, 0.0, 0.0, 1.0],
    ]
)
INTRINSICS = (458.654, 457.296, 367.215, 248.375)  # f_u, f_v, c_u, c_v
RESOLUTION = (752, 480)


def rot_to_quat(R):
    """Rotation matrix -> unit quaternion (x,y,z,w), same convention as Eigen::Quaternion(R)."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        w = 0.25 * s
        x = (R[2, 1] - R[1, 2]) / s
        y = (R[0, 2] - R[2, 0]) / s
        z = (R[1, 0] - R[0, 1]) / s
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = np.zeros(3)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        w = (R[k, j] - R[j, k]) / s
        x, y, z = q
    q = np.array([x, y, z, w])
    return q / np.linalg.norm(q)


def so3_exp(phi):
    th = np.linalg.norm(phi)
    K = np.array([[0, -phi[2], phi[1]], [phi[2], 0, -phi[0]], [-phi[1], phi[0], 0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * (K @ K)


def so3_log(R):
    c = np.clip((np.trace(R) - 1) / 2, -1, 1)
    th = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if th < 1e-9:
        return v / 2
    return th / (2 * np.sin(th)) * v


def euroc_camera():
    """types.h:48-56 Camera: q_CI rotates IMU -> camera, p_C_I camera position in IMU frame
    (datasets/asl_readers.cpp:27-33: q_BS = Quaternion(R_BS).inverse(), p_BS)."""
    R_CI = T_CAM_IMU[:3, :3]
    p_C_I = -R_CI.T @ T_CAM_IMU[:3, 3]
    return {
        "c_u": INTRINSICS[2], "c_v": INTRINSICS[3], "f_u": INTRINSICS[0], "f_v": INTRINSICS[1],
        "b": 0.0, "q_CI": rot_to_quat(R_CI), "p_C_I": p_C_I,
    }


def euroc_noise(feature_cov=7.0, isotropic=False, tuned=False):
    """datasets/asl_msckf.cpp:73-101 with the launch-file name mismatches of SURVEY.md section 5.

    tuned=True replaces the (very loose) EuRoC bias random walks / initial variances by values that
    match the simulator's actual IMU noise (imu_noise_frac=0.05, zero biases); used only by the
    end-to-end trajectory sanity tests, never by the parity or bench configurations.
    """
    f_u, f_v = INTRINSICS[0], INTRINSICS[1]
    if isotropic:
        f_v = f_u
    w_var, dbg_var, a_var, dba_var = 1e-4, 3.6733e-5, 1e-2, 7e-2
    Q = np.diag([w_var] * 3 + [dbg_var] * 3 + [a_var] * 3 + [dba_var] * 3)
    P0 = np.diag([1e-5] * 3 + [1e-2] * 3 + [1e-2] * 3 + [1e-2] * 3 + [1e-12] * 3)
    if tuned:
        Q = np.diag([w_var * 0.01] * 3 + [1e-8] * 3 + [a_var * 0.01] * 3 + [1e-6] * 3)
        P0 = np.diag([1e-5] * 3 + [1e-8] * 3 + [1e-6] * 3 + [1e-6] * 3 + [1e-12] * 3)
    return {
        "u_var_prime": (feature_cov / f_u) ** 2,
        "v_var_prime": (feature_cov / f_v) ** 2,
        "Q_imu": Q,
        "initial_imu_covar": P0,
    }


def euroc_params(max_track_length=50, min_track_length=3, max_cam_states=30):
    """datasets/asl_msckf.cpp:104-125 (+ launch/asl_msckf.launch:28-35)."""
    return {
        "max_gn_cost_norm": (11.0 / INTRINSICS[0]) ** 2,
        "min_rcond": 3e-12,
        "translation_threshold": 0.01,
        # launch keyframe_transl_dist -> redundancy_angle_thresh, keyframe_rot_dist ->
        # redundancy_distance_thresh (swapped in asl_msckf.cpp:112-113)
        "redundancy_angle_thresh": 0.05,
        "redundancy_distance_thresh": 0.05,
        "min_track_length": int(min_track_length),
        "max_track_length": int(max_track_length),
        "max_cam_states": int(max_cam_states),
    }


class Trajectory:
    """Circle of radius 2 m at 0.5 m/s with a +-0.2 m vertical sinusoid (SURVEY.md 8d).

    Body z (the EuRoC camera's optical axis is ~ IMU z) looks radially outward and rotates
    with the circle; a small sinusoidal wobble is superimposed.
    """

    def __init__(self, radius=2.0, speed=0.5):
        self.r = radius
        self.w = speed / radius

    def pos(self, t):
        return np.array([self.r * np.cos(self.w * t), self.r * np.sin(self.w * t), 0.2 * np.sin(0.8 * t)])

    def vel(self, t):
        return np.array([-self.r * self.w * np.sin(self.w * t), self.r * self.w * np.cos(self.w * t),
                         0.16 * np.cos(0.8 * t)])

    def acc(self, t):
        return np.array([-self.r * self.w**2 * np.cos(self.w * t), -self.r * self.w**2 * np.sin(self.w * t),
                         -0.128 * np.sin(0.8 * t)])

    def R_GI(self, t):
        th = self.w * t
        zb = np.array([np.cos(th), np.sin(th), 0.0])
        xb = np.array([0.0, 0.0, 1.0])
        yb = np.cross(zb, xb)
        Rb = np.stack([xb, yb, zb], axis=1)
        phi = np.array([0.05 * np.sin(1.1 * t), 0.04 * np.sin(0.9 * t + 1.0), 0.03 * np.sin(1.3 * t + 2.0)])
        return Rb @ so3_exp(phi)

    def omega_body(self, t, h=1e-4):
        return so3_log(self.R_GI(t - h).T @ self.R_GI(t + h)) / (2 * h)


class StopProfile:
    """The trajectory `base` driven through the time warp s(t): stops of `frames` frames every `every` frames, entered and left
    through quintic ramps of `ramp` frames each, so that the speed s' and s'' are continuous.  Period p starts at t0 + p every
    frame_dt: (every - frames - 2 ramp) frames at full speed (s' = 1), a ramp down (s' = 1 - q(u), q(u) = 6u^5 - 15u^4 + 10u^3),
    the stop (s' = 0), a ramp up (s' = q(u)).  Before t0 it runs at full speed.  With s = s(t): pos = base.pos(s),
    vel = base.vel(s) s', acc = base.acc(s) s'^2 + base.vel(s) s'', R_GI = base.R_GI(s) and omega_body = s' base.omega_body(s),
    so that a reading at rest is exactly omega = 0, a = -C g."""

    def __init__(self, base, t0, frame_dt, every, frames, ramp):
        assert ramp >= 1 and frames >= 1 and every >= frames + 2 * ramp + 1, (every, frames, ramp)
        self.base, self.t0 = base, t0
        self.r, self.w = base.r, base.w
        self.P, self.A, self.D, self.S = every * frame_dt, (every - frames - 2 * ramp) * frame_dt, ramp * frame_dt, frames * frame_dt

    def warp(self, t):
        """(s, s', s'') at time t"""
        if t < self.t0:
            return t, 1.0, 0.0
        n, tau = divmod(t - self.t0, self.P)
        s0 = self.t0 + n * (self.A + self.D)
        A, D, S = self.A, self.D, self.S
        if tau < A:
            return s0 + tau, 1.0, 0.0
        if tau < A + D:
            u = (tau - A) / D
            return s0 + A + D * (u - (u ** 6 - 3 * u ** 5 + 2.5 * u ** 4)), 1.0 - (6 * u ** 5 - 15 * u ** 4 + 10 * u ** 3), \
                -(30 * u ** 4 - 60 * u ** 3 + 30 * u ** 2) / D
        if tau < A + D + S:
            return s0 + A + 0.5 * D, 0.0, 0.0
        u = (tau - A - D - S) / D
        return s0 + A + 0.5 * D + D * (u ** 6 - 3 * u ** 5 + 2.5 * u ** 4), 6 * u ** 5 - 15 * u ** 4 + 10 * u ** 3, \
            (30 * u ** 4 - 60 * u ** 3 + 30 * u ** 2) / D

    def frame_class(self, ta, tb):
        """'stationary' when s' = 0 over all of [ta, tb], 'cruise' when s' = 1 over all of it, else 'ramp'"""
        if ta < self.t0:
            return "cruise" if tb <= self.t0 + self.A else "ramp"
        na, a = divmod(ta - self.t0, self.P)
        nb, b = divmod(tb - self.t0, self.P)
        eps = 1e-9 * self.P  # (frame times are sums of frame_dt: a boundary may land a rounding error either side)
        if na == nb and self.A + self.D - eps <= a and b <= self.A + self.D + self.S + eps:
            return "stationary"
        if (na == nb and b <= self.A + eps) or (nb == na + 1 and b <= eps and a <= self.A + eps):
            return "cruise"
        return "ramp"

    def pos(self, t):
        return self.base.pos(self.warp(t)[0])

    def vel(self, t):
        s, s1, _ = self.warp(t)
        return self.base.vel(s) * s1

    def acc(self, t):
        s, s1, s2 = self.warp(t)
        return self.base.acc(s) * s1 * s1 + self.base.vel(s) * s2

    def R_GI(self, t):
        return self.base.R_GI(self.warp(t)[0])

    def omega_body(self, t):
        s, s1, _ = self.warp(t)
        return s1 * self.base.omega_body(s)


G_VEC = np.array([0.0, 0.0, -9.81])


def imu_samples(traj, t0, n, dT, rng, noise_frac=0.05, Q=None):
    """n readings covering [t0, t0+n*dT): mid-interval rates, small white noise
    (noise_frac of the modelled discrete std sqrt(var/dT))."""
    out = []
    w_std = a_std = 0.0
    if Q is not None and noise_frac > 0:
        w_std = noise_frac * np.sqrt(Q[0, 0] / dT)
        a_std = noise_frac * np.sqrt(Q[6, 6] / dT)
    for k in range(n):
        tm = t0 + (k + 0.5) * dT
        R = traj.R_GI(tm)
        omega = traj.omega_body(tm) + w_std * rng.standard_normal(3)
        a = R.T @ (traj.acc(tm) - G_VEC) + a_std * rng.standard_normal(3)
        out.append((omega, a, dT))
    return out


def true_imu_state(traj, t):
    R = traj.R_GI(t)
    return {
        "p_I_G": traj.pos(t), "v_I_G": traj.vel(t), "b_g": np.zeros(3), "b_a": np.zeros(3),
        "g": G_VEC.copy(), "q_IG": rot_to_quat(R.T),
    }


def cam_pose(traj, t, cam):
    """camera rotation C_CG (global -> cam) and position p_C_G at time t."""
    from_q = cam["q_CI"]
    x, y, z, w = from_q
    R_CI = np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
    ])
    R_GI = traj.R_GI(t)
    C_CG = R_CI @ R_GI.T
    p_C_G = traj.pos(t) + R_GI @ cam["p_C_I"]
    return C_CG, p_C_G


def make_window_workload(n_features=300, n_clones=30, seq=0, imu_per_frame=10, dT=0.005,
                         pixel_sigma=1.0, imu_noise_frac=0.05, isotropic=False,
                         max_cam_states=None):
    """Config B / S recipe (SURVEY.md 8d): N landmarks seen in all M clones; produced
    through the public API so that the marginalize() after frame M processes N x M.

    Returns a dict with camera/noise/params/imu_state and a list of frames:
      frame = {"imu": [(omega,a,dT)...], "state_id": k, "time": t,
               "update": (obs[N,2], ids) or None, "add": (obs[N,2], ids) or None}
    """
    rng = np.random.default_rng(BASE_SEED + seq)
    cam = euroc_camera()
    noise = euroc_noise(isotropic=isotropic)
    params = euroc_params(max_track_length=n_clones, min_track_length=3,
                          max_cam_states=max_cam_states or max(n_clones, 30))
    traj = Trajectory()
    t0 = 1.0 + 0.37 * seq
    frame_dt = imu_per_frame * dT
    # landmarks in the first camera's frame
    C0, p0 = cam_pose(traj, t0, cam)
    depth = rng.uniform(3.0, 15.0, n_features)
    xn = rng.uniform(-0.6, 0.6, n_features)
    yn = rng.uniform(-0.4, 0.4, n_features)
    pts_c0 = np.stack([xn * depth, yn * depth, depth], axis=1)
    pts_G = (C0.T @ pts_c0.T).T + p0
    f_u = INTRINSICS[0]
    sig = pixel_sigma / f_u
    ids = np.arange(1000, 1000 + n_features, dtype=np.uint64)
    frames = []
    for k in range(n_clones):
        t = t0 + k * frame_dt
        C, p = cam_pose(traj, t, cam)
        pc = (C @ (pts_G - p).T).T
        assert np.all(pc[:, 2] > 0.5), "landmark behind camera in synthetic window"
        obs = pc[:, :2] / pc[:, 2:3] + sig * rng.standard_normal((n_features, 2))
        fr = {"imu": [] if k == 0 else imu_samples(traj, t - frame_dt, imu_per_frame, dT, rng,
                                                   imu_noise_frac, noise["Q_imu"]),
              "state_id": k, "time": t, "update": None, "add": None}
        if k == 0:
            fr["add"] = (obs, ids)
        else:
            fr["update"] = (obs, ids)
        frames.append(fr)
    return {"camera": cam, "noise": noise, "params": params, "imu_state": true_imu_state(traj, t0),
            "frames": frames, "landmarks": pts_G, "traj": traj, "t0": t0}


def corrupt_observations(wl, frac_gross=0.1, frac_mild=0.15, seed=0):
    """Turn some landmarks of a window workload into outliers: `gross` ones get a large offset in a few
    frames (triangulation cost / cheirality / gate reject them), `mild` ones a small offset (borderline)."""
    rng = np.random.default_rng(seed)
    frames = wl["frames"]
    n = len(frames[0]["add"][1])
    kinds = rng.random(n)
    for k, fr in enumerate(frames):
        obs = fr["add"][0] if fr["add"] is not None else fr["update"][0]
        for j in range(n):
            if kinds[j] < frac_gross and k % 3 == 1:
                obs[j] += rng.normal(0, 0.3, 2)
            elif kinds[j] < frac_gross + frac_mild and k % 2 == 0:
                obs[j] += rng.normal(0, 0.012, 2)
    return wl


def visible(C, p, pts_G):
    """the stream's visibility rule for a camera with rotation C (global -> cam) at p: depth in (1, 25) m and the pixel at
    least 5 px inside the image.  Returns (vis [N] bool, xn, yn) with the normalised coordinates of every point."""
    f_u, f_v, c_u, c_v = INTRINSICS
    pc = (C @ (pts_G - p).T).T
    z = pc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        xn = pc[:, 0] / z
        yn = pc[:, 1] / z
    u = f_u * xn + c_u
    v = f_v * yn + c_v
    vis = (z > 1.0) & (z < 25.0) & (u > 5) & (u < RESOLUTION[0] - 5) & (v > 5) & (v < RESOLUTION[1] - 5)
    return vis, xn, yn


def make_stream_workload(n_frames=200, seq=0, max_features=100, imu_per_frame=10, dT=0.005,
                         pixel_sigma=1.0, imu_noise_frac=0.05, n_landmarks=6000,
                         max_track_length=50, max_cam_states=30, isotropic=False, dropout=0.02, stop=None):
    """E-sim (SURVEY.md 8d): streamed propagate+update sequence with tracks that appear,
    persist while visible and are lost, <= max_features per frame, ids never reused.

    Stands in for EuRoC MH_03 (not on this box).  Feature bookkeeping mimics the front end
    (corner_detector.cpp TrackHandler): `update` receives the still-tracked features,
    `add` the newly detected ones.  stop = dict(every, frames, ramp): the trajectory stops (StopProfile, from the first frame
    on); None: it never does, and every output is what it was without the option.
    """
    rng = np.random.default_rng(BASE_SEED + seq)
    cam = euroc_camera()
    noise = euroc_noise(isotropic=isotropic)
    params = euroc_params(max_track_length=max_track_length, min_track_length=3,
                          max_cam_states=max_cam_states)
    traj = Trajectory()
    t0 = 1.0 + 0.37 * seq
    frame_dt = imu_per_frame * dT
    if stop is not None:
        traj = StopProfile(traj, t0, frame_dt, stop["every"], stop["frames"], stop["ramp"])
    # landmark shell 3..15 m around the circle (cylindrical)
    ang = rng.uniform(0, 2 * np.pi, n_landmarks)
    rad = traj.r + rng.uniform(3.0, 15.0, n_landmarks)
    hgt = rng.uniform(-6.0, 6.0, n_landmarks)
    pts_G = np.stack([rad * np.cos(ang), rad * np.sin(ang), hgt], axis=1)
    sig = pixel_sigma / INTRINSICS[0]
    tracked = []  # landmark indices currently tracked (order = front-end order)
    next_id = 1
    lm_id = {}
    frames = []
    for k in range(n_frames):
        t = t0 + k * frame_dt
        C, p = cam_pose(traj, t, cam)
        vis, xn, yn = visible(C, p, pts_G)
        still = [i for i in tracked if vis[i] and rng.random() > dropout]
        cand = np.flatnonzero(vis)
        rng.shuffle(cand)
        still_set = set(still)
        new = []
        for i in cand:
            if len(still) + len(new) >= max_features:
                break
            if i not in still_set and i not in lm_id:
                new.append(int(i))
        for i in new:
            lm_id[i] = next_id
            next_id += 1
        # a landmark that was dropped keeps its old id entry so it is never re-detected

        def obs_of(idx):
            idx = np.asarray(idx, dtype=int)
            o = np.stack([xn[idx], yn[idx]], axis=1) if len(idx) else np.zeros((0, 2))
            return o + sig * rng.standard_normal(o.shape)

        fr = {"imu": [] if k == 0 else imu_samples(traj, t - frame_dt, imu_per_frame, dT, rng,
                                                   imu_noise_frac, noise["Q_imu"]),
              "state_id": k, "time": t,
              "update": (obs_of(still), np.array([lm_id[i] for i in still], dtype=np.uint64)),
              "add": (obs_of(new), np.array([lm_id[i] for i in new], dtype=np.uint64))}
        frames.append(fr)
        tracked = still + new
    return {"camera": cam, "noise": noise, "params": params, "imu_state": true_imu_state(traj, t0),
            "frames": frames, "landmarks": pts_G, "traj": traj, "t0": t0}


def drive(filt, wl, upto=None, marginalize_last=True, prune=True, on_frame=None, prune_redundant=False):
    """Run a workload through any object exposing the MSCKF<_S> surface
    (call order of datasets/asl_msckf.cpp:233-294).  `upto` = number of frames."""
    filt.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
    frames = wl["frames"] if upto is None else wl["frames"][:upto]
    for k, fr in enumerate(frames):
        for (omega, a, dT) in fr["imu"]:
            filt.propagate(omega, a, dT)
        filt.augmentState(fr["state_id"], fr["time"])
        if fr["update"] is not None:
            filt.update(fr["update"][0], fr["update"][1])
        if fr["add"] is not None:
            filt.addFeatures(fr["add"][0], fr["add"][1])
        last = k == len(frames) - 1
        if (not last) or marginalize_last:
            filt.marginalize()
            if prune_redundant:
                filt.pruneRedundantStates()
            if prune:
                filt.pruneEmptyStates()
        if on_frame is not None:
            on_frame(k, filt)
    return filt
