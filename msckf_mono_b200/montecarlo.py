"""Monte-Carlo consistency trials of the filter on the synthetic stream (synth.make_stream_workload), measured with NEES on
the device (MSCKFBatch::nees, msckf_b200_batch_nees).

Truth: the stream built with pixel_sigma = 0 and imu_noise_frac = 0.  The generator draws its random numbers whatever the
noise level, so the truth has the same tracks and ids, frame by frame, as the noisy stream.  Truth IMU states come from the
trajectory at each frame's time, truth camera poses per state_id from synth.cam_pose.

Trial k draws from np.random.default_rng([seed, k]) -- its inputs do not depend on how many trials run or on which rank --
and from the noise model the filter is given: pixel noise of variance u_var' / v_var', IMU white noise of std sqrt(Q / dT),
bias random walks of std sqrt(Q_b dT) per reading (the truth biases are recorded per frame), and an initial estimate whose
error is drawn from P0.

Optional position fixes (a GPS or motion-capture stand-in): every `fix_every` frames, after the prune, each trial fuses
z = p_true + N(0, sigma^2 I) into its filter (MSCKFBatch::aidedUpdate, one batched call).  The fix noise of trial k comes from
its own stream np.random.default_rng([seed, k, 1]), so the trial's other inputs are the same with fixes on or off.  The NIS
of the fixes gives a truth-free consistency figure (ANIS against chi^2 with 3 dof per trial).

Optional mapped landmarks (a prior map): every `map_every` frames, after the prune (and after a position fix when both are on),
each trial observes the map -- every `map_stride`-th landmark of the truth stream -- where it is visible from the truth pose of
its newest clone (synth.visible, the stream's own rule), and fuses z = z_true + N(0, diag(u_var', v_var')) with known landmark
positions (MSCKFBatch::landmarkUpdate, one batched call).  The noise of trial k comes from its own stream
np.random.default_rng([seed, k, 2]), so the trial's other inputs are the same with the map on or off.  These map observations
are drawn independently of the tracked-feature pixels of the same landmark in the same image: an idealisation (a real front end
would see one pixel noise in both), which leaves the two measurements uncorrelated.  The NIS of the map updates gives another
truth-free consistency figure (ANIS against chi^2 with 2 dof per used observation).

Optional odometry (wheel or leg odometry, or another tracker's relative motion): every `odo_every` frames, after the prune (and
after a position fix when both are on), each trial fuses ONE stacked update (MSCKFBatch::aidedUpdate(items), one batched call):
the truth body velocity C(q_IG) v_I_G plus N(0, odo_sigma_v^2) per row (rows y, z only with nhc: the rows a non-holonomic
constraint uses; on this trajectory they are not zero, so z is the truth plus noise, not 0), and, once the window holds two
clones, the truth pose of its newest clone relative to the one before plus noise: position N(0, odo_sigma_rel^2 I) in metres,
rotation buildUpdateQuat-style N(0, odo_sigma_rel^2 I) in radians.  The noise of trial k comes from its own stream
np.random.default_rng([seed, k, 3]), 9 standard normals per odometry frame, so the trial's other inputs are the same with
odometry on or off.  The NIS of the stacks gives another truth-free consistency figure (ANIS against chi^2 with the stack's rows).

Optional GNSS (satellite navigation with its antenna off the IMU, and a heading): every `gnss_every` frames, after the odometry,
each trial fuses the truth antenna position p_I_G + C(q_IG)^T lever plus N(0, gnss_sigma^2 I) as ANTENNA_POSITION; every
`heading_every` frames the truth yaw of the IMU axis `heading_axis` plus N(0, heading_sigma^2) as HEADING; both in ONE stacked
update per frame (MSCKFBatch::aidedUpdate(items)).  gnss_delay d > 0 fuses, at frame f, the fix and heading of frame f - d at that
frame's clone (CLONE_ANTENNA_POSITION, CLONE_HEADING, the lever and the axis converted to its camera frame), as a receiver whose
output arrives d images late; an epoch whose clone has left the window is dropped.  gnss_as_position fuses the antenna position
as a plain POSITION fix of the IMU, which shows the lever-arm bias.  The noise of trial k comes from its own streams
np.random.default_rng([seed, k, 6]) (3 standard normals per fix) and [seed, k, 7] (1 per heading), so the trial's other inputs
are the same with GNSS on or off.  The NIS of the stacks gives another truth-free consistency figure.

Optional ranging (UWB-style radio ranges to the surveyed anchors ANCHORS, and a downward rangefinder over the level ground plane
z = plane_height): every `range_every` frames the truth range |p_I_G + C(q_IG)^T range_lever - a| to each anchor plus
N(0, range_sigma^2) as RANGE, and every `plane_every` frames the truth distance along the IMU axis `plane_axis` from
`plane_lever` to the plane plus N(0, plane_sigma^2) as PLANE_RANGE; a frame's ranges and plane range in ONE stacked update.
range_delay d > 0 fuses, at frame f, both of frame f - d at that frame's clone (CLONE_RANGE, CLONE_PLANE_RANGE, the levers and
the axis converted to its camera frame), like gnss_delay.  The noise of trial k comes from its own streams
np.random.default_rng([seed, k, 8]) (one standard normal per anchor) and [seed, k, 9] (1 per plane range), so the trial's other
inputs are the same with ranging on or off.  The NIS of the stacks is recorded and summarised as the GNSS stacks' are.

Error-state convention (the inverse of the filter's state injection q+ = buildUpdateQuat(dtheta) * q): dq = q_true * q_est^-1
with the Hamilton product, dq negated when dq.w < 0, dtheta = -2 vec(dq); every other component is truth - estimate.  Host
vectors here are in the filter's covariance order [dtheta, db_g, dv, db_a, dp, clones (dtheta_C, dp_C)...].
"""
from __future__ import annotations

import math

import numpy as np
from scipy import stats

from . import synth
from .capi import (AID_ANTENNA_POSITION, AID_BODY_VELOCITY, AID_CLONE_ANTENNA_POSITION, AID_CLONE_HEADING,
                   AID_CLONE_PLANE_RANGE, AID_CLONE_RANGE, AID_HEADING, AID_PLANE_RANGE, AID_POSITION, AID_RANGE,
                   AID_RELATIVE_POSE)

COMPONENTS = ("orientation", "position", "pose", "imu", "full")
DOF = {"orientation": 3, "position": 3, "pose": 6, "imu": 15}
# indices of each component in the filter's covariance order (full: the whole state)
BLOCK = {"orientation": [0, 1, 2], "position": [12, 13, 14], "pose": [0, 1, 2, 12, 13, 14], "imu": list(range(15))}


# ---- quaternions (x, y, z, w), Hamilton product, as the filter's quat_mul --------------------------------------------------
def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def quat_inv(q):
    q = np.asarray(q, dtype=np.float64)
    return np.array([-q[0], -q[1], -q[2], q[3]]) / np.dot(q, q)


def quat_error(q_true, q_est):
    """dtheta with q_true = buildUpdateQuat(dtheta) * q_est"""
    d = quat_mul(np.asarray(q_true, dtype=np.float64), quat_inv(q_est))
    return (2.0 if d[3] < 0 else -2.0) * d[:3]


def quat_of_error(dth):
    """the quaternion dq of dtheta (w >= 0): buildUpdateQuat without its renormalisation"""
    v = -0.5 * np.asarray(dth, dtype=np.float64)
    return np.array([v[0], v[1], v[2], np.sqrt(max(0.0, 1.0 - v @ v))])


def quat_to_rot(q):
    """C(q): Eigen's toRotationMatrix, as the filter's quat_to_rot (C(q_CG) maps G to the camera frame)"""
    x, y, z, w = np.asarray(q, dtype=np.float64)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# ---- odometry models (msckf_b200_aid_stack_update's BODY_VELOCITY and RELATIVE_POSE) ---------------------------------------
def body_velocity(imu):
    """v_I = C(q_IG) v_I_G of a 19-double IMU state (p, v, b_g, b_a, g, q_IG)"""
    imu = np.asarray(imu, dtype=np.float64)
    return quat_to_rot(imu[15:19]) @ imu[3:6]


def relative_pose(pose_a, pose_b):
    """(p, q xyzw) of camera pose b relative to camera pose a (each p_C_G (3), q_CG (4)): p = C_a (p_b - p_a), q = q_b * q_a^-1"""
    a, b = np.asarray(pose_a, dtype=np.float64), np.asarray(pose_b, dtype=np.float64)
    return quat_to_rot(a[3:7]) @ (b[0:3] - a[0:3]), quat_mul(b[3:7], quat_inv(a[3:7]))


def odometry_residual(item, imu, poses):
    """r of one BODY_VELOCITY, RELATIVE_POSE, GNSS or range item (a dict as for capi.aid_items) at the state (imu 19+, poses
    [M, 7]), in fp64"""
    z = np.asarray(item["z"], dtype=np.float64)
    if item["model"] in RANGE_MODELS:
        q, p, _ = _range_frame(item, imu, poses)
        if item["model"] in (AID_RANGE, AID_CLONE_RANGE):
            return np.array([z[0] - range_of(p, q, z[4:7], z[1:4])])
        return np.array([z[0] - plane_range_of(p, q, z[1], z[2:5], z[5:8])])
    if item["model"] in GNSS_MODELS:
        q, p, _, rows = _gnss_frame(item, imu, poses)
        if item["model"] in (AID_HEADING, AID_CLONE_HEADING):
            return np.array([wrap_angle(z[0] - heading_of(q, z[1:4]))])
        return (z[0:3] - antenna_position(p, q, z[3:6]))[rows]
    if item["model"] == AID_BODY_VELOCITY:  # the rows of the mask
        return (z - body_velocity(imu))[[j for j in range(3) if (item["a"] >> j) & 1]]
    p, q = relative_pose(poses[item["a"]], poses[item["b"]])
    return np.concatenate([quat_error(z[3:7], q), z[0:3] - p])


def odometry_jacobian(item, imu, poses, n):
    """H [m, n] of one BODY_VELOCITY, RELATIVE_POSE, GNSS or range item in the filter's injection convention, C(q+) = (I -
    [dtheta]x) C(q): the host linearisation of the models msckf_b200_aid_stack_update forms on the device"""
    skew = _skew
    imu, poses = np.asarray(imu, dtype=np.float64), np.asarray(poses, dtype=np.float64)
    if item["model"] in RANGE_MODELS:  # d(C^T v) / dtheta = -C^T [v]x
        q, p, c0 = _range_frame(item, imu, poses)
        C = quat_to_rot(q)
        z = np.asarray(item["z"], dtype=np.float64)
        cp = c0 + 3 if c0 else 12
        H = np.zeros((1, n))
        if item["model"] in (AID_RANGE, AID_CLONE_RANGE):  # u^T d(p + C^T l) with u the unit vector from the anchor
            e = p + C.T @ z[4:7] - z[1:4]
            u = e / np.linalg.norm(e)
            H[0, c0:c0 + 3] = u @ (-C.T @ skew(z[4:7]))
            H[0, cp:cp + 3] = u
            return H
        f = z[5:8] / np.linalg.norm(z[5:8])
        bz = (C.T @ f)[2]
        rho = plane_range_of(p, q, z[1], z[2:5], z[5:8])
        H[0, c0:c0 + 3] = (C.T @ skew(z[2:5] + rho * f))[2] / bz  # through the hit point l + rho f in the body frame
        H[0, cp + 2] = -1.0 / bz
        return H
    if item["model"] in GNSS_MODELS:  # d(C^T l) / dtheta = -C^T [l]x
        q, _, c0, rows = _gnss_frame(item, imu, poses)
        C = quat_to_rot(q)
        z = np.asarray(item["z"], dtype=np.float64)
        if item["model"] in (AID_HEADING, AID_CLONE_HEADING):
            d = C.T @ z[1:4]
            H = np.zeros((1, n))
            H[0, c0:c0 + 3] = np.array([-d[1], d[0], 0.0]) / (d[0] ** 2 + d[1] ** 2) @ (-C.T @ skew(z[1:4]))
            return H
        H = np.zeros((len(rows), n))
        H[:, c0:c0 + 3] = (-C.T @ skew(z[3:6]))[rows]
        cp = c0 + 3 if item["model"] == AID_CLONE_ANTENNA_POSITION else 12
        H[:, cp:cp + 3] = np.eye(3)[rows]
        return H
    if item["model"] == AID_BODY_VELOCITY:
        C = quat_to_rot(imu[15:19])
        rows = [j for j in range(3) if (item["a"] >> j) & 1]
        H = np.zeros((len(rows), n))
        H[:, 0:3] = skew(C @ imu[3:6])[rows]
        H[:, 6:9] = C[rows]
        return H
    a, b = item["a"], item["b"]
    Ca, Cb = quat_to_rot(poses[a, 3:7]), quat_to_rot(poses[b, 3:7])
    ia, ib = 15 + 6 * a, 15 + 6 * b
    H = np.zeros((6, n))
    H[0:3, ia:ia + 3] = -Cb @ Ca.T
    H[0:3, ib:ib + 3] = np.eye(3)
    H[3:6, ia:ia + 3] = skew(Ca @ (poses[b, 0:3] - poses[a, 0:3]))
    H[3:6, ia + 3:ia + 6] = -Ca
    H[3:6, ib + 3:ib + 6] = Ca
    return H


def odometry_items(truth_imu, pose_a, pose_b, noise, sigma_v, sigma_rel, nhc=False):
    """one odometry stack as aid item dicts: the body velocity of truth_imu plus sigma_v noise[0:3] (mask 0b110 with nhc, else
    0b111) and, when pose_a is not None, the pose of pose_b relative to pose_a with position noise sigma_rel noise[3:6] and
    rotation noise sigma_rel noise[6:9]; clones a, b are the window's last two positions (a = -2, b = -1: set by the caller)"""
    mask = 0b110 if nhc else 0b111
    rows = [j for j in range(3) if (mask >> j) & 1]
    items = [{"model": AID_BODY_VELOCITY, "a": mask, "z": body_velocity(truth_imu) + sigma_v * noise[0:3], "R": sigma_v ** 2 * np.eye(len(rows))}]
    if pose_a is not None:
        p, q = relative_pose(pose_a, pose_b)
        q = quat_mul(quat_of_error(sigma_rel * noise[6:9]), q)
        items.append({"model": AID_RELATIVE_POSE, "z": np.concatenate([p + sigma_rel * noise[3:6], q / np.linalg.norm(q)]),
                      "R": sigma_rel ** 2 * np.eye(6)})
    return items


# ---- GNSS models (ANTENNA_POSITION, CLONE_ANTENNA_POSITION, HEADING, CLONE_HEADING) ------------------------------------------
GNSS_MODELS = (AID_ANTENNA_POSITION, AID_CLONE_ANTENNA_POSITION, AID_HEADING, AID_CLONE_HEADING)


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def wrap_angle(x):
    """x wrapped into (-pi, pi]"""
    y = math.remainder(float(x), 2.0 * math.pi)
    return y + 2.0 * math.pi if y <= -math.pi else y


def antenna_position(p, q, lever):
    """p_A_G = p + C(q)^T lever of a body (IMU or camera) at p with orientation q, the lever arm in its frame"""
    return np.asarray(p, dtype=np.float64) + quat_to_rot(q).T @ np.asarray(lever, dtype=np.float64)


def heading_of(q, axis):
    """the yaw in G, atan2(d_y, d_x), of d = C(q)^T axis, the axis in the body frame"""
    d = quat_to_rot(q).T @ np.asarray(axis, dtype=np.float64)
    return math.atan2(d[1], d[0])


def _gnss_frame(item, imu, poses):
    """(q, p, first error-state index of the pose's dtheta, the rows of the mask) of a GNSS item's body"""
    m = item["model"]
    if m in (AID_CLONE_ANTENNA_POSITION, AID_CLONE_HEADING):
        k = item["a"]
        q, p, c0 = poses[k, 3:7], poses[k, 0:3], 15 + 6 * k
    else:
        q, p, c0 = imu[15:19], imu[0:3], 0
    mask = item["b"] if m == AID_CLONE_ANTENNA_POSITION else item.get("a", 0) if m == AID_ANTENNA_POSITION else 1
    return np.asarray(q, dtype=np.float64), np.asarray(p, dtype=np.float64), c0, [j for j in range(3) if (mask >> j) & 1]


def camera_frame(camera, lever=None, axis=None):
    """an IMU-frame lever arm (l_C = C(q_CI) (l_I - p_C_I)) or axis (f_C = C(q_CI) f_I) in the camera frame"""
    C = quat_to_rot(camera["q_CI"])
    if lever is not None:
        return C @ (np.asarray(lever, dtype=np.float64) - np.asarray(camera["p_C_I"], dtype=np.float64))
    return C @ np.asarray(axis, dtype=np.float64)


def gnss_items(truth_imu, camera, noise_p, noise_psi, sigma, lever, sigma_psi, axis, clone=None, as_position=False):
    """the GNSS stack of one epoch as aid item dicts, from the truth IMU state of that epoch: with noise_p (3 standard normals)
    the antenna position p_I_G + C(q_IG)^T lever plus sigma noise_p, with noise_psi (1) the yaw of the IMU axis `axis` plus
    sigma_psi noise_psi.  clone = k fuses both at clone k (the lever and the axis in its camera frame); as_position fuses the
    antenna position as a plain POSITION fix (the lever ignored: the bias it leaves is the point)"""
    imu = np.asarray(truth_imu, dtype=np.float64)
    items = []
    if noise_p is not None:
        z = antenna_position(imu[0:3], imu[15:19], lever) + sigma * np.asarray(noise_p)
        R = sigma ** 2 * np.eye(3)
        if as_position:
            items.append({"model": AID_POSITION, "z": z, "R": R})
        elif clone is None:
            items.append({"model": AID_ANTENNA_POSITION, "a": 0b111, "z": np.r_[z, lever], "R": R})
        else:
            items.append({"model": AID_CLONE_ANTENNA_POSITION, "a": clone, "b": 0b111,
                          "z": np.r_[z, camera_frame(camera, lever=lever)], "R": R})
    if noise_psi is not None:
        psi = wrap_angle(heading_of(imu[15:19], axis) + sigma_psi * float(np.asarray(noise_psi).ravel()[0]))
        R = np.array([[sigma_psi ** 2]])
        if clone is None:
            items.append({"model": AID_HEADING, "z": np.r_[psi, axis], "R": R})
        else:
            items.append({"model": AID_CLONE_HEADING, "a": clone, "z": np.r_[psi, camera_frame(camera, axis=axis)], "R": R})
    return items


# ---- range models (RANGE, CLONE_RANGE, PLANE_RANGE, CLONE_PLANE_RANGE) --------------------------------------------------------
RANGE_MODELS = (AID_RANGE, AID_CLONE_RANGE, AID_PLANE_RANGE, AID_CLONE_PLANE_RANGE)
# the ranging scene around the synthetic circle (radius 2 m about the origin, heights within +-0.2 m): four surveyed anchors, not
# coplanar, and a level ground plane below the trajectory.  The synthetic IMU's x axis points up: a downward beam is -x.
ANCHORS = np.array([[5.0, 5.0, -1.0], [-5.0, 5.0, 2.0], [-5.0, -5.0, -1.0], [5.0, -5.0, 2.0]])
PLANE_HEIGHT = -1.5
PLANE_AXIS = (-1.0, 0.0, 0.0)


def range_of(p, q, lever, anchor):
    """|p + C(q)^T lever - anchor|: the range from an antenna at lever in the frame of a body at p with orientation q"""
    return float(np.linalg.norm(antenna_position(p, q, lever) - np.asarray(anchor, dtype=np.float64)))


def plane_range_of(p, q, h, lever, axis):
    """the distance along axis (body frame, any length) from a sensor at lever in the body frame to the plane {x : x_z = h}:
    (h - (p + C^T lever)_z) / b_z with b = C^T axis / |axis| (negative when the plane is behind the sensor)"""
    axis = np.asarray(axis, dtype=np.float64)
    b = quat_to_rot(q).T @ (axis / np.linalg.norm(axis))
    return float((h - antenna_position(p, q, lever)[2]) / b[2])


def _range_frame(item, imu, poses):
    """(q, p, first error-state index of the pose's dtheta) of a range item's body"""
    if item["model"] in (AID_CLONE_RANGE, AID_CLONE_PLANE_RANGE):
        k = item["a"]
        return np.asarray(poses[k, 3:7], dtype=np.float64), np.asarray(poses[k, 0:3], dtype=np.float64), 15 + 6 * k
    return np.asarray(imu[15:19], dtype=np.float64), np.asarray(imu[0:3], dtype=np.float64), 0


def range_items(truth_imu, camera, noise_r, noise_h, sigma, lever, sigma_h, h, plane_lever, axis, clone=None, anchors=ANCHORS):
    """the ranging stack of one epoch as aid item dicts, from the truth IMU state of that epoch: with noise_r (one standard
    normal per anchor) the range from the antenna at lever (IMU frame) to each anchor plus sigma noise_r, with noise_h (1) the
    distance along axis from plane_lever (IMU frame) to the plane z = h plus sigma_h noise_h.  clone = k fuses them at clone k
    (the levers and the axis in its camera frame)"""
    imu = np.asarray(truth_imu, dtype=np.float64)
    p, q = imu[0:3], imu[15:19]
    items = []
    if noise_r is not None:
        lv = lever if clone is None else camera_frame(camera, lever=lever)
        for a, nr in zip(np.asarray(anchors, dtype=np.float64), np.asarray(noise_r).ravel()):
            z = np.r_[range_of(p, q, lever, a) + sigma * nr, a, lv]
            if clone is None:
                items.append({"model": AID_RANGE, "z": z, "R": np.array([[sigma ** 2]])})
            else:
                items.append({"model": AID_CLONE_RANGE, "a": clone, "z": z, "R": np.array([[sigma ** 2]])})
    if noise_h is not None:
        rho = plane_range_of(p, q, h, plane_lever, axis) + sigma_h * float(np.asarray(noise_h).ravel()[0])
        R = np.array([[sigma_h ** 2]])
        if clone is None:
            items.append({"model": AID_PLANE_RANGE, "z": np.r_[rho, h, plane_lever, axis], "R": R})
        else:
            items.append({"model": AID_CLONE_PLANE_RANGE, "a": clone,
                          "z": np.r_[rho, h, camera_frame(camera, lever=plane_lever), camera_frame(camera, axis=axis)], "R": R})
    return items


# ---- states: {"imu": 19 doubles (p, v, b_g, b_a, g, q_IG), "poses": [M, 7] (p_C_G, q_CG) or None} ----------------------
def error_state(truth, est):
    """truth - estimate in the filter's covariance order (15, or 15 + 6M when both carry poses)"""
    t, e = np.asarray(truth["imu"], dtype=np.float64), np.asarray(est["imu"], dtype=np.float64)
    out = [quat_error(t[15:19], e[15:19]), t[6:9] - e[6:9], t[3:6] - e[3:6], t[9:12] - e[9:12], t[0:3] - e[0:3]]
    if truth.get("poses") is not None and est.get("poses") is not None:
        for pt, pe in zip(np.asarray(truth["poses"], dtype=np.float64), np.asarray(est["poses"], dtype=np.float64)):
            out += [quat_error(pt[3:7], pe[3:7]), pt[0:3] - pe[0:3]]
    return np.concatenate(out)


def _apply(base, e, sign):
    b = np.asarray(base["imu"], dtype=np.float64).copy()
    e = np.asarray(e, dtype=np.float64)
    out = b.copy()
    dq = quat_of_error(e[0:3])
    out[15:19] = quat_mul(dq, b[15:19]) if sign > 0 else quat_mul(quat_inv(dq), b[15:19])
    for dst, src in ((6, 3), (3, 6), (9, 9), (0, 12)):
        out[dst:dst + 3] = b[dst:dst + 3] + sign * e[src:src + 3]
    poses = None
    if base.get("poses") is not None:
        poses = np.asarray(base["poses"], dtype=np.float64).copy()
        for k in range(len(poses)):
            ek = e[15 + 6 * k:21 + 6 * k]
            dq = quat_of_error(ek[0:3])
            poses[k, 3:7] = quat_mul(dq, poses[k, 3:7]) if sign > 0 else quat_mul(quat_inv(dq), poses[k, 3:7])
            poses[k, 0:3] = poses[k, 0:3] + sign * ek[3:6]
    return {"imu": out, "poses": poses}


def perturb(est, e):
    """the truth whose error against est is e: error_state(perturb(est, e), est) == e"""
    return _apply(est, e, +1)


def estimate_of(truth, e):
    """the estimate whose error against truth is e: error_state(truth, estimate_of(truth, e)) == e"""
    return _apply(truth, e, -1)


def imu_vector(s):
    """19 doubles from a synth state dict"""
    return np.concatenate([np.asarray(s[k], dtype=np.float64) for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG")])


def imu_dict(v):
    v = np.asarray(v, dtype=np.float64)
    return {"p_I_G": v[0:3], "v_I_G": v[3:6], "b_g": v[6:9], "b_a": v[9:12], "g": v[12:15], "q_IG": v[15:19]}


# ---- truth and trials ------------------------------------------------------------------------------------------------------
def make_truth(n_frames=200, seq=0, max_features=60, max_track_length=20, max_cam_states=20, noise=None, stop=None):
    """the noise-free stream, with the truth IMU state per frame (zero biases) and the truth camera pose per state_id.
    stop = dict(every, frames, ramp): the trajectory stops (synth.StopProfile), and "frame_class" holds per frame the class of
    the interval since the previous frame: "stationary" (at rest all through), "ramp" or "cruise" (frame 0: None)."""
    wl = synth.make_stream_workload(n_frames=n_frames, seq=seq, max_features=max_features, max_track_length=max_track_length,
                                    max_cam_states=max_cam_states, pixel_sigma=0.0, imu_noise_frac=0.0, stop=stop)
    wl["noise"] = synth.euroc_noise(tuned=True) if noise is None else noise
    traj, cam = wl["traj"], wl["camera"]
    wl["truth_imu"] = np.array([imu_vector(synth.true_imu_state(traj, fr["time"])) for fr in wl["frames"]])
    poses = []
    for fr in wl["frames"]:
        C, p = synth.cam_pose(traj, fr["time"], cam)
        poses.append(np.concatenate([p, synth.rot_to_quat(C)]))
    wl["truth_pose"] = np.array(poses)  # row = state_id (= frame index)
    if stop is not None:
        fr = wl["frames"]
        wl["frame_class"] = [None] + [traj.frame_class(fr[k - 1]["time"], fr[k]["time"]) for k in range(1, len(fr))]
    return wl


def map_observations(truth, frame, stride):
    """(map indices, noise-free normalised coordinates) of the map landmarks visible from the truth camera pose of `frame`"""
    C, p = synth.cam_pose(truth["traj"], truth["frames"][frame]["time"], truth["camera"])
    pts = truth["landmarks"][::stride]
    vis, xn, yn = synth.visible(C, p, pts)
    idx = np.flatnonzero(vis)
    return idx, np.stack([xn[idx], yn[idx]], axis=1)


def make_trial(truth, k, seed=0, fix_every=0, fix_sigma=1.0, map_every=0, map_stride=20, odo_every=0, map_start=0, map_sigma=0.0,
               map_clones=1, gnss_every=0, heading_every=0, range_every=0, plane_every=0, range_start=0, gnss_start=0):
    """trial k's inputs: the truth stream with noise drawn from the filter's model; records the injected noise.  With
    fix_every > 0, "fixes" holds per frame None or the noisy position fix z = p_true + N(0, fix_sigma^2 I).  With
    map_every > 0, "maps" holds per frame None or (map indices, p_L [n, 3], noisy z [n, 2]) of the visible map landmarks, None
    before frame map_start (the map noise of those frames is still drawn, so a frame's map is the same for every map_start).  With
    odo_every > 0, "odometry" holds per frame None or the 9 standard normals of that frame's odometry noise (odometry_items).
    map_sigma > 0: the trial's map ("map_points", and the p_L of "maps") is the truth map plus N(0, map_sigma^2 I), drawn once
    from np.random.default_rng([seed, k, 4]).  map_clones K > 1 (K <= map_every): a map frame also observes the map from the
    K - 1 frames before it, and its entry gets a fourth array, how many frames back each observation is (0: the newest); their
    pixel noise comes from np.random.default_rng([seed, k, 5]), so the newest frame's noise is the same for every K.  With
    gnss_every > 0, "gnss" holds per frame (the epoch of that frame) None or the 3 standard normals of its antenna-position noise,
    from np.random.default_rng([seed, k, 6]); with heading_every > 0, "heading" holds None or 1 standard normal, from
    np.random.default_rng([seed, k, 7]) (gnss_items).  With range_every > 0, "range" holds per frame None or one standard normal
    per anchor of ANCHORS, from np.random.default_rng([seed, k, 8]); with plane_every > 0, "plane" holds None or 1 standard
    normal, from np.random.default_rng([seed, k, 9]) (range_items).  range_start / gnss_start > 0: the "range" and "plane" /
    "gnss" and "heading" entries of the epochs before that frame are None (their noise is still drawn, so an epoch's noise is the
    same for every start)."""
    rng = np.random.default_rng([seed, k])
    nz = truth["noise"]
    Q = np.asarray(nz["Q_imu"], dtype=np.float64)
    P0 = np.asarray(nz["initial_imu_covar"], dtype=np.float64)
    Lw, Lbg, La, Lba = (np.linalg.cholesky(Q[i:i + 3, i:i + 3]) for i in (0, 3, 6, 9))
    e0 = np.linalg.cholesky(P0 + 0.0) @ rng.standard_normal(15)
    imu0 = imu_vector(truth["imu_state"])
    est0 = estimate_of({"imu": imu0, "poses": None}, e0)["imu"]
    b_g, b_a = np.zeros(3), np.zeros(3)
    frames, bias, inj = [], [], {"pixel": [], "gyro": [], "accel": [], "bias_g": [], "bias_a": [], "dT": []}
    su, sv = np.sqrt(nz["u_var_prime"]), np.sqrt(nz["v_var_prime"])
    for fr in truth["frames"]:
        imu = []
        for (w, a, dT) in fr["imu"]:
            nw, na = Lw @ rng.standard_normal(3) / np.sqrt(dT), La @ rng.standard_normal(3) / np.sqrt(dT)
            imu.append((np.asarray(w) + b_g + nw, np.asarray(a) + b_a + na, dT))
            dbg, dba = Lbg @ rng.standard_normal(3) * np.sqrt(dT), Lba @ rng.standard_normal(3) * np.sqrt(dT)
            b_g, b_a = b_g + dbg, b_a + dba
            inj["gyro"].append(nw); inj["accel"].append(na); inj["bias_g"].append(dbg); inj["bias_a"].append(dba); inj["dT"].append(dT)
        out = {"imu": imu, "state_id": fr["state_id"], "time": fr["time"]}
        for key in ("update", "add"):
            z, ids = fr[key]
            n = rng.standard_normal(z.shape) * np.array([su, sv])
            out[key] = (z + n, ids)
            inj["pixel"].append(n)
        frames.append(out)
        bias.append(np.concatenate([b_g, b_a]))
    inj = {key: (np.concatenate(v) if key == "pixel" else np.array(v)) for key, v in inj.items()}
    out = {"k": k, "frames": frames, "imu_state": imu_dict(est0), "e0": e0, "truth_bias": np.array(bias), "injected": inj}
    if fix_every > 0:
        frng = np.random.default_rng([seed, k, 1])
        out["fixes"] = [truth["truth_imu"][f][0:3] + fix_sigma * frng.standard_normal(3) if (f + 1) % fix_every == 0 else None
                        for f in range(len(truth["frames"]))]
    if map_every > 0:
        assert 1 <= map_clones <= map_every, "map_clones must be 1 .. map_every (no clone is observed twice)"
        mrng = np.random.default_rng([seed, k, 2])
        crng = np.random.default_rng([seed, k, 5])  # pixel noise of the older clones' map observations (map_clones > 1)
        su, sv = np.sqrt(nz["u_var_prime"]), np.sqrt(nz["v_var_prime"])
        pts = truth["landmarks"][::map_stride]
        if map_sigma > 0:
            pts = pts + map_sigma * np.random.default_rng([seed, k, 4]).standard_normal(pts.shape)
            out["map_points"] = pts
        out["maps"] = []
        for f in range(len(truth["frames"])):
            if (f + 1) % map_every:
                out["maps"].append(None)
                continue
            idx, z = map_observations(truth, f, map_stride)
            z = z + mrng.standard_normal(z.shape) * np.array([su, sv])
            if map_clones > 1:
                parts = [(idx, z, np.zeros(len(idx), dtype=int))]
                for j in range(1, min(map_clones, f + 1)):
                    ij, zj = map_observations(truth, f - j, map_stride)
                    parts.append((ij, zj + crng.standard_normal(zj.shape) * np.array([su, sv]), np.full(len(ij), j)))
                idx, z, ago = (np.concatenate([q[i] for q in parts]) for i in range(3))
                out["maps"].append((idx, pts[idx], z.reshape(-1, 2), ago) if f >= map_start else None)
            else:
                out["maps"].append((idx, pts[idx], z) if f >= map_start else None)
    if odo_every > 0:
        orng = np.random.default_rng([seed, k, 3])
        out["odometry"] = [orng.standard_normal(9) if (f + 1) % odo_every == 0 else None for f in range(len(truth["frames"]))]
    if gnss_every > 0:
        grng = np.random.default_rng([seed, k, 6])
        out["gnss"] = [grng.standard_normal(3) if (f + 1) % gnss_every == 0 else None for f in range(len(truth["frames"]))]
    if heading_every > 0:
        hrng = np.random.default_rng([seed, k, 7])
        out["heading"] = [hrng.standard_normal(1) if (f + 1) % heading_every == 0 else None for f in range(len(truth["frames"]))]
    if range_every > 0:
        rrng = np.random.default_rng([seed, k, 8])
        out["range"] = [rrng.standard_normal(len(ANCHORS)) if (f + 1) % range_every == 0 else None for f in range(len(truth["frames"]))]
    if plane_every > 0:
        prng = np.random.default_rng([seed, k, 9])
        out["plane"] = [prng.standard_normal(1) if (f + 1) % plane_every == 0 else None for f in range(len(truth["frames"]))]
    for key, start in (("gnss", gnss_start), ("heading", gnss_start), ("range", range_start), ("plane", range_start)):
        if key in out and start > 0:
            out[key] = [None if f < start else x for f, x in enumerate(out[key])]
    return out


def truth_imu_of(truth, trial, frame):
    """truth IMU state (19) of a trial at a frame: the trajectory's, with the trial's biases"""
    v = truth["truth_imu"][frame].copy()
    v[6:12] = trial["truth_bias"][frame]
    return v


# ---- summaries ---------------------------------------------------------------------------------------------------------------
def trial_record(nees_rows, pos_err2, fix_nis=(), map_rows=(), odo_rows=(), map_first=None, gnss_rows=None, range_rows=None,
                 range_first=None, gnss_first=None, frame_class=None, standstill_rows=None):
    """one trial's per-frame NEES (list of result dicts), squared position errors, the NIS of its position fixes, of its
    map updates (result dicts of landmark_update: nis, dof, used, applied, plus the observation count n) and of its odometry
    stacks (result dicts of aid_stack_update: nis, dof, applied), as plain lists; map_first (a dict of plain numbers: frame,
    squared position error before and after, nis, dof, iterations, converged) describes the first map update; gnss_rows
    (result dicts of aid_stack_update, dof 0 for an epoch whose clone had left the window) the GNSS stacks, range_rows (the
    same) the ranging stacks; range_first / gnss_first (as map_first) the first ranging / GNSS stack; frame_class (the truth's
    per frame, with stops) and standstill_rows (per frame from frame 1 on, result dicts of standstill_update)"""
    rec = _trial_record(nees_rows, pos_err2, fix_nis, map_rows, odo_rows)
    if frame_class is not None:
        rec["frame_class"] = list(frame_class)
    if standstill_rows is not None:
        rec["standstill"] = {k: [float(r[k]) if k in ("nis", "scatter") else int(r[k]) for r in standstill_rows]
                             for k in ("nis", "dof", "applied", "outcome", "scatter")}
    for key, first in (("map_first", map_first), ("range_first", range_first), ("gnss_first", gnss_first)):
        if first is not None:
            rec[key] = dict(first)
    for key, rows in (("gnss", gnss_rows), ("range", range_rows)):
        if rows is not None:
            rec[key] = {k: [float(r[k]) if k == "nis" else int(r[k]) for r in rows] for k in ("nis", "dof", "applied", "status")}
            rec[key].update(_fault_counts(rows))
    return rec


def _fault_counts(rows):
    """the injected faults of a trial's stacks (each row's "faults": the item indices made faulty) and what became of them: with
    FDE item states (row "items"), faults excluded, clean items excluded, faults missed (used in an applied stack), stacks
    rejected (outcome 2 or 3); without, a fault in an applied stack is missed and a stack not applied is rejected"""
    c = {"injected": 0, "faults_excluded": 0, "clean_excluded": 0, "faults_missed": 0, "stacks_rejected": 0}
    for r in rows:
        faults = set(r.get("faults", ()))
        c["injected"] += len(faults)
        if "items" in r:
            for j, it in enumerate(r["items"]):
                c["faults_excluded" if j in faults else "clean_excluded"] += it["state"] == 1
                c["faults_missed"] += j in faults and it["state"] == 0
            c["stacks_rejected"] += r["outcome"] in (2, 3)
        elif r["dof"] > 0:
            c["faults_missed"] += len(faults) if r["applied"] else 0
            c["stacks_rejected"] += r["status"] == 0 and not r["applied"]
    return c


def _trial_record(nees_rows, pos_err2, fix_nis, map_rows, odo_rows):
    return {"nees": {c: [float(r[c]) for r in nees_rows] for c in COMPONENTS},
            "dim": {c: [int(r["dim_full"]) if c == "full" else DOF[c] for r in nees_rows] for c in COMPONENTS},
            "first_bad_pivot": [int(r["first_bad_pivot"]) for r in nees_rows],
            "pos_err2": [float(x) for x in pos_err2],
            "fix_nis": [float(x) for x in fix_nis],
            "map": {key: [float(r[key]) if key == "nis" else int(r[key]) for r in map_rows]
                    for key in ("nis", "dof", "used", "applied", "n") + (CONS_KEYS if map_rows and "wrong" in map_rows[0] else ())},
            "odometry": {key: [float(r[key]) if key == "nis" else int(r[key]) for r in odo_rows] for key in ("nis", "dof", "applied")}}


# per map update with wrong matches injected or a consensus: wrong matches, those left out of the update (any flag but 0: excluded
# by consensus, gated out or behind the camera), right ones, those used (flag 0), and the consensus status (-1: none ran)
CONS_KEYS = ("wrong", "wrong_excluded", "right", "right_kept", "cons_status")


def chi2_bounds(total_dof, n, lo=0.025, hi=0.975):
    """two-sided 95 % bounds of the ANEES of n trials with total_dof degrees of freedom in all: chi2_{total}(q) / n"""
    return float(stats.chi2.ppf(lo, total_dof) / n), float(stats.chi2.ppf(hi, total_dof) / n)


def summarize(records):
    """records {trial: trial_record}: per component, ANEES per frame with its 95 % chi^2 bounds, the run's mean ANEES and the
    fraction of frames inside the bounds; the position RMSE over trials per frame and over the run"""
    keys = sorted(records)
    N = len(keys)
    nf = len(records[keys[0]]["pos_err2"])
    out = {"trials": N, "frames": nf, "components": {}}
    for c in COMPONENTS:
        V = np.array([records[k]["nees"][c] for k in keys])
        D = np.array([records[k]["dim"][c] for k in keys])
        anees, lo, hi, inside = [], [], [], []
        for f in range(nf):
            if not np.all(np.isfinite(V[:, f])) or D[:, f].sum() == 0:
                anees.append(float("nan")); lo.append(float("nan")); hi.append(float("nan")); inside.append(False)
                continue
            a = float(V[:, f].mean())
            b = chi2_bounds(int(D[:, f].sum()), N)
            anees.append(a); lo.append(b[0]); hi.append(b[1]); inside.append(b[0] <= a <= b[1])
        fin = [a for a in anees if np.isfinite(a)]
        out["components"][c] = {"anees": anees, "lower": lo, "upper": hi,
                                "mean_anees": float(np.mean(fin)) if fin else float("nan"),
                                "mean_dof": float(D.mean()),
                                "frames_inside": float(np.mean(inside)), "frames_finite": len(fin)}
    E = np.array([records[k]["pos_err2"] for k in keys])
    out["pos_rmse"] = [float(x) for x in np.sqrt(E.mean(axis=0))]
    out["pos_rmse_run"] = float(np.sqrt(E.mean()))
    F = np.array([records[k].get("fix_nis", []) for k in keys], dtype=np.float64)
    if F.size:  # ANIS of the position fixes: 3 dof per trial and fix
        lo, hi = chi2_bounds(3 * N, N)
        anis = F.mean(axis=0)
        out["fixes"] = {"anis": [float(a) for a in anis], "lower": lo, "upper": hi, "dof": 3, "mean_anis": float(anis.mean()),
                        "fixes_inside": float(np.mean((anis >= lo) & (anis <= hi)))}
    mp = [records[k].get("map") for k in keys]
    if all(m is not None and len(m["nis"]) for m in mp):  # ANIS of the map updates: 2 dof per used observation
        V = np.array([m["nis"] for m in mp]); D = np.array([m["dof"] for m in mp])
        anis, lo, hi = V.sum(axis=0) / N, [], []
        for d in D.sum(axis=0):
            b = chi2_bounds(int(d), N) if d > 0 else (float("nan"), float("nan"))
            lo.append(b[0]); hi.append(b[1])
        inside = [lo_ <= a <= hi_ for a, lo_, hi_ in zip(anis, lo, hi)]
        tot = chi2_bounds(int(D.sum()), N * len(anis))
        n_obs = sum(sum(m["n"]) for m in mp)
        out["map"] = {"anis": [float(a) for a in anis], "lower": lo, "upper": hi, "dof": [int(d) for d in D.sum(axis=0)],
                      "mean_anis": float(V.sum() / (N * len(anis))), "mean_dof": float(D.sum() / (N * len(anis))),
                      "run_bounds": list(tot), "updates_inside": float(np.mean(inside)),
                      "applied": float(np.mean([a for m in mp for a in m["applied"]])),
                      "observations": int(n_obs), "gated": float(1.0 - sum(sum(m["used"]) for m in mp) / max(n_obs, 1))}
    for key in ("map_first", "range_first", "gnss_first"):
        mf = [records[k].get(key) for k in keys]
        if not all(m is not None for m in mf):
            continue
        # the first map update, ranging or GNSS stack: position error before / after, its ANIS, the IMU-state ANEES after
        f0 = mf[0]["frame"]
        d = int(sum(m["dof"] for m in mf))
        imu = out["components"]["imu"]
        out[key] = {"frame": int(f0), "pos_rmse_before": float(np.sqrt(np.mean([m["pos_err2_before"] for m in mf]))),
                    "pos_rmse_after": float(np.sqrt(np.mean([m["pos_err2_after"] for m in mf]))),
                    "anis": float(sum(m["nis"] for m in mf) / N), "mean_dof": d / N,
                    "bounds": list(chi2_bounds(d, N)) if d > 0 else [float("nan")] * 2,
                    "imu_anees": imu["anees"][f0], "imu_bounds": [imu["lower"][f0], imu["upper"][f0]],
                    "iterations": float(np.mean([m["iterations"] for m in mf])),
                    "converged": float(np.mean([m["converged"] for m in mf]))}
    od = [records[k].get("odometry") for k in keys]
    if all(o is not None and len(o["nis"]) for o in od):  # ANIS of the odometry stacks: the stack's rows per trial and update
        V = np.array([o["nis"] for o in od]); D = np.array([o["dof"] for o in od])
        anis, dof = V.sum(axis=0) / N, D.sum(axis=0)
        lo, hi = zip(*[chi2_bounds(int(d), N) for d in dof])
        out["odometry"] = {"anis": [float(a) for a in anis], "lower": list(lo), "upper": list(hi), "dof": [int(d) for d in dof],
                           "mean_anis": float(V.sum() / V.size), "mean_dof": float(D.sum() / D.size),
                           "run_bounds": list(chi2_bounds(int(D.sum()), V.size)),
                           "updates_inside": float(np.mean([l_ <= a <= h_ for a, l_, h_ in zip(anis, lo, hi)])),
                           "applied": float(np.mean([a for o in od for a in o["applied"]]))}
    if all("frame_class" in records[k] for k in keys):  # the stops: position-error growth over each, and standstill detection
        out["stops"] = stop_summary([records[k] for k in keys])
    for key in ("gnss", "range"):  # ANIS of the GNSS and of the ranging stacks: the stack's rows per trial and epoch fused
        gn = [records[k].get(key) for k in keys]
        if not all(g is not None and len(g["nis"]) for g in gn):
            continue
        V = np.array([g["nis"] for g in gn]); D = np.array([g["dof"] for g in gn])
        A = np.array([g["applied"] for g in gn])
        fused = (D > 0) & np.isfinite(V)  # (a dropped epoch, or status 1 / 2: no NIS)
        used = fused & (A > 0)  # (a stack the gate or FDE rejected is not in the ANIS)
        V, D = np.where(used, V, 0.0), np.where(used, D, 0)
        n_used, dof = used.sum(axis=0), D.sum(axis=0)
        keep = n_used > 0
        anis = V.sum(axis=0)[keep] / n_used[keep]
        lo, hi = zip(*[chi2_bounds(int(d), int(c)) for d, c in zip(dof[keep], n_used[keep])]) if keep.any() else ((), ())
        out[key] = {"anis": [float(a) for a in anis], "lower": list(lo), "upper": list(hi), "dof": [int(d) for d in dof[keep]],
                    "mean_anis": float(V.sum() / max(used.sum(), 1)), "mean_dof": float(D.sum() / max(used.sum(), 1)),
                    "run_bounds": list(chi2_bounds(int(D.sum()), int(used.sum()))) if used.any() else [float("nan")] * 2,
                    "updates_inside": float(np.mean([l_ <= a <= h_ for a, l_, h_ in zip(anis, lo, hi)])) if keep.any() else float("nan"),
                    "applied": float(A[fused].mean()) if fused.any() else 0.0,
                    "degenerate": int(sum(s == 2 for g in gn for s in g["status"])),
                    **{c: int(sum(g.get(c, 0) for g in gn)) for c in ("injected", "faults_excluded", "clean_excluded", "faults_missed",
                                                                      "stacks_rejected")}}
    return out


def stop_summary(recs):
    """Over trial records with frame classes: the stops (maximal runs of stationary frames), the mean growth of the position
    error |e| over a stop (from the frame before it to its last frame), and with standstill rows the fraction of frames
    detected (outcome 0) per frame class and the ANIS of the applied stacks against the 9-dof run bounds"""
    cls = recs[0]["frame_class"]
    stops, f = [], 1
    while f < len(cls):
        if cls[f] == "stationary":
            g = f
            while g + 1 < len(cls) and cls[g + 1] == "stationary":
                g += 1
            stops.append((f, g))
            f = g + 1
        else:
            f += 1
    growth = [float(np.sqrt(r["pos_err2"][b]) - np.sqrt(r["pos_err2"][a - 1])) for r in recs for a, b in stops]
    out = {"stops": [list(s) for s in stops], "frames": {c: int(sum(x == c for x in cls)) for c in ("stationary", "ramp", "cruise")},
           "pos_err_growth_per_stop": float(np.mean(growth)) if growth else float("nan")}
    if all("standstill" in r for r in recs):
        det = {c: [] for c in ("stationary", "ramp", "cruise")}
        for r in recs:
            for f, o in enumerate(r["standstill"]["outcome"], start=1):
                det[cls[f]].append(o == 0)
        out["detected"] = {c: float(np.mean(v)) if v else float("nan") for c, v in det.items()}
        V = np.array([x for r in recs for x, a in zip(r["standstill"]["nis"], r["standstill"]["applied"]) if a])
        out["applied"] = int(V.size)
        out["anis"] = float(V.mean()) if V.size else float("nan")
        out["run_bounds"] = list(chi2_bounds(9 * int(V.size), int(V.size))) if V.size else [float("nan")] * 2
        out["dof"] = 9
    return out


# ---- the batched run ---------------------------------------------------------------------------------------------------------
def map_call(tr, f, fi, uncertain, S):
    """one filter's map observations at frame fi: (state_ids, z, p_L) for landmark_update or, uncertain, (state_ids, landmark,
    z, p_L, Sigma) for map_update with each distinct landmark once and Sigma = S; only clones still in the window; None when
    nothing is left"""
    m = tr["maps"][fi]
    idx, p, z = m[0], m[1], m[2]
    ago = m[3] if len(m) > 3 else np.zeros(len(idx), dtype=int)
    ids = np.array([tr["frames"][fi - a]["state_id"] for a in ago], dtype=np.int64)
    keep = np.isin(ids, f.getCamStates()["state_id"]) if len(m) > 3 else np.ones(len(idx), dtype=bool)
    if not keep.any():
        return None
    ids, idx, p, z = ids[keep], idx[keep], p[keep], z[keep]
    if not uncertain:
        return ids, z, p
    u, first, inv = np.unique(idx, return_index=True, return_inverse=True)
    return ids, inv, z, p[first], np.repeat(S, len(u), axis=0)


def _epoch_stacks(fb, fs, trs, g, delay, keys, out, items, faults=None, fde=None, iterate=None):
    """one batched stack per filter of the epoch g = f - delay when a trial input of `keys` (two noise lists of make_trial) has
    noise there: items(g, noise of keys[0], noise of keys[1], clone) with clone None at delay 0, else the window position of
    the epoch's clone; a filter whose epoch clone has left the window sends nothing and records dof 0.  faults(i, g, items), when
    given, makes some of filter i's items faulty in place and returns their indices (kept as the row's "faults"); fde, when
    given, sends the stacks through fault detection and exclusion; iterate (max_iter, tol), when given, iterates them.  Appends
    each filter's result to out[i]."""
    noise = [tuple(tr[key][g] if key in tr else None for key in keys) for tr in trs] if g >= 0 else []
    if g < 0 or not any(x is not None for x in noise[0]):
        return
    stacks = []
    for f, tr, (n_a, n_b) in zip(fs, trs, noise):
        clone = None
        if delay:
            ids = list(f.getCamStates()["state_id"])
            if tr["frames"][g]["state_id"] not in ids:  # the epoch's clone has left the window
                stacks.append(None)
                continue
            clone = ids.index(tr["frames"][g]["state_id"])
        stacks.append(items(g, n_a, n_b, clone))
    bad = [faults(i, g, s) if faults is not None and s is not None else [] for i, s in enumerate(stacks)]
    kw = {} if iterate is None else {"max_iter": iterate[0], "tol": iterate[1]}
    for i, r in enumerate(fb.aid_stack_update(stacks, **kw) if fde is None else fb.aid_stack_update(stacks, fde=fde, **kw)):
        out[i].append({"nis": 0.0, "dof": 0, "applied": 0, "status": 0} if r is None else dict(r, faults=bad[i]))


def run(trials, truth, dtype=np.float64, seed=0, on_frame=None, fix_every=0, fix_sigma=1.0, map_every=0, map_stride=20, map_chi2=0.0,
        odo_every=0, odo_sigma_v=0.05, odo_sigma_rel=0.01, nhc=False, map_start=0, map_iterations=1, map_sigma=0.0,
        map_uncertain=False, map_clones=1, gnss_every=0, gnss_sigma=0.1, gnss_lever=(0.0, 0.0, 0.0), gnss_delay=0,
        gnss_as_position=False, heading_every=0, heading_sigma=0.01, heading_axis=(1.0, 0.0, 0.0), range_every=0, range_sigma=0.1,
        range_lever=(0.0, 0.0, 0.0), range_delay=0, plane_every=0, plane_sigma=0.02, plane_height=PLANE_HEIGHT, plane_axis=PLANE_AXIS,
        plane_lever=(0.0, 0.0, 0.0), range_outlier_rate=0.0, range_outlier_bias=1.0, gnss_outlier_rate=0.0, gnss_outlier_jump=5.0,
        fde_alpha=0.0, fde_max_exclude=2, range_start=0, gnss_start=0, aid_iterations=1, aid_tol=1e-10, map_outlier_rate=0.0,
        map_consensus=0, map_consensus_thresh=13.8, map_min_inliers=6, standstill=None):
    """Trials (indices) as one fully batched MSCKFBatch stream: per frame propagate, augmentState, update / addFeatures,
    marginalize, pruneEmptyStates, [every fix_every frames one batched position fix of standard deviation fix_sigma],
    [every odo_every frames one batched odometry stack (odometry_items)],
    [one batched GNSS stack (gnss_items) in a frame whose epoch f - gnss_delay has an antenna fix (every gnss_every frames,
    lever arm gnss_lever in the IMU frame) or a heading (every heading_every frames, of heading_axis); at the IMU when
    gnss_delay = 0, else at that epoch's clone while it is in the window],
    [one batched ranging stack (range_items) in a frame whose epoch f - range_delay has anchor ranges (every range_every frames,
    antenna at range_lever in the IMU frame, standard deviation range_sigma) or a plane range (every plane_every frames, along
    plane_axis from plane_lever to the plane z = plane_height, standard deviation plane_sigma); at the IMU or the epoch's clone
    as for GNSS; each anchor range made range_outlier_bias m long (NLOS) with probability range_outlier_rate, drawn from the
    stream default_rng([seed, k, 10]) per frame, and each antenna fix moved gnss_outlier_jump m horizontally in a random
    direction with probability gnss_outlier_rate, from [seed, k, 11]; fde_alpha > 0 sends the GNSS and ranging stacks through
    fault detection and exclusion with thresholds capi.fde_thresholds(fde_alpha) and fde_max_exclude (0: the stack gate only),
    fde_alpha = 0 fuses them ungated; range_start / gnss_start > 0 fuse no ranging / GNSS epoch before that frame (the first
    one after it is also recorded on its own, as range_first / gnss_first in trial_record); aid_iterations K > 1 iterates the
    GNSS, ranging and odometry stacks (at most K linearisations, converged at a step <= aid_tol)],
    [every map_every frames from frame map_start on, one batched mapped-landmark update from the newest clone, gated per
    observation at map_chi2 > 0, iterated up to map_iterations linearisations; the map carries N(0, map_sigma^2 I) errors and
    is observed from the map_clones newest clones that are still in the window (make_trial); map_uncertain passes
    Sigma = map_sigma^2 I per landmark (MSCKFBatch::landmarkUpdate over mapObservation / mapLandmark), else the map is taken as
    exact; each map observation is a wrong match with probability map_outlier_rate (its p_L swapped for another map
    landmark's, drawn from the stream default_rng([seed, k, 12]); no draw when the rate is 0), and map_consensus H > 0 selects the
    inliers by a consensus of H hypotheses (threshold map_consensus_thresh, min_inliers map_min_inliers, seed [seed, k, frame])
    before each map update (exact map only); with either, each map row also counts wrong matches left out of the update and right ones used],
    refreshState,
    (standstill = a cfg dict as for capi.standstill_struct: from frame 1 on, before augmentState, one batched standstill update
    of each filter's readings of the frame interval; a filter at rest (outcome 0) skips that frame's augmentState / update /
    addFeatures / marginalize / pruneEmptyStates and keeps propagating; no random draw), then one batched NEES with each filter's truth window looked up by the state_ids of getCamStates.  The first
    map update is also recorded on its own (trial_record's map_first; the state is read just before it).
    Returns ({trial: trial_record}, {trial: final (covariance, imu [29], poses [M, 7])})."""
    from . import engine_filter
    from .capi import AID_POSITION
    from .cview import FilterBatch
    assert not map_uncertain or map_sigma > 0, "map_uncertain needs map_sigma > 0"
    assert not (map_uncertain and map_consensus), "the consensus runs on the exact-map update here"
    assert not (gnss_as_position and gnss_delay), "gnss_as_position fuses at the IMU: no delay"
    trs = [make_trial(truth, k, seed, fix_every, fix_sigma, map_every, map_stride, odo_every, map_start, map_sigma, map_clones,
                      gnss_every, heading_every, range_every, plane_every, range_start=range_start, gnss_start=gnss_start)
           for k in trials]
    iterate = None if aid_iterations == 1 else (int(aid_iterations), float(aid_tol))
    it_kw = {} if iterate is None else {"max_iter": iterate[0], "tol": iterate[1]}
    gnss = [[] for _ in trs] if gnss_every > 0 or heading_every > 0 else None
    ranging = [[] for _ in trs] if range_every > 0 or plane_every > 0 else None
    lever, axis = np.asarray(gnss_lever, dtype=np.float64), np.asarray(heading_axis, dtype=np.float64)
    r_lever, p_lever, p_axis = (np.asarray(v, dtype=np.float64) for v in (range_lever, plane_lever, plane_axis))
    n_fr = len(truth["frames"])
    # NLOS ranges (flags per frame and anchor) and GNSS jumps (flag and direction per frame) of each trial; no draws when off
    r_out = [np.random.default_rng([seed, tr["k"], 10]).random((n_fr, len(ANCHORS))) < range_outlier_rate if range_outlier_rate > 0
             else None for tr in trs]
    g_out = []
    for tr in trs:
        if gnss_outlier_rate > 0:
            rg = np.random.default_rng([seed, tr["k"], 11])
            g_out.append((rg.random(n_fr) < gnss_outlier_rate, rg.uniform(0.0, 2.0 * np.pi, n_fr)))
        else:
            g_out.append(None)

    m_rng = [np.random.default_rng([seed, tr["k"], 12]) if map_outlier_rate > 0 else None for tr in trs]
    m_pts = [tr.get("map_points", truth["landmarks"][::map_stride]) for tr in trs]

    def map_faults(i, o):
        """make some of filter i's map matches wrong in place; their mask"""
        if o is None:
            return None
        n = len(o[0])
        if m_rng[i] is None:
            return np.zeros(n, dtype=bool)
        bad = m_rng[i].random(n) < map_outlier_rate
        pts = m_pts[i]
        for j in np.flatnonzero(bad):
            cur = int(np.flatnonzero(np.all(pts == o[2][j], axis=1))[0])
            o[2][j] = pts[(cur + 1 + int(m_rng[i].integers(len(pts) - 1))) % len(pts)]
        return bad

    def range_faults(i, g, items):
        if r_out[i] is None or not items or items[0]["model"] not in (AID_RANGE, AID_CLONE_RANGE):
            return []
        bad = [j for j in range(len(ANCHORS)) if r_out[i][g, j]]
        for j in bad:
            items[j]["z"] = np.r_[items[j]["z"][0] + range_outlier_bias, items[j]["z"][1:]]
        return bad

    def gnss_faults(i, g, items):
        if g_out[i] is None or not items or items[0]["model"] not in (AID_ANTENNA_POSITION, AID_CLONE_ANTENNA_POSITION, AID_POSITION):
            return []
        flag, ang = g_out[i]
        if not flag[g]:
            return []
        z = np.array(items[0]["z"], dtype=np.float64)
        z[0:2] += gnss_outlier_jump * np.array([np.cos(ang[g]), np.sin(ang[g])])
        items[0]["z"] = z
        return [0]

    fde = None
    if fde_alpha > 0:
        from .capi import fde_thresholds
        fde = {"chi2": fde_thresholds(fde_alpha), "max_exclude": int(fde_max_exclude)}
    S_map = np.tile([map_sigma ** 2, 0.0, map_sigma ** 2, 0.0, 0.0, map_sigma ** 2], (1, 1))
    first = [None for _ in trs]
    first_r = [None for _ in trs] if range_start > 0 else None
    first_g = [None for _ in trs] if gnss_start > 0 else None

    def first_stack(first_x, rows, fi, g, keys, send):
        """send an epoch's stacks; the first one sent is also recorded on its own (the state read just before it)"""
        now = first_x is not None and first_x[0] is None and g >= 0 and any(trs[0][k][g] is not None for k in keys if k in trs[0])
        if now:
            fb.refreshState()
            for i, (f, tr) in enumerate(zip(fs, trs)):
                first_x[i] = {"frame": fi, "pos_err2_before": float(np.sum((truth_imu_of(truth, tr, fi)[0:3] - f.getImuState()["p_I_G"]) ** 2))}
        send()
        if now:
            for i in range(len(trs)):
                r = rows[i][-1]
                first_x[i].update(nis=float(r["nis"]), dof=int(r["dof"]), iterations=int(r.get("iterations", r["applied"])),
                                  converged=int(r.get("converged", 0)))

    R_fix = (fix_sigma ** 2) * np.eye(3)
    still = [[] for _ in trs]
    nis = [[] for _ in trs]
    maps = [[] for _ in trs]
    odo = [[] for _ in trs]
    fs = [engine_filter(dtype) for _ in trs]
    for f, tr in zip(fs, trs):
        f.initialize(truth["camera"], truth["noise"], truth["params"], tr["imu_state"])
    fb = FilterBatch(fs)
    rows = [[] for _ in trs]
    err2 = [[] for _ in trs]
    for fi in range(len(truth["frames"])):
        frs = [tr["frames"][fi] for tr in trs]
        for i, fr in enumerate(frs):
            for (w, a, dT) in fr["imu"]:
                fb.propagate(i, w, a, dT)
        skip = [False] * len(trs)
        if standstill is not None and fi > 0:
            res = fb.standstill_update([np.array([np.r_[w, a, dT] for (w, a, dT) in fr["imu"]]) for fr in frs], standstill)
            for i, r in enumerate(res):
                still[i].append(r)
                skip[i] = r["outcome"] == 0
        if not any(skip):
            fb.augmentState([fr["state_id"] for fr in frs], [fr["time"] for fr in frs])
            for f, fr in zip(fs, frs):
                f.update(*fr["update"])
                f.addFeatures(*fr["add"])
            fb.marginalize()
            fb.pruneEmptyStates()
        elif not all(skip):  # the filters still moving step on their own
            for f, fr, sk in zip(fs, frs, skip):
                if not sk:
                    f.augmentState(fr["state_id"], fr["time"])
                    f.update(*fr["update"])
                    f.addFeatures(*fr["add"])
                    f.marginalize()
                    f.pruneEmptyStates()
        if fix_every > 0 and trs[0]["fixes"][fi] is not None:
            res = fb.aid_update([{"model": AID_POSITION, "z": tr["fixes"][fi], "R": R_fix} for tr in trs])
            for i, r in enumerate(res):
                nis[i].append(r["nis"])
        if odo_every > 0 and trs[0]["odometry"][fi] is not None:
            stacks = []
            for f, tr in zip(fs, trs):
                ids = f.getCamStates()["state_id"]
                pa, pb = (truth["truth_pose"][ids[-2]], truth["truth_pose"][ids[-1]]) if len(ids) >= 2 else (None, None)
                items = odometry_items(truth["truth_imu"][fi], pa, pb, tr["odometry"][fi], odo_sigma_v, odo_sigma_rel, nhc)
                if len(items) > 1:
                    items[1].update(a=len(ids) - 2, b=len(ids) - 1)
                stacks.append(items)
            for i, r in enumerate(fb.aid_stack_update(stacks, **it_kw)):
                odo[i].append(r)
        if gnss is not None:  # the epoch whose GNSS output arrives at this frame
            first_stack(first_g, gnss, fi, fi - gnss_delay, ("gnss", "heading"), lambda: _epoch_stacks(
                fb, fs, trs, fi - gnss_delay, gnss_delay, ("gnss", "heading"), gnss,
                lambda g, n_p, n_psi, clone: gnss_items(truth["truth_imu"][g], truth["camera"], n_p, n_psi, gnss_sigma, lever,
                                                        heading_sigma, axis, clone, gnss_as_position),
                gnss_faults if gnss_outlier_rate > 0 else None, fde, iterate))
        if ranging is not None:  # the epoch whose ranges arrive at this frame
            first_stack(first_r, ranging, fi, fi - range_delay, ("range", "plane"), lambda: _epoch_stacks(
                fb, fs, trs, fi - range_delay, range_delay, ("range", "plane"), ranging,
                lambda g, n_r, n_h, clone: range_items(truth["truth_imu"][g], truth["camera"], n_r, n_h, range_sigma, r_lever,
                                                       plane_sigma, plane_height, p_lever, p_axis, clone),
                range_faults if range_outlier_rate > 0 else None, fde, iterate))
        if map_every > 0 and trs[0]["maps"][fi] is not None:
            obs = [map_call(tr, f, fi, map_uncertain, S_map) for tr, f in zip(trs, fs)]
            track = map_outlier_rate > 0 or map_consensus > 0
            if track:
                obs = [None if o is None else (o[0], o[1], np.array(o[2], dtype=np.float64)) for o in obs]
                wrong = [map_faults(i, o) for i, o in enumerate(obs)]
            if first[0] is None:
                fb.refreshState()
                for i, (f, tr) in enumerate(zip(fs, trs)):
                    first[i] = {"frame": fi, "pos_err2_before": float(np.sum((truth_imu_of(truth, tr, fi)[0:3] - f.getImuState()["p_I_G"]) ** 2))}
            if map_uncertain:
                res = fb.map_update(obs, chi2_obs=map_chi2, max_iter=map_iterations)
            elif map_consensus > 0:
                cons = [{"hypotheses": map_consensus, "thresh": map_consensus_thresh, "min_inliers": map_min_inliers,
                         "seed": int(np.random.SeedSequence([seed, tr["k"], fi]).generate_state(1, np.uint64)[0])} for tr in trs]
                res = fb.landmark_update(obs, chi2_obs=map_chi2, max_iter=map_iterations, consensus=cons)
            else:
                res = fb.landmark_update(obs, chi2_obs=map_chi2, max_iter=map_iterations)
            for i, r in enumerate(res):
                row = {"nis": 0.0, "dof": 0, "used": 0, "applied": 0, "n": 0} if r is None else dict(r, n=len(r["flag"]))
                if track:
                    w = wrong[i] if r is not None else np.zeros(0, dtype=bool)
                    fl = r["flag"] if r is not None else np.zeros(0, dtype=np.int32)
                    row.update(wrong=int(w.sum()), wrong_excluded=int((w & (fl != 0)).sum()), right=int((~w).sum()),
                               right_kept=int((~w & (fl == 0)).sum()),
                               cons_status=int(r["consensus"]["status"]) if r is not None and "consensus" in r else -1)
                maps[i].append(row)
                if first[i]["frame"] == fi:
                    first[i].update({k: (float if k == "nis" else int)(r[k]) if r is not None else 0 for k in ("nis", "dof", "iterations", "converged")})
        fb.refreshState()
        timu, tposes = [], []
        for i, (f, tr) in enumerate(zip(fs, trs)):
            ids = f.getCamStates()["state_id"]
            timu.append(truth_imu_of(truth, tr, fi))
            tposes.append(truth["truth_pose"][ids])
            err2[i].append(float(np.sum((timu[-1][0:3] - f.getImuState()["p_I_G"]) ** 2)))
            for fx in (first, first_r, first_g):
                if fx is not None and fx[i] is not None and fx[i]["frame"] == fi:
                    fx[i]["pos_err2_after"] = err2[i][-1]
        res = fb.nees(timu, tposes)
        for i, r in enumerate(res):
            rows[i].append(r)
        if on_frame is not None:
            on_frame(fi, fs, res)
    fb.close()
    records = {tr["k"]: trial_record(rows[i], err2[i], nis[i], maps[i], odo[i], first[i], None if gnss is None else gnss[i],
                                     None if ranging is None else ranging[i], None if first_r is None else first_r[i],
                                     None if first_g is None else first_g[i], truth.get("frame_class"),
                                     still[i] if standstill is not None else None)
               for i, tr in enumerate(trs)}
    final = {}
    for f, tr in zip(fs, trs):
        s = f.getImuState()
        cs = f.getCamStates()
        final[tr["k"]] = (f.getCovariance(), np.concatenate([s[key] for key in s]), np.hstack([cs["p_C_G"], cs["q_CG"]]))
        f.close()
    return records, final
