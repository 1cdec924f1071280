"""A dense numpy fp64 reference of one vision update at caller-given feature positions, and a builder of windows of any shape
for it.

The update is the one of the engine's RESIDUALIZE mode (pruneRedundantStates, msckf.h:545-614): per track the residual and the
observability-projected Jacobian of oracle/msckf_numpy.py projected on an orthonormal basis A_j of the left null space of H_f,
the chi-square gate, then the stacked update.  The pixel noise is D_j = diag(u_var, v_var, u_var, ...) per track, projected to
R_o,j = A_j^T D_j A_j:
  * gamma_j = r~^T (H_o,j P H_o,j^T + u_var I)^-1 r~, accepted when gamma_j < chi2_table[L_j] (msckf.h:1103-1124: u_var only,
    whatever v_var is);
  * isotropic noise (u_var = v_var = sigma^2): every R_o,j is sigma^2 I whatever basis is used, so the accepted rows H_o, r_o are
    compressed by an economic QR H_o = Q_1 T (any such Q_1 gives the same update, R_n = sigma^2 I) and the update uses the
    innovation S = T P T^T + sigma^2 I >= sigma^2 I: no P^-1, so the filter's own ill-conditioned P works;
  * anisotropic noise, m <= n: the plain update in the full measurement space, R_o = blkdiag(R_o,j);
  * anisotropic noise, m > n: the exact-subspace update (DESIGN.md 3, 4.4): Q_1 an orthonormal basis of span(E_15) + range(H_o),
    taken from the singular vectors of [E_15 | H_c] above the rank gap (rank_of), T = Q_1^T H_o, r = Q_1^T r_o,
    R = Q_1^T R_o Q_1 summed track by track (R_o itself is never formed).  A Householder Q_1 would add basis vectors outside
    that span at a clone no track sees, and under anisotropic noise they move the update;
  * P+ in Joseph form, dx = K r, and the state injection of msckf_numpy (IMU quaternion not renormalised, clones' are);
  * the rank of the compressed system: m when m <= n (the reference's Q is square), else the numerical rank of
    [E_15 | H_o(:, 15:)] (DESIGN.md 4.4), split in the gap of its singular values (null directions ~1e-14, or ~1e-8 at poses rounded to fp32;
    real ones ~1e-2, ~1e-4 when only a few tracks make m just above n).

State layout (msckf_b200_get_state): imu [29] p, v, b_g, b_a, g, q_IG, p_null, v_null, q_null; clone poses [M, 7] p_C_G, q_CG.
A track is a dict: idx [L] ascending window positions, obs [L, 2] normalised coordinates, pfg [3] feature position."""
from types import SimpleNamespace

import numpy as np
import scipy.linalg as sla

from msckf_mono_b200 import synth
from oracle.msckf_numpy import MSCKF as NumpyMSCKF, CamState, chi2_table, quat_mul, quat_normalized, quat_to_rot, skew

CHI2 = chi2_table(np.float64)  # CHI2[L]: the gate of a track of L observations (table[dof + 1], dof = L - 1)
NOISE = synth.euroc_noise(isotropic=True, tuned=True)
SIGMA2 = float(NOISE["u_var_prime"])
# a wide circle (30 m radius, 0.5 m/s) sampled at 100 Hz, 10 readings per clone: consecutive clones 5 cm apart, and a window of
# 137 clones turns by 0.23 rad only, so a landmark in front of the middle clone of a 98-clone track is in front of all of them
TRAJ = synth.Trajectory(radius=30.0)
T0, DT, READINGS_PER_CLONE = 1.0, 0.01, 10
# singular values of the column-normalised [E_15 | H_c] relative to the largest: the null directions lie below NULL_SV, the
# real ones above REAL_SV (asserted); the rank counts those above their geometric mean
NULL_SV, REAL_SV = 1e-7, 1e-5
# ceilings that separate rounding from a wrong result in the engine's agreement with this reference, whatever was measured
# (tests/test_update_shapes_gpu.py, tests/test_update_noise_gpu.py); dx, P, state, gamma, p_f_G as measured there
CONTRACT = {"float64": {"dx": 1e-4, "P": 1e-5, "state": 1e-4, "gamma": 1e-6, "p_f_G": 1e-6},
            "float32": {"dx": 5e-2, "P": 1e-3, "state": 5e-2, "gamma": 1e-2, "p_f_G": 1e-2}}


def pixel_noise(ratio, dtype=np.float64):
    """(u_var, v_var) as a filter of `dtype` holds them: u_var = SIGMA2 and v_var = ratio * SIGMA2, or EuRoC's own pair
    (v_var 0.6 % above u_var: f_u > f_v) for ratio "euroc"; rounded to dtype, in fp64"""
    if ratio == "euroc":
        nz = synth.euroc_noise(tuned=True)
        u, v = nz["u_var_prime"], nz["v_var_prime"]
    else:
        u, v = SIGMA2, ratio * SIGMA2
    return float(np.dtype(dtype).type(u)), float(np.dtype(dtype).type(v))


def setup(noise=None):
    """(camera, noise, params, imu_state) of a filter for the builder: EuRoC camera, pixel noise (u_var, v_var) (default
    isotropic, SIGMA2)"""
    params = synth.euroc_params(max_track_length=98, min_track_length=2, max_cam_states=192)
    nz = NOISE if noise is None else dict(NOISE, u_var_prime=noise[0], v_var_prime=noise[1])
    return synth.euroc_camera(), nz, params, synth.true_imu_state(TRAJ, T0)


def head_lengths(case, M):
    """(track lengths, outlier tracks) that place the first 15 stacked rows (the ones the engine keeps explicit when m > n)
    across track edges in a given way, followed by long tracks so that m > n:
      "edge": five 3-observation tracks (3 rows each), row 15 on a track edge;
      "straddle": 5-observation tracks (7 rows each), the third track holds rows 14 .. 20;
      "whole": a 12-observation track (21 rows) holds the whole head;
      "pairs": fifteen 2-observation tracks (one row each);
      "gated": the second of three 5-observation tracks gated out (an outlier), the fourth track reaches row 15"""
    head = {"edge": [3] * 5, "straddle": [5] * 3, "whole": [12], "pairs": [2] * 15, "gated": [5] * 3}[case]
    return head + [M, M - 1, M // 2, M] * 2, ((1,) if case == "gated" else ())


HEAD_CASES = ["edge", "straddle", "whole", "pairs", "gated"]


def readings(k):
    """[READINGS_PER_CLONE, 7] noise-free IMU readings (omega, a, dT) between clone k - 1 and clone k"""
    rs = synth.imu_samples(TRAJ, T0 + (k - 1) * READINGS_PER_CLONE * DT, READINGS_PER_CLONE, DT, np.random.default_rng(0), 0.0)
    return np.array([np.concatenate([w, a, [dt]]) for w, a, dt in rs])


def numpy_filter(M, dtype=np.float64, drop_null_rows=True, noise=None):
    """msckf_numpy's filter driven through the builder's M clones"""
    f = NumpyMSCKF(dtype, drop_null_rows=drop_null_rows)
    f.initialize(*setup(noise))
    for k in range(M):
        if k:
            for r in readings(k):
                f.propagate(r[0:3], r[3:6], r[6])
        f.augmentState(k, T0 + k * READINGS_PER_CLONE * DT)
    return f


def numpy_state(f):
    """(P, imu [29], poses [M, 7]) of a msckf_numpy filter in the engine's layout, fp64"""
    s = f.imu
    imu = np.concatenate([s[k] for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG", "p_I_G_null", "v_I_G_null", "q_IG_null")])
    poses = np.array([np.concatenate([c.p_C_G, c.q_CG]) for c in f.cam_states]).reshape(-1, 7)
    return f.getCovariance().astype(np.float64), imu.astype(np.float64), poses.astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------ tracks
def landmark(rng, pose):
    """a point 3..8 m in front of a clone (p_C_G, q_CG)"""
    d = rng.uniform(3.0, 8.0)
    pc = np.array([rng.uniform(-0.3, 0.3) * d, rng.uniform(-0.2, 0.2) * d, d])
    return quat_to_rot(pose[3:7]).T @ pc + pose[0:3]


def project(pose, p):
    pc = quat_to_rot(pose[3:7]) @ (p - pose[0:3])
    return pc, pc[0:2] / pc[2]


def make_tracks(rng, poses, lengths, unseen=(), outliers=(), noise=np.sqrt(SIGMA2) / 10, offset=0.01):
    """tracks of the given lengths over the clones of `poses` except `unseen` (lengths clamped to the clones left).  Track j takes
    its clones by style j % 4: contiguous from a position past 0, contiguous up to the newest clone, a random non-contiguous
    subset, contiguous from clone 0.  The landmark sits in front of the middle clone of the subset (positive depth in every
    observing clone is asserted); the observations carry pixel noise of `noise` (below the model's sigma, so that clean tracks
    pass the gate by far), tracks j in `outliers` a gross error in every third observation; p_f_G is the landmark plus a
    centimetre-level offset."""
    vis = np.array([k for k in range(len(poses)) if k not in set(unseen)])
    out = []
    for j, L in enumerate(lengths):
        L = min(L, len(vis))
        style = j % 4
        if style == 0:
            pos = np.arange(L) + (int(rng.integers(1, len(vis) - L + 1)) if len(vis) > L else 0)
        elif style == 1:
            pos = np.arange(len(vis) - L, len(vis))
        elif style == 2:
            pos = np.sort(rng.choice(len(vis), L, replace=False))
        else:
            pos = np.arange(L)
        idx = vis[pos]
        p = landmark(rng, poses[idx[len(idx) // 2]])
        obs = np.empty((L, 2))
        for i, k in enumerate(idx):
            pc, obs[i] = project(poses[k], p)
            assert pc[2] > 1.0, (j, k, pc)
        obs += noise * rng.normal(size=obs.shape)
        if j in outliers:
            obs[1::3] += 0.1 * rng.choice([-1.0, 1.0], size=obs[1::3].shape)
        out.append({"idx": idx.astype(np.int32), "obs": obs, "pfg": p + offset * rng.normal(size=3) / np.sqrt(3)})
    return out


def gate_delta(L, dtype):
    """how far threshold_tracks places a track of L observations from its threshold, relative to CHI2[L]: fp64 1e-9 (over
    100 x the engine's measured gamma error); fp32 0.4 x the relative distance from CHI2[L] to the nearer neighbouring entry
    (CHI2[L - 1], or CHI2[L + 1] below L = 98), so that a gate reading a neighbouring entry flips one track of each pair"""
    if np.dtype(dtype) == np.float64:
        return 1e-9
    near = [CHI2[L - 1]] + ([CHI2[L + 1]] if L + 1 < len(CHI2) else [])
    return 0.4 * min(abs(x / CHI2[L] - 1) for x in near)


def threshold_tracks(rng, P, imu, poses, lengths, sides, dtype, delta):
    """(tracks, gamma): tracks of the given lengths (make_tracks' clone subsets and landmarks, p_f_G the landmark itself) whose
    reference gamma is CHI2[L] (1 + side delta), side -1 (accepted) or +1 (rejected) per track, delta a scalar or one per
    track; as an engine of `dtype` receives them (observations and p_f_G rounded to dtype, in fp64), at the covariance P and
    state (imu, poses) the update will see.  The observations are the exact projections of p_f_G plus s d, d a random
    pixel-noise direction: H_o and A_j do not depend on z, so gamma(s) = s^2 gamma(1).  s is rescaled to the target and the
    gamma of the rounded track recomputed, four times (rounding to fp32 moves gamma by ~1e-5 of itself)"""
    tracks = rounded(make_tracks(rng, poses, lengths, noise=0.0, offset=0.0), dtype)
    delta = np.broadcast_to(np.asarray(delta, dtype=np.float64), (len(tracks),))
    target = np.array([CHI2[len(t["idx"])] * (1 + s * d) for t, s, d in zip(tracks, sides, delta)])
    exact = [np.array([project(poses[k], t["pfg"])[1] for k in t["idx"]]) for t in tracks]
    dirs = [np.sqrt(SIGMA2) * rng.normal(size=x.shape) for x in exact]
    scale = np.ones(len(tracks))
    for it in range(5):
        cur = [dict(t, obs=(x + s * d).astype(dtype).astype(np.float64)) for t, x, d, s in zip(tracks, exact, dirs, scale)]
        gam, _ = gate(P, project_tracks(imu, poses, cur), cur)
        scale = scale * np.sqrt(target / gam)
    return cur, gam


def threshold_sides(lengths):
    """a pair of tracks per length: -1 (just below the threshold: accepted) / +1 (just above: rejected), the pair in the order
    (-1, +1) at even lengths and (+1, -1) at odd ones, so that accepted and rejected tracks alternate and a CTA of two tracks
    holds one of each, in both orders; (track lengths, sides)"""
    return [L for L in lengths for _ in (0, 1)], [s if L % 2 == 0 else -s for L in lengths for s in (-1, 1)]


def threshold_pairs(rng, P, imu, poses, lengths, dtype):
    """(tracks, gamma, target, sides) of threshold_sides' pairs of the given lengths at gate_delta's distance from CHI2[L]"""
    ls, sides = threshold_sides(lengths)
    delta = np.array([gate_delta(L, dtype) for L in ls])
    tracks, gam = threshold_tracks(rng, P, imu, poses, ls, sides, dtype, delta)
    target = np.array([CHI2[L] * (1 + s * d) for L, s, d in zip(ls, sides, delta)])
    return tracks, gam, target, np.array(sides)


def pack(tracks, dtype):
    """(obs_offset, obs, clone_index, p_f_G) arrays of capi.TrackBatch"""
    off = np.concatenate([[0], np.cumsum([len(t["idx"]) for t in tracks])]).astype(np.int32)
    obs = np.concatenate([t["obs"] for t in tracks]).astype(dtype) if tracks else np.zeros((0, 2), dtype)
    idx = np.concatenate([t["idx"] for t in tracks]).astype(np.int32) if tracks else np.zeros(0, np.int32)
    pfg = np.array([t["pfg"] for t in tracks], dtype=dtype).reshape(-1, 3)
    return off, obs, idx, pfg


def rounded(tracks, dtype):
    """the tracks as an engine of `dtype` receives them (observations and p_f_G rounded to dtype), in fp64"""
    return [dict(t, obs=t["obs"].astype(dtype).astype(np.float64), pfg=t["pfg"].astype(dtype).astype(np.float64)) for t in tracks]


# --------------------------------------------------------------------------------------------------------------- reference
def _view(imu, poses):
    """a msckf_numpy filter object holding just what its residual / Jacobian helpers read: the clones and g"""
    f = NumpyMSCKF(np.float64)
    f.imu = {"g": np.asarray(imu[12:15], dtype=np.float64)}
    f.cam_states = [CamState(np.asarray(p[0:3], np.float64), np.asarray(p[3:7], np.float64), 0.0, k) for k, p in enumerate(poses)]
    return f


def project_tracks(imu, poses, tracks):
    """per track (H_o,j [2L-3, n], r_o,j [2L-3], A_j [2L, 2L-3]) on msckf_numpy's null-space basis A_j (any orthonormal one
    would do, with R_o,j = A_j^T D_j A_j formed on the same basis), or None for a track of one observation (no row left after
    the projection)"""
    f = _view(imu, poses)
    out = []
    for t in tracks:
        idx = [int(k) for k in t["idx"]]
        if len(idx) < 2:
            out.append(None)
            continue
        r = f._calc_residual(np.asarray(t["pfg"], np.float64), [f.cam_states[k] for k in idx], list(t["obs"]))
        H_o, A = f._calc_meas_jacobian(np.asarray(t["pfg"], np.float64), idx)
        out.append((H_o, A.T @ r, A))
    return out


def noise_block(A, u_var, v_var):
    """R_o,j = A_j^T D_j A_j, D_j = diag(u_var, v_var, u_var, ...)"""
    d = np.tile([u_var, v_var], A.shape[0] // 2)
    return A.T @ (d[:, None] * A)


def gate(P, blocks, tracks, sigma2=SIGMA2):
    """(gamma [N] (NaN for a track of one observation), accepted [N] bool); sigma2 is u_var, whatever v_var is"""
    gam = np.full(len(blocks), np.nan)
    for j, (b, t) in enumerate(zip(blocks, tracks)):
        if b is None:
            continue
        H, r = b[0], b[1]
        cols = np.concatenate([np.arange(15 + 6 * k, 21 + 6 * k) for k in np.unique(t["idx"])])
        Hc = H[:, cols]
        gam[j] = float(r @ np.linalg.solve(Hc @ P[np.ix_(cols, cols)] @ Hc.T + sigma2 * np.eye(len(r)), r))
    lengths = np.array([len(t["idx"]) for t in tracks])
    acc = np.array([np.isfinite(g) and g < CHI2[L] for g, L in zip(gam, lengths)], dtype=bool)
    return gam, acc


def compressed_update(P, H_o, r_o, sigma2=SIGMA2):
    """(dx, P+) of the stacked system through its economic QR (Joseph form)"""
    n = P.shape[0]
    Q1, T = sla.qr(H_o, mode="economic")
    rn = Q1.T @ r_o
    S = T @ P @ T.T + sigma2 * np.eye(T.shape[0])
    K = sla.solve(S, T @ P, assume_a="pos").T
    A = np.eye(n) - K @ T
    Pn = A @ P @ A.T + sigma2 * (K @ K.T)
    return K @ rn, (Pn + Pn.T) / 2


def dense_update(P, H_o, r_o, sigma2=SIGMA2):
    """(dx, P+) of the uncompressed m x m innovation form (Joseph form): the cross-check of compressed_update.  sigma2 is the
    measurement noise: a scalar (sigma2 I) or the m x m matrix"""
    n, m = P.shape[0], H_o.shape[0]
    iso = np.ndim(sigma2) == 0
    S = H_o @ P @ H_o.T + (sigma2 * np.eye(m) if iso else sigma2)
    K = sla.solve(S, H_o @ P, assume_a="pos").T
    A = np.eye(n) - K @ H_o
    Pn = A @ P @ A.T + (sigma2 * (K @ K.T) if iso else K @ sigma2 @ K.T)
    return K @ r_o, (Pn + Pn.T) / 2


def subspace_update(P, H_o, r_o, Ro_blocks, Q1):
    """(dx, P+) of the exact-subspace update (Joseph form): the stacked system projected on the orthonormal basis Q1 [m, rank]
    (rank_of), its noise Q1^T R_o Q1 formed from each track's rows of Q1 and its R_o,j (Ro_blocks, in stacking order)"""
    R = np.zeros((Q1.shape[1], Q1.shape[1]))
    off = 0
    for Rb in Ro_blocks:
        Qb = Q1[off:off + Rb.shape[0]]
        R += Qb.T @ Rb @ Qb
        off += Rb.shape[0]
    return dense_update(P, Q1.T @ H_o, Q1.T @ r_o, (R + R.T) / 2)


def inject(imu, poses, dx):
    """the state injection of msckf_numpy (msckf.h:1373-1391): IMU quaternion not renormalised, clone quaternions renormalised"""
    buq = lambda d: NumpyMSCKF._build_update_quat(SimpleNamespace(S=np.float64, dt=np.float64), d)  # noqa: E731
    imu, poses = imu.copy(), poses.copy()
    imu[15:19] = quat_mul(buq(dx[0:3]), imu[15:19])
    imu[6:9] += dx[3:6]; imu[3:6] += dx[6:9]; imu[9:12] += dx[9:12]; imu[0:3] += dx[12:15]
    for k in range(len(poses)):
        poses[k, 3:7] = quat_normalized(quat_mul(buq(dx[15 + 6 * k:18 + 6 * k]), poses[k, 3:7]))
        poses[k, 0:3] += dx[18 + 6 * k:21 + 6 * k]
    return imu, poses


def rank_of(H_o, basis=False):
    """(rank, relative singular values of the column-normalised [E_15 | H_c] or None when m <= n); with basis, also an
    orthonormal basis [m, rank] of span(E_15) + range(H_o): its leading left singular vectors (None when m <= n)"""
    m, n = H_o.shape
    if m <= n:
        return (m, None, None) if basis else (m, None)
    B = np.hstack([np.eye(m)[:, :15], H_o[:, 15:]])
    nrm = np.linalg.norm(B, axis=0)
    B = B[:, nrm > 0] / nrm[nrm > 0]  # the columns of a clone no track sees are zero (Gamma's diagonal is exactly 0 there)
    Q, R = sla.qr(B, mode="economic")
    W, s, _ = np.linalg.svd(R)
    s = s / s[0]
    rank = min(int(np.sum(s > np.sqrt(NULL_SV * REAL_SV))), m, n)
    return (rank, s, Q @ W[:, :rank]) if basis else (rank, s)


def reference(P, imu, poses, tracks, noise=None, blocks=None):
    """the whole update on fp64 inputs at pixel noise (u_var, v_var) (default isotropic, SIGMA2; pass the values the filter
    holds, see pixel_noise): dict gamma, accepted, rows [N], m, rank, sv (see rank_of), H_o, r_o and, when a track is
    accepted, dx, P, imu, poses after the update (else P, imu, poses unchanged and dx None)"""
    u_var, v_var = (SIGMA2, SIGMA2) if noise is None else noise
    P = np.asarray(P, np.float64)
    blocks = project_tracks(imu, poses, tracks) if blocks is None else blocks
    gam, acc = gate(P, blocks, tracks, u_var)
    rows = np.array([0 if b is None or not a else b[0].shape[0] for b, a in zip(blocks, acc)], dtype=int)
    n = P.shape[0]
    H_o = np.vstack([b[0] for b, a in zip(blocks, acc) if a]) if acc.any() else np.zeros((0, n))
    r_o = np.concatenate([b[1] for b, a in zip(blocks, acc) if a]) if acc.any() else np.zeros(0)
    out = {"gamma": gam, "accepted": acc, "rows": rows, "m": int(rows.sum()), "H_o": H_o, "r_o": r_o,
           "dx": None, "P": P, "imu": np.asarray(imu, np.float64), "poses": np.asarray(poses, np.float64), "rank": 0, "sv": None}
    if out["m"] and u_var == v_var:
        out["rank"], out["sv"] = rank_of(H_o)
        out["dx"], out["P"] = compressed_update(P, H_o, r_o, u_var)
    elif out["m"]:
        out["rank"], out["sv"], Q1 = rank_of(H_o, basis=True)
        Ro = [noise_block(b[2], u_var, v_var) for b, a in zip(blocks, acc) if a]
        if Q1 is None:
            out["dx"], out["P"] = dense_update(P, H_o, r_o, sla.block_diag(*Ro))
        else:
            out["dx"], out["P"] = subspace_update(P, H_o, r_o, Ro, Q1)
    if out["m"]:
        out["imu"], out["poses"] = inject(np.asarray(imu, np.float64), np.asarray(poses, np.float64), out["dx"])
    return out


def _unprojected(imu, poses, t):
    """(X_j [2L, n], U_j [2L, 3]) of a track: its measurement Jacobian with the observability projection, before the left
    null-space projection (as msckf_numpy's _calc_meas_jacobian forms it), and an orthonormal basis of range(H_f)"""
    g = np.asarray(imu[12:15], np.float64)
    n, L = 15 + 6 * len(poses), len(t["idx"])
    X, Hf = np.zeros((2 * L, n)), np.zeros((2 * L, 3))
    for i, k in enumerate(t["idx"]):
        C = quat_to_rot(poses[k, 3:7])
        d = t["pfg"] - poses[k, 0:3]
        pc = C @ d
        J = np.array([[1.0, 0.0, -pc[0] / pc[2]], [0.0, 1.0, -pc[1] / pc[2]]]) / pc[2]
        A = np.hstack([J @ skew(pc), -J @ C])
        u = np.concatenate([C @ g, skew(d) @ g])
        H = A - np.outer(A @ u, u) / (u @ u)
        Hf[2 * i:2 * i + 2] = -H[:, 3:6]
        X[2 * i:2 * i + 2, 15 + 6 * k:21 + 6 * k] = H
    return X, np.linalg.qr(Hf, mode="complete")[0][:, :3]


def skip_cholesky_pivots(G, thr=1e-9):
    """the relative pivots (pivot / original diagonal) of a Cholesky of G that skips a column whose pivot is not above thr
    times its original diagonal, in column order: the engine's rank decision (DESIGN.md 4.4)"""
    G = np.array(G, dtype=np.float64)
    d0 = np.diag(G).copy()
    piv = np.zeros(len(G))
    for k in range(len(G)):
        p = G[k, k]
        piv[k] = p / d0[k] if d0[k] > 0 else 0.0
        if not (d0[k] > 0 and p > thr * d0[k]):
            G[k, :] = 0.0
            G[:, k] = 0.0
            continue
        col = G[k:, k] / np.sqrt(p)
        G[k:, k:] -= np.outer(col, col)
    return piv


def gram_noise(imu, poses, tracks, ref):
    """the largest rounding-noise pivot of the rank decision evaluated in fp64 in the engine's own Gram form: Gamma =
    [[I, H_h], [H_h^T, Lambda]], Lambda = sum_j X_j^T X_j - Z_j^T Z_j, Z_j = U_j^T X_j over the accepted tracks (DESIGN.md
    4.4), factorised by skip_cholesky_pivots, the pivots beyond the reference's rank; 0 when m <= n (no decision).  The
    Gram form's noise is a property of the formula, not of the kernel that evaluates it: on 130 threshold tracks over 70
    clones it reaches 3e-9 where the reference's own H_o^T H_o gives 5e-10 (tests/test_gate_threshold_cpu.py)"""
    if ref["sv"] is None:
        return 0.0
    n = ref["H_o"].shape[1]
    G = np.zeros((n, n))
    for t, a in zip(tracks, ref["accepted"]):
        if a:
            X, U = _unprojected(imu, poses, t)
            Z = U.T @ X
            G += X.T @ X - Z.T @ Z
    Hh = ref["H_o"][:15, 15:]
    G[:15, :15] = np.eye(15)
    G[:15, 15:] = Hh
    G[15:, :15] = Hh.T
    pv = np.sort(skip_cholesky_pivots(G))[::-1]
    return float(np.abs(pv[ref["rank"]:]).max()) if n > ref["rank"] else 0.0


def gate_margin(ref, tracks):
    """smallest |gamma / threshold - 1| over the tracks with a row (a flag within 10 % of its threshold could flip on rounding)"""
    r = [abs(g / CHI2[len(t["idx"])] - 1) for g, t in zip(ref["gamma"], tracks) if np.isfinite(g)]
    return min(r) if r else np.inf
