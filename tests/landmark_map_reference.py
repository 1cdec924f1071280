"""Dense fp64 reference of the mapped-landmark update with map uncertainty (msckf_b200_map_landmark_update: the landmark ids
and Sigma_L of msckf_b200_landmark_map).

Observation i of landmark l from clone k has the residual and clone block X_i of the exact-map update
(tests/test_landmark_gpu.py) and the landmark block F_i = J C = -X_i[:, 3:6].  With the true landmark at p_L + dp_l,
dp_l ~ N(0, Sigma_l), the used observations' stacked noise is R (x) I + F Sigma F^T, where F Sigma F^T couples the rows of
one landmark across its clones.  `dense` builds that system; `numpy_update` of tests/test_aid_gpu.py applies it (Joseph form,
the oracle's injection).  `schmidt` is the same update done the long way: x augmented by every dp_l, a joint Joseph update,
the landmarks dropped; `rows` is the engine's compressed row count; `iekf` the iterated form with the map marginalised."""
import numpy as np

from oracle.msckf_numpy import quat_mul, quat_to_rot
from tests.landmark_iter_reference import boxplus, build_update_quat
from tests.test_aid_gpu import numpy_update
from tests.test_landmark_gpu import jacobian, project


def sym(s):
    """3 x 3 from the lower triangle xx, yx, yy, zx, zy, zz"""
    s = np.asarray(s, dtype=np.float64)
    return np.array([[s[0], s[1], s[3]], [s[1], s[2], s[4]], [s[3], s[4], s[5]]])


def tri(S):
    S = np.asarray(S)
    return np.array([S[0, 0], S[1, 0], S[1, 1], S[2, 0], S[2, 1], S[2, 2]])


def dense(P, poses, clone, z, p_L, landmark, Sigma, R, chi2=0.0):
    """(H, r, Rb, F, lm) of the used observations (F [2u, 3] the landmark blocks, lm [u] their landmarks), gamma, flag.
    gamma_i = r^T (X P_kk X^T + F Sigma F^T + R)^-1 r."""
    n = P.shape[0]
    Sg = [sym(s) for s in np.asarray(Sigma).reshape(-1, 6)]
    Hs, rs, Fs, lms, gam, flag = [], [], [], [], [], []
    for k, zi, pl, l in zip(clone, z, p_L, landmark):
        pc, zh = project(poses[k], pl)
        if not (pc[0, 2] > 0 and np.all(np.isfinite(zh))):
            gam.append(np.nan); flag.append(2)
            continue
        r = zi - zh[0]
        X = jacobian(poses[k], pl)
        F = -X[:, 3:6]
        Pk = P[15 + 6 * k:21 + 6 * k, 15 + 6 * k:21 + 6 * k]
        g = float(r @ np.linalg.solve(X @ Pk @ X.T + F @ Sg[l] @ F.T + R, r))
        gam.append(g)
        f = 1 if (chi2 > 0 and g > chi2) else 0
        flag.append(f)
        if f == 0:
            H = np.zeros((2, n))
            H[:, 15 + 6 * k:21 + 6 * k] = X
            Hs.append(H); rs.append(r); Fs.append(F); lms.append(l)
    u = len(Hs)
    H = np.vstack(Hs) if Hs else np.zeros((0, n))
    r = np.concatenate(rs) if rs else np.zeros(0)
    F = np.vstack(Fs) if Fs else np.zeros((0, 3))
    Rb = np.kron(np.eye(u), R)
    for a in range(u):
        for b in range(u):
            if lms[a] == lms[b]:
                Rb[2 * a:2 * a + 2, 2 * b:2 * b + 2] += F[2 * a:2 * a + 2] @ Sg[lms[a]] @ F[2 * b:2 * b + 2].T
    return H, r, Rb, F, np.array(lms, dtype=int), np.array(gam), np.array(flag)


def schmidt(P, imu, poses, H, r, F, lm, Sigma, R):
    """the joint update of (x, dp_0 .. dp_L-1) with the landmarks' prior Sigma, independent of x, in Joseph form; returns
    numpy_update's tuple for the x part (P, imu, poses, NIS, |dx|)"""
    n, L = P.shape[0], len(np.asarray(Sigma).reshape(-1, 6))
    Pa = np.zeros((n + 3 * L, n + 3 * L))
    Pa[:n, :n] = P
    for l, s in enumerate(np.asarray(Sigma).reshape(-1, 6)):
        Pa[n + 3 * l:n + 3 * l + 3, n + 3 * l:n + 3 * l + 3] = sym(s)
    Ha = np.zeros((len(r), n + 3 * L))
    Ha[:, :n] = H
    for a, l in enumerate(lm):
        Ha[2 * a:2 * a + 2, n + 3 * l:n + 3 * l + 3] = F[2 * a:2 * a + 2]
    Rb = np.kron(np.eye(len(r) // 2), R)
    S = Ha @ Pa @ Ha.T + Rb
    K = np.linalg.solve(S, Ha @ Pa).T
    A = np.eye(n + 3 * L) - K @ Ha
    Pn = A @ Pa @ A.T + K @ Rb @ K.T
    dx = (K @ r)[:n]
    imu, poses = inject(imu, poses, dx)
    return Pn[:n, :n], imu, poses, float(r @ np.linalg.solve(S, r)), float(np.linalg.norm(dx))


def inject(imu, poses, dx):
    """numpy_update's state injection of dx"""
    imu, poses = np.array(imu, dtype=np.float64), np.array(poses, dtype=np.float64)
    imu[15:19] = quat_mul(build_update_quat(dx[0:3]), imu[15:19])
    imu[6:9] += dx[3:6]; imu[3:6] += dx[6:9]; imu[9:12] += dx[9:12]; imu[0:3] += dx[12:15]
    return imu, boxplus(poses, dx)


def rows(clone, landmark, flag):
    """rows of the compressed system: per clone min(2 a_k, 6) over the used observations of landmarks seen from one clone,
    plus per group of landmarks with one clone set of >= 2 clones (the input's sets) min(2 used, 6 c)"""
    clone, landmark, flag = np.asarray(clone), np.asarray(landmark), np.asarray(flag)
    sets = {}
    for l in np.unique(landmark):
        sets.setdefault(tuple(sorted(clone[landmark == l])), []).append(l)
    m = 0
    single = {}
    for cs, ls in sets.items():
        used = int(sum(np.sum((landmark == l) & (flag == 0)) for l in ls))
        if len(cs) == 1:
            single[cs[0]] = single.get(cs[0], 0) + used
        else:
            m += min(2 * used, 6 * len(cs))
    return m + sum(min(2 * u, 6) for u in single.values())


def linearise(n, poses, clone, z, p_L, landmark, Sigma, R, used):
    """(H, r, Rb) of the used observations at clone poses `poses` (F at those poses too), or None when one of them is behind
    the camera / not finite"""
    for k, pl in zip(np.asarray(clone)[used], np.asarray(p_L)[used]):
        pc, zh = project(poses[k], pl)
        if not (pc[0, 2] > 0 and np.all(np.isfinite(zh))):
            return None
    sel = np.flatnonzero(used)
    H, r, Rb, _, _, _, _ = dense(np.zeros((n, n)), poses, np.asarray(clone)[sel], np.asarray(z)[sel], np.asarray(p_L)[sel],
                                 np.asarray(landmark)[sel], Sigma, R)
    return H, r, Rb


def iekf(P, imu, poses, clone, z, p_L, landmark, Sigma, R, chi2=0.0, max_iter=1, tol=1e-10):
    """landmark_iter_reference.iekf with the map marginalised at every linearisation (the landmarks stay at p_L)"""
    P = np.asarray(P, dtype=np.float64)
    n = P.shape[0]
    H, r, Rb, _, _, gam, flag = dense(P, poses, clone, z, p_L, landmark, Sigma, R, chi2)
    used = flag == 0
    out = {"gamma": gam, "flag": flag, "used": int(used.sum()), "dof": len(r), "iterations": 0, "converged": 0, "step": 0.0}
    if not used.any():
        return dict(out, P=P.copy(), imu=np.array(imu, float), poses=np.array(poses, float), nis=0.0, applied=0)
    out["nis"] = float(r @ np.linalg.solve(H @ P @ H.T + Rb, r))
    delta = np.zeros(n)
    it = 1
    while True:
        K = np.linalg.solve(H @ P @ H.T + Rb, H @ P).T
        new = K @ (r + H @ delta)
        if it >= max_iter:
            break
        out["step"] = float(np.abs(new - delta).max())
        if out["step"] <= tol:
            out["converged"] = 1
            break
        nxt = linearise(n, boxplus(poses, new), clone, z, p_L, landmark, Sigma, R, used)
        if nxt is None:
            break
        delta = new
        H, r, Rb = nxt
        it += 1
    Pn, imun, posesn, _, _ = numpy_update(P, np.array(imu, float), np.array(poses, float), H, r + H @ delta, Rb)
    return dict(out, P=Pn, imu=imun, poses=posesn, applied=1, iterations=it)


def landmarks_seen_from(rng, poses, clones, depth=(3.0, 12.0)):
    """one landmark position in G that every clone in `clones` sees in front of it (the first clone sets the point; the
    others are checked, and the draw is repeated until they see it at positive depth inside a wide field of view)"""
    while True:
        k0 = clones[0]
        d = rng.uniform(*depth)
        pc = np.array([rng.uniform(-0.3, 0.3) * d, rng.uniform(-0.2, 0.2) * d, d])
        pl = quat_to_rot(poses[k0, 3:7]).T @ pc + poses[k0, 0:3]
        ok = True
        for k in clones[1:]:
            q = quat_to_rot(poses[k, 3:7]) @ (pl - poses[k, 0:3])
            ok &= q[2] > 0.5 and abs(q[0] / q[2]) < 1.5 and abs(q[1] / q[2]) < 1.5
        if ok:
            return pl
