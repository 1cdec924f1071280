"""The vision reference under anisotropic pixel noise (tests/vision_reference.py with u_var != v_var), which
tests/test_update_noise_gpu.py holds the engine to, and a numpy restatement of the engine's Gram form (DESIGN.md 4.4) that shows
what those GPU tests can see.

  * the reference reproduces msckf_numpy's exact-subspace update (drop_null_rows=True) where every clone is seen, at EuRoC's
    anisotropy (v_var 0.6 % above u_var), 4 and 1/4, for m <= n and m > n; it does not depend on the null-space basis of any
    track but through the span of the first 15 stacked rows (DESIGN.md 4.4); with u_var = v_var it is the isotropic
    reference, bit for bit;
  * at a clone no track sees, msckf_numpy's unpivoted QR keeps basis vectors outside span(E_15) + range(H_o): its update
    differs from the exact-subspace one (pinned here), and the Gram form on the non-orthonormal basis [E_15 | H_c] with a
    skip-Cholesky rank decision agrees with the reference instead;
  * each of five slips in the terms that carry the noise (a du / dv swap in Y_q, in D2 or in the explicit head rows' noise,
    the head rows' -(A_h^T D U) Z correction dropped, G2 = 2 Z^T Y_q) changes nothing under isotropic noise, and moves dx or P
    past the fp64 contract of the GPU tests at v_var = 4 u_var."""
import numpy as np
import pytest
import scipy.linalg as sla

from oracle.msckf_numpy import quat_to_rot, skew
from tests import vision_reference as vr
from tests.test_update_reference_cpu import CASES, numpy_update, rel

RATIOS = ["euroc", 4.0, 0.25]
# CASES with every clone seen (the 12-clone window without its unseen clone 5): m <= n, m > n, m > n
SEEN = [c[:2] + ((),) + c[3:] for c in CASES]
SLIPS = ["Yq du/dv", "D2 du/dv", "head du/dv", "no s_adu Z", "G2 = 2 Z^T Yq"]


def window(M, lengths, unseen, outliers, noise, seed=None):
    """(msckf_numpy filter at `noise`, P, imu, poses, tracks) of the builder's window"""
    f = vr.numpy_filter(M, noise=noise)
    P, imu, poses = vr.numpy_state(f)
    tracks = vr.make_tracks(np.random.default_rng(M if seed is None else seed), poses, lengths, unseen=unseen, outliers=outliers)
    return f, P, imu, poses, tracks


# ------------------------------------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("M,lengths,unseen,outliers", SEEN)
def test_reference_matches_msckf_numpy_at_anisotropic_noise(M, lengths, unseen, outliers, ratio):
    nz = vr.pixel_noise(ratio)
    assert nz[0] != nz[1]
    f, P, imu, poses, tracks = window(M, lengths, unseen, outliers, nz)
    ref = vr.reference(P, imu, poses, tracks, noise=nz)
    assert vr.gate_margin(ref, tracks) > 0.1
    gam, acc = numpy_update(f, tracks)
    assert np.array_equal(acc, ref["accepted"]) and ref["accepted"].sum() == len(lengths) - len(outliers) - lengths.count(1)
    fin = np.isfinite(gam)
    assert np.array_equal(fin, np.isfinite(ref["gamma"])) and rel(ref["gamma"][fin], gam[fin]) < 1e-12
    lu = f.last_update
    assert ref["m"] == lu["H_o"].shape[0] and ref["rank"] == lu["T_H"].shape[0]
    assert rel(ref["dx"], lu["deltaX"]) < 1e-12 and rel(ref["P"], f.getCovariance()) < 1e-12
    _, imu1, poses1 = vr.numpy_state(f)
    assert np.abs(ref["imu"] - imu1).max() < 1e-12 and np.abs(ref["poses"] - poses1).max() < 1e-12


def rotated(rng, blocks, accepted, head):
    """the blocks on another basis of every track's null space, A_j -> A_j U_j (so H_o,j -> U_j^T H_o,j, r_o,j -> U_j^T r_o,j,
    R_o,j -> U_j^T R_o,j U_j) with U_j random orthogonal; an accepted track with rows on both sides of stacked row `head` is
    rotated within each side only"""
    out, off = [], 0
    for b, a in zip(blocks, accepted):
        if b is None:
            out.append(None)
            continue
        k = len(b[1])
        cut = min(max(head - off, 0), k) if a else 0
        off += k if a else 0
        U = sla.block_diag(*[np.linalg.qr(rng.normal(size=(s, s)))[0] for s in (cut, k - cut) if s])
        out.append((U.T @ b[0], U.T @ b[1], b[2] @ U))
    return out


@pytest.mark.parametrize("M,lengths,unseen,outliers", CASES)
def test_reference_does_not_depend_on_the_null_space_basis_at_anisotropic_noise(M, lengths, unseen, outliers):
    """any orthogonal change of every track's basis changes nothing, as long as the first 15 stacked rows (span(E_15) of the
    exact subspace, the rows the engine keeps explicit when m > n) span what they spanned.  The 12-clone window's first track
    has 17 rows: a rotation across its row 15 moves E_15 out of the span of the original basis and, under anisotropic noise,
    the update with it (pinned)."""
    nz = vr.pixel_noise(4.0)
    _, P, imu, poses, tracks = window(M, lengths, unseen, outliers, nz)
    ref = vr.reference(P, imu, poses, tracks, noise=nz)
    blocks = vr.project_tracks(imu, poses, tracks)
    rng = np.random.default_rng(M + 7)
    fin = np.isfinite(ref["gamma"])
    for head, same in ((15, True), (0, ref["m"] <= P.shape[0] or M != 12)):
        rot = vr.reference(P, imu, poses, tracks, noise=nz, blocks=rotated(rng, blocks, ref["accepted"], head))
        assert np.array_equal(rot["accepted"], ref["accepted"]) and rot["rank"] == ref["rank"]
        assert rel(rot["gamma"][fin], ref["gamma"][fin]) < 1e-12
        d = max(rel(rot["dx"], ref["dx"]), rel(rot["P"], ref["P"]))
        assert d < 1e-12 if same else d > 1e-6, (head, d)


@pytest.mark.parametrize("M,lengths,unseen,outliers", CASES)
def test_isotropic_noise_is_the_isotropic_reference_bit_for_bit(M, lengths, unseen, outliers):
    _, P, imu, poses, tracks = window(M, lengths, unseen, outliers, None)
    a = vr.reference(P, imu, poses, tracks)
    b = vr.reference(P, imu, poses, tracks, noise=(vr.SIGMA2, vr.SIGMA2))
    for k in ("gamma", "accepted", "dx", "P", "imu", "poses"):
        assert np.array_equal(a[k], b[k], equal_nan=k == "gamma"), k


def test_gate_uses_u_var_only():
    """gamma is the same whatever v_var is (msckf.h:1103-1124)"""
    M, lengths, unseen, outliers = CASES[1]
    _, P, imu, poses, tracks = window(M, lengths, unseen, outliers, None)
    g = [vr.reference(P, imu, poses, tracks, noise=(vr.SIGMA2, r * vr.SIGMA2))["gamma"] for r in (1.0, 4.0, 0.25)]
    assert np.array_equal(g[0], g[1], equal_nan=True) and np.array_equal(g[0], g[2], equal_nan=True)


# ------------------------------------------------------------------------------------------- the engine's Gram form, restated
def track_factors(imu, poses, t):
    """(X_j [2L, n], r_j [2L], U_j [2L, 3], A_j [2L, 2L-3]) of a track: the observability-projected 2 x 6 blocks of
    msckf_numpy._calc_meas_jacobian, the raw residual, and the Householder Q of the column-pivoted QR of H_f split into its
    first three columns and the null-space basis (the A_j of vr.project_tracks)"""
    f = vr._view(imu, poses)
    idx = [int(k) for k in t["idx"]]
    L, n = len(idx), 15 + 6 * len(poses)
    X, Hf = np.zeros((2 * L, n)), np.zeros((2 * L, 3))
    g = np.asarray(imu[12:15], np.float64)
    for i, k in enumerate(idx):
        C, pcg = quat_to_rot(poses[k, 3:7]), poses[k, 0:3]
        pc = C @ (t["pfg"] - pcg)
        J = np.array([[1, 0, -pc[0] / pc[2]], [0, 1, -pc[1] / pc[2]]]) / pc[2]
        A = np.hstack([J @ skew(pc), -J @ C])
        u = np.concatenate([C @ g, skew(t["pfg"] - pcg) @ g])
        Hx = A - np.outer(A @ u, u) / np.dot(u, u)
        X[2 * i:2 * i + 2, 15 + 6 * k:21 + 6 * k] = Hx
        Hf[2 * i:2 * i + 2] = -Hx[:, 3:6]
    Q = sla.qr(Hf, mode="full", pivoting=True)[0]
    r = f._calc_residual(np.asarray(t["pfg"], np.float64), [f.cam_states[k] for k in idx], list(t["obs"]))
    return X, r, Q[:, :3], Q[:, 3:]


def skip_cholesky(G, m):
    """indices kept by the natural-order skip Cholesky of Gamma: k is dropped when its pivot (Gamma_kk less its projection on
    the kept columns) is at most 1e-9 Gamma_kk, or when min(m, n) columns are kept already"""
    keep, Lk = [], np.zeros((0, 0))
    for k in range(G.shape[0]):
        if len(keep) >= m or G[k, k] <= 0:
            continue
        l = sla.solve_triangular(Lk, G[keep, k], lower=True) if keep else np.zeros(0)
        d = G[k, k] - l @ l
        if d > 1e-9 * G[k, k]:
            Lk = np.block([[Lk, np.zeros((len(keep), 1))], [l[None, :], np.sqrt(d) * np.ones((1, 1))]])
            keep.append(k)
    return np.array(keep)


def gram_update(P, imu, poses, tracks, accepted, noise, slips=()):
    """(dx, P+, rank) of the engine's update (DESIGN.md 4.4) in numpy fp64: m <= n, every stacked row explicit
    (T = H_o, R = blkdiag(A_j^T D A_j)); m > n, the basis Q'' = [E_15 | H_c] with the first 15 stacked rows explicit (R_hh
    and R_hH = A_h^T D X - (A_h^T D U) Z) and the rest in Gram form,
        Lambda = D1 - Z^T Z,  Psi = D2 - G2,  G2 = Z^T Yq + Yq^T Z,  beta = sum X^T r - Z^T (U^T r),
        Z_j = U_j^T X_j,  Yq_j = U_j^T D X_j - 1/2 (U_j^T D U_j) Z_j,  D1 = sum X^T X,  D2 = sum X^T D X,
    its rank decided by a skip Cholesky of Gamma = Q''^T Q''.  `slips` (from SLIPS) restate the term wrongly."""
    u_var, v_var = noise
    n = P.shape[0]
    fac = [track_factors(imu, poses, t) for t, a in zip(tracks, accepted) if a]
    D = [np.tile([u_var, v_var], len(r) // 2) for _, r, _, _ in fac]
    Ds = [np.tile([v_var, u_var], len(r) // 2) for _, r, _, _ in fac]  # du and dv swapped
    H_o = np.vstack([A.T @ X for X, _, _, A in fac])
    r_o = np.concatenate([A.T @ r for _, r, _, A in fac])
    m = H_o.shape[0]
    dh = Ds if "head du/dv" in slips else D
    if m <= n:
        T, rr, rank = H_o, r_o, m
        R = sla.block_diag(*[A.T @ (d[:, None] * A) for (_, _, _, A), d in zip(fac, dh)])
    else:
        c = n - 15
        # the explicit head rows: stacked row h is column t of track j's A_j
        own = [(j, t) for j, (_, _, _, A) in enumerate(fac) for t in range(A.shape[1])][:15]
        R_hh, R_hH = np.zeros((15, 15)), np.zeros((15, c))
        for h, (j, t) in enumerate(own):
            X, _, U, A = fac[j]
            a = dh[j] * A[:, t]  # D a_h
            for h2, (j2, t2) in enumerate(own):
                if j2 == j:
                    R_hh[h, h2] = a @ A[:, t2]
            R_hH[h] = a @ X[:, 15:]
            if "no s_adu Z" not in slips:
                R_hH[h] -= (a @ U) @ (U.T @ X[:, 15:])
        D1, D2, G1, G2 = (np.zeros((c, c)) for _ in range(4))
        beta = np.zeros(c)
        for (X, r, U, A), d, ds in zip(fac, D, Ds):
            Xc = X[:, 15:]
            Z = U.T @ Xc
            dy = ds if "Yq du/dv" in slips else d
            Yq = U.T @ (dy[:, None] * Xc) - 0.5 * (U.T @ (dy[:, None] * U)) @ Z
            D1 += Xc.T @ Xc
            D2 += Xc.T @ ((ds if "D2 du/dv" in slips else d)[:, None] * Xc)
            G1 += Z.T @ Z
            G2 += 2 * Z.T @ Yq if "G2 = 2 Z^T Yq" in slips else Z.T @ Yq + Yq.T @ Z
            beta += Xc.T @ r - Z.T @ (U.T @ r)
        Lam, Psi = D1 - G1, D2 - G2
        Hh = H_o[:15, 15:]
        Gam = np.block([[np.eye(15), Hh], [Hh.T, Lam]])
        Tpp = np.vstack([H_o[:15], np.hstack([np.zeros((c, 15)), Lam])])
        rpp = np.concatenate([r_o[:15], beta])
        Rpp = np.block([[R_hh, R_hH], [R_hH.T, Psi]])
        keep = skip_cholesky(Gam, min(m, n))
        T, rr, R, rank = Tpp[keep], rpp[keep], Rpp[np.ix_(keep, keep)], len(keep)
    S = T @ P @ T.T + R
    K = sla.solve(S, T @ P).T  # LU: a slip may leave R'' indefinite
    Aj = np.eye(n) - K @ T
    Pn = Aj @ P @ Aj.T + K @ R @ K.T
    return K @ rr, (Pn + Pn.T) / 2, rank


def test_unseen_clone_exact_subspace_differs_from_msckf_numpy_and_matches_the_gram_form():
    """CASES' 12-clone window (clone 5 unseen, m > n) at v_var = 4 u_var: msckf_numpy's QR keeps 6 basis vectors outside
    span(E_15) + range(H_o) per unseen clone, which move its update away from the exact-subspace reference; the Gram form
    restated on [E_15 | H_c] (another basis of the same span, rank by a skip Cholesky) agrees with the reference"""
    M, lengths, unseen, outliers = CASES[2]
    nz = vr.pixel_noise(4.0)
    f, P, imu, poses, tracks = window(M, lengths, unseen, outliers, nz)
    ref = vr.reference(P, imu, poses, tracks, noise=nz)
    assert ref["m"] > P.shape[0]
    _, acc = numpy_update(f, tracks)
    assert np.array_equal(acc, ref["accepted"])
    lu = f.last_update
    assert lu["T_H"].shape[0] == ref["rank"] + 6 * len(unseen)
    d = rel(ref["dx"], lu["deltaX"])
    print(f"unseen clone, v_var = 4 u_var: msckf_numpy's dx differs from the exact-subspace reference by {d:.2e}")
    assert d > 1e-3
    dx, Pn, rank = gram_update(P, imu, poses, tracks, ref["accepted"], nz)
    print(f"Gram form against the reference: dx {rel(dx, ref['dx']):.2e} P {rel(Pn, ref['P']):.2e}")
    assert rank == ref["rank"] and rel(dx, ref["dx"]) < 1e-10 and rel(Pn, ref["P"]) < 1e-10


@pytest.mark.parametrize("ratio", ["euroc", 4.0])
@pytest.mark.parametrize("M,lengths,unseen,outliers", CASES)
def test_gram_form_matches_the_reference(M, lengths, unseen, outliers, ratio):
    nz = vr.pixel_noise(ratio)
    _, P, imu, poses, tracks = window(M, lengths, unseen, outliers, nz)
    ref = vr.reference(P, imu, poses, tracks, noise=nz)
    dx, Pn, rank = gram_update(P, imu, poses, tracks, ref["accepted"], nz)
    assert rank == ref["rank"] and rel(dx, ref["dx"]) < 1e-10 and rel(Pn, ref["P"]) < 1e-10


# (label, M, lengths, unseen, outliers, slips it must expose): an m <= n window, m > n windows with and without an unseen
# clone, and the head-row cases of the GPU tests
DETECT = ([("m<=n", *CASES[0], ["head du/dv"]), ("m>n", *CASES[1], SLIPS), ("m>n unseen", *CASES[2], SLIPS)]
          + [(f"head {h}", 12, *vr.head_lengths(h, 12)[:1], (), vr.head_lengths(h, 12)[1], ["no s_adu Z"])
             for h in vr.HEAD_CASES])


@pytest.mark.parametrize("label,M,lengths,unseen,outliers,expose", DETECT, ids=[d[0] for d in DETECT])
def test_noise_slips_are_invisible_isotropic_and_caught_at_ratio_4(label, M, lengths, unseen, outliers, expose):
    lim = vr.CONTRACT["float64"]
    for ratio in (1.0, 4.0):
        nz = vr.pixel_noise(ratio)
        _, P, imu, poses, tracks = window(M, lengths, unseen, outliers, nz)
        ref = vr.reference(P, imu, poses, tracks, noise=nz)
        dx0, P0, _ = gram_update(P, imu, poses, tracks, ref["accepted"], nz)
        for s in SLIPS:
            dx1, P1, _ = gram_update(P, imu, poses, tracks, ref["accepted"], nz, slips=(s,))
            ddx, dP = rel(dx1, dx0), rel(P1, P0)
            print(f"{label} v_var/u_var {ratio:g}, {s}: dx {ddx:.2e} P {dP:.2e}")
            if ratio == 1.0:
                # the swaps are exact no-ops; the other two differ from the right term by rounding only (the dropped correction
                # is sigma^2 (A_h^T U) Z with A_h^T U ~ 1e-17; Z^T Yq - Yq^T Z = sigma^2 Z^T (I - U^T U) Z / 2 with U^T U = I to
                # 1e-16), which the update's conditioning (the Gram form squares cond(H_c)) carries to below 1e-10 in dx
                assert ddx <= (1e-12 if "du/dv" in s else 1e-10) and dP <= 1e-12, (label, s, ddx, dP)
            elif s in expose:
                assert ddx > lim["dx"] or dP > lim["P"], (label, s, ddx, dP)
