"""The form of the chi-square gate that k_jac evaluates (DESIGN.md 4.3), against the dense gate of tests/vision_reference.py.

A track's gate is gamma = r_o^T (A^T Y A + u_var I)^-1 r_o with Y = H_x P H_x^T, r_o = A^T r and A the trailing 2L - 3 columns
of the orthogonal Q = [U A] of H_f's QR.  The kernel never forms A^T Y A: with M = Y + u_var I = L L^T (SPD), z = A A^T r =
r - U (U^T r), a = L^-1 z, B = L^-1 U and c = B^T a, the Schur complement of (Q^T M Q)^-1 = Q^T M^-1 Q gives

    gamma = a^T a - c^T (B^T B)^-1 c.

Checked in fp64 on isotropic and anisotropic windows (the gate reads u_var only; the window's covariance differs) of 2, 3,
12 and 30 clones, on tracks of 2 to 30 observations with and without gross outliers.  The subtraction cancels little:
a^T a / gamma stays close to 1, so the form loses no precision in fp32 either."""
import numpy as np
import pytest
import scipy.linalg as sla

from tests import vision_reference as vr

WINDOWS = [2, 3, 12, 30]
RATIOS = [1.0, "euroc", 4.0]


def gate_form(P, imu, poses, tracks, u_var):
    """(gamma [N], a^T a [N]) of the Cholesky form; NaN for a track of one observation"""
    f = vr._view(imu, poses)
    # the full Q of H_f's column-pivoted QR in place of its trailing columns: _calc_meas_jacobian then returns Q^T H_x
    f.left_nullspace = lambda H_f: sla.qr(H_f, mode="full", pivoting=True)[0]
    gam, ata = np.full(len(tracks), np.nan), np.full(len(tracks), np.nan)
    for j, t in enumerate(tracks):
        idx = [int(k) for k in t["idx"]]
        if len(idx) < 2:
            continue
        r = f._calc_residual(np.asarray(t["pfg"], np.float64), [f.cam_states[k] for k in idx], list(t["obs"]))
        QtH, Q = f._calc_meas_jacobian(np.asarray(t["pfg"], np.float64), idx)
        H_x, U = Q @ QtH, Q[:, :3]
        M = H_x @ P @ H_x.T + u_var * np.eye(len(r))
        Lc = np.linalg.cholesky(M)
        z = r - U @ (U.T @ r)
        a = sla.solve_triangular(Lc, z, lower=True)
        B = sla.solve_triangular(Lc, U, lower=True)
        c = B.T @ a
        ata[j] = a @ a
        gam[j] = ata[j] - c @ np.linalg.solve(B.T @ B, c)
    return gam, ata


@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("M", WINDOWS)
def test_cholesky_form_of_the_gate_matches_the_dense_gate(M, ratio):
    u_var, v_var = vr.pixel_noise(ratio) if ratio != 1.0 else (vr.SIGMA2, vr.SIGMA2)
    f = vr.numpy_filter(M, noise=(u_var, v_var))
    P, imu, poses = vr.numpy_state(f)
    lengths = [L for L in range(2, 31) if L <= M] * (2 if M < 12 else 1)
    outliers = tuple(range(1, len(lengths), 5))
    tracks = vr.make_tracks(np.random.default_rng(100 + M), poses, lengths, outliers=outliers)
    ref, _ = vr.gate(P, vr.project_tracks(imu, poses, tracks), tracks, u_var)
    gam, ata = gate_form(P, imu, poses, tracks, u_var)
    assert np.all(np.isfinite(ref)) and np.all(np.isfinite(gam))
    assert np.max(np.abs(gam - ref) / (1 + ref)) < 1e-12
    # a^T a >= gamma (the subtracted term is a PSD form); the ratio measures what the subtraction cancels
    ratio_max = float(np.max(ata / ref))
    assert np.all(ata >= ref * (1 - 1e-12)) and ratio_max < 2.0, ratio_max
