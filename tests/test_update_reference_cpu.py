"""The dense fp64 reference of one vision update (tests/vision_reference.py) that tests/test_update_shapes_gpu.py holds the
engine to: on small windows it must reproduce msckf_numpy's own update (exact-subspace mode, drop_null_rows=True) driven through
the same state, the uncompressed m x m innovation form, and itself on another basis of every track's null space.  A wrong
reference would make every comparison against it meaningless."""
import numpy as np
import pytest

from tests import vision_reference as vr


def numpy_update(f, tracks):
    """loop B + measurementUpdate of msckf_numpy at the tracks' p_f_G (what marginalize does after triangulation,
    msckf.h:404-449): (gamma [N], accepted [N])"""
    H_blocks, r_blocks, Ro_blocks, gam, acc = [], [], [], [], []
    u_var, v_var = f.noise["u_var_prime"], f.noise["v_var_prime"]
    for t in tracks:
        idx = [int(k) for k in t["idx"]]
        if len(idx) < 2:
            gam.append(np.nan); acc.append(False)
            continue
        r = f._calc_residual(t["pfg"], [f.cam_states[k] for k in idx], list(t["obs"]))
        H_o, A = f._calc_meas_jacobian(t["pfg"], idx)
        r_o = A.T @ r
        ok, g = f._gating_test(H_o, r_o, len(idx) - 1)
        gam.append(g); acc.append(ok)
        if ok:
            H_blocks.append(H_o); r_blocks.append(r_o)
            Ro_blocks.append(A.T @ (np.tile([u_var, v_var], len(idx))[:, None] * A))
    if H_blocks:
        f._measurement_update(np.vstack(H_blocks), np.concatenate(r_blocks), Ro_blocks)
    return np.array(gam), np.array(acc)


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


# (M, lengths, unseen clones, outlier tracks): m <= n and m > n, a clone no track sees, gross outliers, one-observation tracks
CASES = [(5, [5, 4, 3, 2, 1, 5], (), (1,)),
         (9, [9, 9, 9, 8, 9, 9, 3, 2, 1, 9], (), (2, 6)),
         (12, [10, 10, 10, 10, 10, 10, 10, 7, 4, 2, 1], (5,), (3,))]


@pytest.mark.parametrize("M,lengths,unseen,outliers", CASES)
def test_reference_matches_msckf_numpy_and_the_dense_form(M, lengths, unseen, outliers):
    f = vr.numpy_filter(M)
    P, imu, poses = vr.numpy_state(f)
    tracks = vr.make_tracks(np.random.default_rng(M), poses, lengths, unseen=unseen, outliers=outliers)
    ref = vr.reference(P, imu, poses, tracks)
    n = P.shape[0]
    assert vr.gate_margin(ref, tracks) > 0.1
    assert not ref["accepted"][[j for j, L in enumerate(lengths) if L == 1]].any()
    assert not ref["accepted"][list(outliers)].any() and ref["accepted"].sum() == len(lengths) - len(outliers) - lengths.count(1)
    gam, acc = numpy_update(f, tracks)
    assert np.array_equal(acc, ref["accepted"])
    fin = np.isfinite(gam)
    assert np.array_equal(fin, np.isfinite(ref["gamma"])) and rel(ref["gamma"][fin], gam[fin]) < 1e-12
    lu = f.last_update
    assert ref["m"] == lu["H_o"].shape[0]
    # msckf_numpy keeps the rows of R that the (unpivoted) QR builds at a clone no track sees: its zero columns leave their
    # rows to the later columns.  The compressed system's rank counts the independent basis vectors, as the engine does.
    assert ref["rank"] + (6 * len(unseen) if ref["m"] > n else 0) == lu["T_H"].shape[0]
    if ref["m"] > n:
        s = ref["sv"]
        assert np.all((s < vr.NULL_SV) | (s > vr.REAL_SV)), s  # a clean gap
    assert rel(ref["dx"], lu["deltaX"]) < 1e-12
    assert rel(ref["P"], f.getCovariance()) < 1e-12
    _, imu1, poses1 = vr.numpy_state(f)
    assert np.abs(ref["imu"] - imu1).max() < 1e-12 and np.abs(ref["poses"] - poses1).max() < 1e-12
    # the uncompressed m x m innovation form
    dx_d, P_d = vr.dense_update(P, ref["H_o"], ref["r_o"])
    assert rel(ref["dx"], dx_d) < 1e-12 and rel(ref["P"], P_d) < 1e-12


def test_reference_does_not_depend_on_the_null_space_basis():
    """a random orthogonal change of every track's basis A_j -> A_j U_j changes nothing (isotropic noise)"""
    M = 9
    P, imu, poses = vr.numpy_state(vr.numpy_filter(M))
    rng = np.random.default_rng(4)
    tracks = vr.make_tracks(rng, poses, [9, 9, 9, 9, 9, 9, 7, 3, 2], outliers=(4,))
    ref = vr.reference(P, imu, poses, tracks)
    assert ref["m"] > P.shape[0]
    blocks = []
    for b in vr.project_tracks(imu, poses, tracks):
        U = np.linalg.qr(rng.normal(size=(len(b[1]), len(b[1]))))[0]
        blocks.append((U.T @ b[0], U.T @ b[1]))
    rot = vr.reference(P, imu, poses, tracks, blocks=blocks)
    assert np.array_equal(rot["accepted"], ref["accepted"]) and rot["rank"] == ref["rank"]
    assert rel(rot["gamma"], ref["gamma"]) < 1e-12
    assert rel(rot["dx"], ref["dx"]) < 1e-12 and rel(rot["P"], ref["P"]) < 1e-12


def test_no_accepted_track_changes_nothing():
    P, imu, poses = vr.numpy_state(vr.numpy_filter(4))
    tracks = vr.make_tracks(np.random.default_rng(1), poses, [4, 3, 1], outliers=(0, 1))
    ref = vr.reference(P, imu, poses, tracks)
    assert not ref["accepted"].any() and ref["m"] == 0 and ref["dx"] is None
    assert np.array_equal(ref["P"], P) and np.array_equal(ref["imu"], imu) and np.array_equal(ref["poses"], poses)
