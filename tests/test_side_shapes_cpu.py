"""The side-update shape grid of tests/side_shapes.py without a GPU: the constants it is built for are the sources' constants,
it reaches both sides of every host decision and every cap exactly, and the information-form update equals the dense Joseph
form of test_aid_gpu.numpy_update."""
import numpy as np
import pytest

from tests import side_shapes as ss
from tests.test_aid_gpu import numpy_update


def test_mirrored_constants_are_the_sources():
    assert ss.parse_constants() == ss.K


def test_aid_grid_reaches_both_sides_of_the_storage_switch():
    K = ss.K
    rows = set()
    for m, (last, first) in ss.AID_EDGES.items():
        assert not ss.aid_global(last, m), m
        if first is None:  # shared at every window
            assert not ss.aid_global(K["kMaxKeep"], m) and last == K["kMaxKeep"]
        else:
            assert first == last + 1 and ss.aid_global(first, m), m
        rows.add(m)
        assert (last, m) in ss.aid_cases() and (first is None or (first, m) in ss.aid_cases())
    assert min(rows) == 1 and max(rows) == K["kAidMaxRows"] and K["kAidMaxRows"] - 1 in rows
    windows = {M for M, _ in ss.aid_cases()}
    assert {0, 1, K["kMaxKeep"] - 1, K["kMaxKeep"]} <= windows
    # the stacks: exactly m rows, at most kAidMaxItems items, the cap reached
    for (M, m) in ss.aid_cases():
        st = ss.aid_stack(M, m)
        assert sum(r for _, r, _ in st) == m and 1 <= len(st) <= K["kAidMaxItems"], (M, m)
    assert max(len(ss.aid_stack(M, m)) for M, m in ss.aid_cases()) == K["kAidMaxItems"]
    # the batch: two launch chunks; the first mixes shared and global members of different row counts
    assert ss.chunks(len(ss.AID_BATCH), K["kBatchMembers"]) == 2
    first = ss.AID_BATCH[:K["kBatchMembers"]]
    sides = {ss.aid_global(M, m) for M, m in first}
    assert sides == {False, True}
    assert len({m for M, m in first if ss.aid_global(M, m)}) >= 2 and len({m for M, m in first if not ss.aid_global(M, m)}) >= 2


def test_nees_grid():
    K = ss.K
    ns = [ss.n_of(M) for M in ss.NEES_WINDOWS]
    assert {n % 32 for n in ns} >= {1, 31} and ss.n_of(K["kMaxKeep"]) in ns and ss.n_of(K["kMaxKeep"]) % 32 == 15
    assert max(ss.chunks(n) for n in ns) == ss.chunks(ss.n_of(K["kMaxKeep"])) == 37
    M, k = ss.NEES_BREAK
    assert M == K["kMaxKeep"] and k < M and ss.chunks(15 + 6 * k + 1) > 1  # the first bad pivot lies past the first panel


def test_landmark_grid_reaches_every_panel_edge_and_cap():
    K = ss.K
    rows = []
    for r in ss.LMK_SWEEP_ROWS:
        c = ss.sweep_counts(ss.LMK_WINDOW, r)
        assert ss.lmk_rows(c) == r and max(c) < ss.LMK_WINDOW, r
        rows.append(r)
    for edge in (32, 64):  # both sides of the first two panel edges of k_lmk_gain's factor and k_lmk_downdate's p0 loop
        assert edge in rows and edge + 2 in rows and ss.chunks(edge) < ss.chunks(edge + 2)
    assert 30 in rows and ss.chunks(30) == 1
    assert max(rows) == K["kLmkMaxRows"] == 6 * K["kMaxKeep"]
    assert ss.lmk_rows(ss.sweep_counts(ss.LMK_WINDOW, 1152)) == 1152 and len(ss.sweep_counts(ss.LMK_WINDOW, 1152)) == K["kMaxKeep"]
    assert max(ss.LMK_PER_CLONE) == K["kLmkMaxPerClone"] and min(ss.LMK_PER_CLONE) == K["kLmkMaxPerClone"] - 1
    assert sum(ss.LMK_FULL.values()) == K["kLmkMaxObs"] and max(ss.LMK_FULL.values()) == K["kLmkMaxPerClone"]
    assert max(ss.LMK_WINDOWS) == K["kMaxKeep"] and all(M > 90 for M in ss.LMK_WINDOWS)
    assert set(ss.LMK_ITER_ROWS) == {180, K["kLmkMaxRows"]}
    # gating: the planned rows ld above a panel edge, the used rows below it, the gated clone between used clones
    for counts in ss.LMK_GATE:
        clones = sorted(counts)
        mid = clones[len(clones) // 2]
        ld = ss.lmk_rows(counts)
        m = ss.lmk_rows({k: a for k, a in counts.items() if k != mid})
        assert ss.chunks(ld) > ss.chunks(m) and clones[0] < mid < clones[-1], (ld, m)
    assert ss.lmk_tiles(ss.n_of(192)) == 37 * 38 // 2


def test_map_grid_reaches_every_cap():
    K = ss.K
    assert ss.map_rows(ss.MAP_ROWS) == K["kLmkMaxRows"] and ss.map_rows(ss.MAP_PAST) > K["kLmkMaxRows"]
    assert ss.map_rows(ss.MAP_PAST) == K["kLmkMaxRows"] + 2  # (every term of the planned rows is even)
    assert len({tuple(cs) for cs in ss.MAP_SETS}) == K["kLmkMaxSets"] and all(len(cs) >= 2 for cs in ss.MAP_SETS)
    assert len(ss.MAP_FULL_SET) * len(ss.MAP_FULL_SET[0]) == K["kLmkMaxPerSet"] and len(ss.MAP_FULL_SET[0]) == K["kLmkMapClones"]
    assert max(max(cs) for cs in ss.MAP_END) == K["kMaxKeep"] - 1 and len(ss.MAP_END[0]) == K["kLmkMapClones"]
    assert max(max(cs) for cs in ss.MAP_ROWS) == K["kMaxKeep"] - 1
    for sets in (ss.MAP_END, ss.MAP_FULL_SET, ss.MAP_SETS, ss.MAP_ROWS):
        assert ss.map_rows(sets) <= K["kLmkMaxRows"]


def _random_state(rng, M):
    imu = np.zeros(29)
    imu[0:15] = rng.normal(size=15)
    q = rng.normal(size=4)
    imu[15:19] = q / np.linalg.norm(q)
    poses = rng.normal(size=(M, 7))
    poses[:, 3:7] /= np.linalg.norm(poses[:, 3:7], axis=1, keepdims=True)
    return imu, poses


@pytest.mark.parametrize("M,k,b", [(0, 3, 2), (4, 10, 2), (12, 40, 2), (12, 7, 3), (30, 100, 2)])
def test_information_form_equals_the_joseph_form(M, k, b):
    rng = np.random.default_rng(100 + M + k)
    n = ss.n_of(M)
    A = rng.normal(size=(n, n))
    P = A @ A.T / n + np.eye(n)
    imu, poses = _random_state(rng, M)
    H = rng.normal(size=(k * b, n)) / np.sqrt(n)
    Rs = []
    for _ in range(k):
        B = rng.normal(size=(b, b))
        Rs.append(0.05 * (B @ B.T / b + 0.5 * np.eye(b)))
    from scipy.linalg import block_diag
    # r drawn from the model, N(0, H P H^T + R): (the information form's NIS subtracts b^T P+ b from r^T R^-1 r)
    r = np.linalg.cholesky(H @ P @ H.T + block_diag(*Rs)) @ rng.normal(size=k * b)
    ref = numpy_update(P, imu, poses, H, r, block_diag(*Rs))
    got = ss.information_update(P, imu, poses, H, r, np.array(Rs))
    assert np.abs(got[0] - ref[0]).max() <= 1e-12 * np.abs(ref[0]).max()
    assert np.abs(got[1] - ref[1]).max() <= 1e-12 * np.abs(ref[1]).max()
    if M:
        assert np.abs(got[2] - ref[2]).max() <= 1e-12 * np.abs(ref[2]).max()
    assert abs(got[3] - ref[3]) <= 1e-12 * ref[3] and abs(got[4] - ref[4]) <= 1e-12 * ref[4]
