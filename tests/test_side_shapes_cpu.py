"""The side-update shape grid of tests/side_shapes.py without a GPU: the constants it is built for are the sources' constants,
it reaches both sides of every host decision and every cap exactly, and the information-form update equals the dense Joseph
form of test_aid_gpu.numpy_update.  The FDE grid: recipes that fit their windows, the launches past the default 48 KB of
shared memory and the kernel's static shared memory behind them, the range models on both paths, and the exclusion order of
the depth recipes under tests/aid_fde_reference.py."""
from pathlib import Path

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


# ---- fault detection and exclusion (k_aid<S, NM, true>) and the range models ----------------------------------------------
RANGE_NAMES = ("RANGE", "CLONE_RANGE", "PLANE_RANGE", "CLONE_PLANE_RANGE")


def _fde_recipes():
    """(M, m, recipe) of every FDE stack the GPU tests run"""
    out = [(M, m, ss.fde_stack(M, m)) for M, m in ss.aid_cases() + ss.AID_OPT_IN]
    return out + [(M, 32, ss.FDE_DEPTH) for M in ss.FDE_DEPTH_WINDOWS]


def _clone(M, clone):
    return M - 1 if clone == -1 else clone


def _random_cov(rng, M):
    n = ss.n_of(M)
    A = rng.normal(size=(n, n))
    return A @ A.T / n + np.eye(n)


def test_fde_recipes_fit_their_windows():
    K = ss.K
    for M, m, recipe in _fde_recipes():
        assert sum(r for _, r, _ in recipe) == m and 1 <= len(recipe) <= K["kAidMaxItems"], (M, m)
        for model, rows, clone in recipe:
            if model.startswith("CLONE_"):
                assert M >= 1 and 0 <= _clone(M, clone) < M, (M, m, model, clone)
            else:
                assert clone is None, (M, m, model)
            assert M >= 2 or model != "RELATIVE_POSE", (M, m)
            assert rows in ss.FDE_MASK or model not in ("ANTENNA_POSITION", "CLONE_ANTENNA_POSITION", "BODY_VELOCITY")
        if m == K["kAidMaxRows"]:  # every warp of an exclusion round, a 6-row block among them
            assert len(recipe) == K["kAidMaxItems"] and any(r == 6 for _, r, _ in recipe), M
    # the items of each recipe have the rows it says (recipe_items asserts it) at a state of that window
    from tests import aid_fde_reference as ref
    rng = np.random.default_rng(7)
    for M, m, recipe in _fde_recipes():
        imu, poses = _random_state(rng, M)
        assert sum(len(it["R"]) for it in ref.recipe_items(rng, recipe, imu, poses, M)) == m
    # the fault patterns: the last item, a 6-row item, two items apart with a kept item between them
    for M, m, recipe in _fde_recipes():
        pats = {name: (f, k) for name, f, k in ss.fde_faults(recipe)}
        assert pats["last"][0] == (len(recipe) - 1,)
        if any(r == 6 for _, r, _ in recipe[:-1]):
            assert recipe[pats["six"][0][0]][1] == 6
        if len(recipe) >= 3:
            i, j = pats["pair"][0]
            assert j - i >= 2
            assert [k for name, f, k in ss.fde_faults(recipe) if name == "pair"] == [2, 1]


def test_fde_grid_reaches_both_sides_of_every_row_count():
    for m, (last, first) in ss.AID_EDGES.items():
        cases = [(M, mm) for M, mm in ss.aid_cases() if mm == m]
        assert (last, m) in cases and not ss.aid_global(last, m)
        if first is not None:
            assert (first, m) in cases and ss.aid_global(first, m)
    a, b = ss.FDE_DEPTH_WINDOWS
    assert not ss.aid_global(a, 32) and ss.aid_global(b, 32)
    # the batch's first launch chunk: past the default limit, other shared-side members and global-side members
    first = [ss.FDE_BATCH[i % len(ss.FDE_BATCH)] for i in range(ss.K["kBatchMembers"])]
    assert set(ss.FDE_BATCH_OPT_IN) <= set(first) and {ss.aid_global(M, m) for M, m in first} == {False, True}
    assert any(not ss.aid_global(M, m) and (M, m) not in ss.AID_OPT_IN for M, m in first)


def test_opt_in_shapes_are_the_enumeration():
    assert ss.AID_OPT_IN == ss.aid_opt_in() and len(ss.AID_OPT_IN) == 29
    for M, m in ss.AID_OPT_IN:  # FDE launches only: the plain form stays under the default limit everywhere
        assert ss.aid_launch_smem(M, m, True) > ss.AID_DEFAULT_SMEM >= ss.aid_launch_smem(M, m, False)
    assert all(ss.aid_launch_smem(M, m, False) <= ss.AID_DEFAULT_SMEM for M in range(ss.K["kMaxKeep"] + 1)
               for m in range(1, ss.K["kAidMaxRows"] + 1))
    # the band: dynamic bytes in (48 KB - the FDE form's static, kAidSmemMax]
    for M, m in ss.AID_OPT_IN:
        assert ss.AID_DEFAULT_SMEM - ss.AID_STATIC_SMEM["fde"] < ss.aid_ws_bytes(ss.n_of(M), m) <= ss.K["kAidSmemMax"]
    # the last shared windows of AID_EDGES for m = 32, 16, 9, 6 and 3 are in the band, and in the batch's first chunk
    assert {(e[0], m) for m, e in ss.AID_EDGES.items() if (e[0], m) in ss.AID_OPT_IN} == set(ss.FDE_BATCH_OPT_IN)
    assert {m for _, m in ss.FDE_BATCH_OPT_IN} == {32, 16, 9, 6, 3}


def test_every_range_model_on_both_sides_and_at_the_last_clone():
    sides = {name: set() for name in RANGE_NAMES}
    clones = {name: set() for name in RANGE_NAMES if name.startswith("CLONE_")}
    at_end = set()
    for M, m in ss.aid_cases():
        for model, _, clone in ss.fde_stack(M, m):
            if model in sides:
                sides[model].add(ss.aid_global(M, m))
            if model in clones and M >= 2:
                clones[model].add("last" if clone == -1 else clone)
                if M == ss.K["kMaxKeep"] and _clone(M, clone) == M - 1:
                    at_end.add(model)
    assert all(s == {False, True} for s in sides.values()), sides
    assert all({"last", 0} <= c for c in clones.values()), clones
    assert at_end == set(clones), at_end


def test_depth_recipes_exclude_in_the_intended_order():
    from msckf_mono_b200 import capi
    from tests import aid_fde_reference as ref
    chi2 = capi.fde_thresholds(0.01)
    rng = np.random.default_rng(8)
    for M in ss.FDE_DEPTH_WINDOWS:
        imu, poses = _random_state(rng, M)
        P = _random_cov(rng, M)
        for k in range(1, 9):
            items = ref.recipe_items(rng, ss.FDE_DEPTH, imu, poses, M)
            items = ref.with_faults(rng, items, range(k), ss.FDE_DEPTH_RATIOS[:k], imu, poses, P, chi2)
            K = min(k, ss.K["kAidMaxItems"] - 1)
            want = ref.fde(items, imu, poses, P, chi2, K)
            assert [j for j, _ in want["excluded"]] == list(range(K)) and want["margin"] >= 0.05, (M, k, want["excluded"])
            assert want["outcome"] == (1 if k < 8 else 2) and len(want["kept"]) == 8 - K
            if k < 8:
                assert ref.fde(items, imu, poses, P, chi2, k - 1)["outcome"] == 2
        items = ref.with_faults(rng, ref.recipe_items(rng, ss.FDE_DEPTH, imu, poses, M), range(8), [ss.FDE_SPREAD_RATIO] * 8,
                                imu, poses, P, chi2)
        want = ref.fde(items, imu, poses, P, chi2, 7)
        assert want["outcome"] == 3 and len(want["kept"]) >= 2, want


def test_exclusion_statistic_is_the_nis_difference():
    """t_j = y_j^T B_j^-1 y_j equals NIS_A - NIS_{A minus j} (DESIGN 4.15)"""
    from scipy.linalg import block_diag
    from tests import aid_fde_reference as ref
    rng = np.random.default_rng(9)
    d = [6, 3, 1, 6, 2, 1, 3, 6]
    m = sum(d)
    G = rng.normal(size=(m, m))
    S = G @ G.T / m + block_diag(*[0.1 * np.eye(k) for k in d])
    r = rng.normal(size=m) * 3.0
    first = np.cumsum([0] + d)
    blocks = [np.arange(first[j], first[j + 1]) for j in range(len(d))]
    for A in (list(range(len(d))), [0, 2, 3, 5, 7], [1, 4]):
        rows = np.concatenate([blocks[j] for j in A])
        t = ref.exclusion_tests(S, r, [blocks[j] for j in A])
        nis = ref.set_nis(S, r, rows)
        for j, tj in zip(A, t):
            rest = np.concatenate([blocks[k] for k in A if k != j])
            assert abs(tj - (nis - ref.set_nis(S, r, rest))) <= 1e-10 * nis, (A, j)


def test_k_aid_static_shared_memory_is_the_mirror():
    """cuobjdump's SHARED of each of the 8 k_aid instantiations, less sm_90's 1 KB reservation, is AID_STATIC_SMEM of its form"""
    import re
    import shutil
    import subprocess
    lib = ss.CSRC.parent / "libmsckf_b200.so"
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not lib.exists() or not Path(tool).exists():
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "--dump-resource-usage", str(lib)], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (_ZN2mb5k_aidI([df])Li(\d+)ELb([01])E\w*):\s*\n\s*REG:\d+ STACK:\d+ SHARED:(\d+)", out)
    forms = {(s, int(nm), fde == "1"): int(shared) for _, s, nm, fde, shared in found}
    assert set(forms) == {(s, nm, f) for s in "df" for nm in (1, ss.K["kBatchMembers"]) for f in (False, True)}, sorted(forms)
    for (_, _, f), shared in forms.items():
        assert shared - 1024 == ss.AID_STATIC_SMEM["fde" if f else "plain"], (f, shared)
