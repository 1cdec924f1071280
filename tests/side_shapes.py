"""The shapes the side-update kernels (k_aid, k_nees, k_lmk_*) dispatch on, as the host decides them, the grids of
tests/test_side_shapes_gpu.py and tests/test_aid_fde_shapes_gpu.py that reach both sides of each decision and every cap, and
the information-form update for stacked systems too large for the dense Joseph form.

The constants are read from the CUDA sources (`parse_constants`) and checked against `MIRROR` by
tests/test_side_shapes_cpu.py: a threshold moved in the code fails there instead of leaving the grid on one side of it."""
import re
from pathlib import Path

import numpy as np

CSRC = Path(__file__).resolve().parent.parent / "msckf_mono_b200" / "csrc"
# name -> (source that defines it, the value the grid below is built for); a name is defined before the names that use it
MIRROR = {"kAidSmemMax": ("engine.cu", 32 * 1024), "kAidMaxRows": ("aid_kernels.cuh", 32), "kAidMaxItems": ("aid_kernels.cuh", 8),
          "kMaxKeep": ("state_kernels.cuh", 192), "kBatchMembers": ("state_kernels.cuh", 32),
          "kLmkMaxPerClone": ("landmark_kernels.cuh", 256), "kLmkMaxObs": ("landmark_kernels.cuh", 4096),
          "kLmkMaxRows": ("landmark_kernels.cuh", 1152), "kLmkMaxPerSet": ("landmark_kernels.cuh", 256),
          "kLmkMaxSets": ("landmark_kernels.cuh", 256), "kLmkMapClones": ("landmark_kernels.cuh", 8),
          "kLmkNB": ("landmark_kernels.cuh", 32), "kLmkThreads": ("landmark_kernels.cuh", 256),
          "kLmkMaxHyp": ("landmark_kernels.cuh", 1024), "kConsWarps": ("consensus_kernels.cuh", 8)}
K = {k: v for k, (_, v) in MIRROR.items()}


def parse_constants():
    """the MIRROR names as the sources define them: `constexpr int|size_t kName = <integers, * + - ( ) and earlier names>;`"""
    out = {}
    for name, (fn, _) in MIRROR.items():
        found = re.findall(r"constexpr\s+(?:int|size_t)\s+" + name + r"\s*=\s*([^;]+);", (CSRC / fn).read_text())
        assert len(found) == 1, (name, fn, found)
        expr = re.sub(r"\bmb::", "", found[0])
        assert re.fullmatch(r"[\w\s*+()-]+", expr), (name, expr)
        out[name] = int(eval(expr, {"__builtins__": {}}, dict(out)))  # noqa: S307 (integers and names parsed above)
    return out


def n_of(M):
    return 15 + 6 * M


def chunks(count, size=32):
    """ceil(count / size): panels of a factor over `count` columns, p0 steps of the downdate, launch chunks of members"""
    return -(-count // size)


# ---- k_aid: W^T and dx (n (m + 1) doubles) in dynamic shared memory up to kAidSmemMax bytes, else in the global workspace
def aid_ws_bytes(n, m):
    return 8 * n * (m + 1)


def aid_global(M, m):
    return aid_ws_bytes(n_of(M), m) > K["kAidSmemMax"]


def aid_dynamic_smem(M, m):
    """the dynamic shared memory of a k_aid launch of one member"""
    return 0 if aid_global(M, m) else aid_ws_bytes(n_of(M), m)


# row count -> (last window on the shared side, first window on the global side; None: shared at every window)
AID_EDGES = {1: (192, None), 3: (168, 169), 6: (95, 96), 9: (65, 66), 16: (37, 38), 31: (18, 19), 32: (18, 19)}
AID_END_WINDOWS = (0, 1, 191, 192)  # with m = 1 and 32: the first and last rows and columns of P
AID_END_ROWS = (1, 32)
# stacks of model items with exactly m rows, every clone item at the window's last clone (M - 1) unless it says 0:
# (model, rows, clone); RELATIVE_POSE is between clones 0 and M - 1.  The models of windows of < 2 clones stand apart.
AID_STACKS = {
    1: [("CLONE_HEADING", 1, -1)],
    3: [("CLONE_ANTENNA_POSITION", 3, -1)],
    6: [("RELATIVE_POSE", 6, None)],
    9: [("RELATIVE_POSE", 6, None), ("CLONE_ANTENNA_POSITION", 3, -1)],
    16: [("CLONE_POSE", 6, -1), ("RELATIVE_POSE", 6, None), ("BODY_VELOCITY", 3, None), ("CLONE_HEADING", 1, -1)],
    31: [("CLONE_POSE", 6, -1), ("RELATIVE_POSE", 6, None), ("POSE", 6, None), ("CLONE_ANTENNA_POSITION", 3, -1),
         ("ANTENNA_POSITION", 3, None), ("BODY_VELOCITY", 3, None), ("VELOCITY", 3, None), ("CLONE_HEADING", 1, -1)],
    32: [("CLONE_POSE", 6, -1), ("RELATIVE_POSE", 6, None), ("POSE", 6, None), ("CLONE_POSE", 6, 0),
         ("CLONE_ANTENNA_POSITION", 3, -1), ("BODY_VELOCITY", 3, None), ("CLONE_HEADING", 1, -1), ("HEADING", 1, None)],
}
AID_STACKS_SMALL = {  # windows of 0 and 1 clones (M = 1: the clone items at clone 0)
    (0, 1): [("HEADING", 1, None)],
    (0, 32): [("POSE", 6, None)] * 5 + [("HEADING", 1, None)] * 2,
    (1, 1): [("CLONE_HEADING", 1, -1)],
    (1, 32): [("CLONE_POSE", 6, -1), ("POSE", 6, None), ("CLONE_POSE", 6, -1), ("POSE", 6, None),
              ("CLONE_ANTENNA_POSITION", 3, -1), ("ANTENNA_POSITION", 3, None), ("HEADING", 1, None), ("CLONE_HEADING", 1, -1)],
}


def aid_stack(M, m):
    return AID_STACKS_SMALL[(M, m)] if M < 2 else AID_STACKS[m]


def aid_cases():
    """(M, m) of every single-call case: each row count at its last shared and first global window, and the end windows"""
    out = []
    for m, (a, b) in AID_EDGES.items():
        out += [(a, m)] + ([(b, m)] if b is not None else [])
    return out + [(M, m) for M in AID_END_WINDOWS for m in AID_END_ROWS if (M, m) not in out]


# a device batch of 33 LINEAR members (two launch chunks), chunk 0 mixing shared and global members of different m
AID_BATCH = [((18, 19, 37, 38, 65, 66, 95, 96, 168, 169, 0)[i % 11], (31, 32, 16, 9, 6, 3, 1)[i % 7]) for i in range(33)]

# ---- k_aid's launch: its static shared memory per form (-Xptxas -v, sm_90a, both dtypes, NM = 1 and 32; cuobjdump's SHARED is
# 1 KB more, sm_90's reservation) plus the dynamic bytes above.  A launch past the default 48 KB per CTA needs the kernel's
# raised dynamic limit: AID_OPT_IN lists those shapes (today FDE launches only, the plain form's 13 792 B leave 35 360 B)
AID_STATIC_SMEM = {"plain": 13792, "fde": 16976}
AID_DEFAULT_SMEM = 48 * 1024


def aid_launch_smem(M, m, fde):
    return AID_STATIC_SMEM["fde" if fde else "plain"] + aid_dynamic_smem(M, m)


AID_OPT_IN = [(18, 32), (20, 29), (21, 28), (27, 22), (28, 21), (30, 20), (33, 18), (35, 17), (37, 16), (40, 15), (43, 14),
              (46, 13), (50, 12), (54, 11), (59, 10), (65, 9), (72, 8), (73, 8), (82, 7), (94, 6), (95, 6), (110, 5), (111, 5),
              (132, 4), (133, 4), (134, 4), (166, 3), (167, 3), (168, 3)]


def aid_opt_in():
    """(M, m) of every window and row count whose k_aid launch, in either form, takes more than the default 48 KB"""
    return [(M, m) for M in range(K["kMaxKeep"] + 1) for m in range(1, K["kAidMaxRows"] + 1)
            if max(aid_launch_smem(M, m, f) for f in (False, True)) > AID_DEFAULT_SMEM]


# ---- k_aid<S, NM, true>: fault detection and exclusion over the items of a stack.  Recipes as AID_STACKS, (model, rows, clone),
# with exactly m rows in at most 8 items; ANTENNA_POSITION and BODY_VELOCITY take the mask of their rows (FDE_MASK).  The four
# range models sit on both storage sides, their clone forms at clone M - 1 and at clone 0; window 192's stacks put both at clone
# 191.  m = 32 fills all 8 warps of an exclusion round, with 6-row items (s_blk: 36 + 6 doubles per warp).  Items of equal
# rows observe different parts of the state where they can (a clone >= 0 is that clone): a fault that two such items explain
# alike is a tie of the exclusion test, not a check of it.
FDE_MASK = {1: 0b100, 2: 0b101, 3: 0b111}
_FDE_32 = [("CLONE_POSE", 6, -1), ("CLONE_POSE", 6, 5), ("POSE", 6, None), ("CLONE_POSE", 6, 0),
           ("CLONE_ANTENNA_POSITION", 3, 9), ("BODY_VELOCITY", 3, None)]
FDE_STACKS = {
    1: [("CLONE_RANGE", 1, -1)],
    3: [("RANGE", 1, None), ("PLANE_RANGE", 1, None), ("CLONE_RANGE", 1, 0)],
    6: [("CLONE_PLANE_RANGE", 1, -1), ("PLANE_RANGE", 1, None), ("CLONE_RANGE", 1, 0), ("RANGE", 1, None), ("BODY_VELOCITY", 2, None)],
    9: [("CLONE_RANGE", 1, -1), ("RELATIVE_POSE", 6, None), ("ANTENNA_POSITION", 2, None)],
    16: [("CLONE_POSE", 6, -1), ("RANGE", 1, None), ("RELATIVE_POSE", 6, None), ("CLONE_PLANE_RANGE", 1, 0), ("BODY_VELOCITY", 2, None)],
    31: [("POSE", 6, None), ("CLONE_POSE", 6, 5), ("CLONE_POSE", 6, 0), ("CLONE_POSE", 6, -1), ("CLONE_ANTENNA_POSITION", 3, 9),
         ("ANTENNA_POSITION", 2, None), ("PLANE_RANGE", 1, None), ("CLONE_RANGE", 1, -1)],
    32: _FDE_32 + [("RANGE", 1, None), ("CLONE_PLANE_RANGE", 1, 0)],
}
FDE_STACKS_AT = {  # the end windows' stacks where they differ from FDE_STACKS, and windows of 0 and 1 clones
    (191, 1): [("CLONE_PLANE_RANGE", 1, -1)],
    (191, 32): _FDE_32 + [("CLONE_RANGE", 1, -1), ("CLONE_PLANE_RANGE", 1, -1)],
    (192, 32): _FDE_32 + [("CLONE_RANGE", 1, -1), ("CLONE_PLANE_RANGE", 1, -1)],
    (0, 1): [("RANGE", 1, None)],
    (0, 32): [("POSE", 6, None)] * 4 + [("ANTENNA_POSITION", 3, None), ("PLANE_RANGE", 1, None), ("BODY_VELOCITY", 3, None),
                                        ("RANGE", 1, None)],
    (1, 1): [("CLONE_PLANE_RANGE", 1, -1)],
    (1, 32): [("CLONE_POSE", 6, -1), ("POSE", 6, None), ("CLONE_POSE", 6, -1), ("POSE", 6, None), ("CLONE_ANTENNA_POSITION", 3, -1),
              ("BODY_VELOCITY", 3, None), ("CLONE_RANGE", 1, -1), ("PLANE_RANGE", 1, None)],
}
FDE_DEPTH_WINDOWS = AID_EDGES[32]  # the exclusion depth at m = 32, one window on each storage side
# 8 items on separate parts of the state (a fault in one moves no other item's test much): faults of strictly decreasing size
# in the first k leave in that order, and at k = 7 one item is left
FDE_DEPTH = [("CLONE_POSE", 6, 0), ("CLONE_POSE", 6, -1), ("POSE", 6, None), ("CLONE_POSE", 6, 9), ("CLONE_ANTENNA_POSITION", 3, 5),
             ("CLONE_ANTENNA_POSITION", 3, 14), ("CLONE_RANGE", 1, 12), ("CLONE_PLANE_RANGE", 1, 3)]
FDE_DEPTH_RATIOS = [300.0 / 2 ** i for i in range(8)]  # each fault alone, in thresholds chi2[d_j - 1] of its item
FDE_SPREAD_RATIO = 0.75  # every item this far off: the stack fails, no single item explains it (outcome 3, all 8 in A)
FDE_BATCH_OPT_IN = [(e[0], m) for m, e in AID_EDGES.items() if (e[0], m) in AID_OPT_IN]  # AID_EDGES' last shared windows among them
# the shapes of a 33-member FDE batch, in turn: chunk 0 mixes them with other shapes of both storage paths
FDE_BATCH = FDE_BATCH_OPT_IN + [(20, 29), (133, 4), (0, 32), (1, 32), (192, 1), (18, 31), (19, 32), (38, 16), (96, 6), (169, 3)]


def fde_fill(M, m):
    """m rows in at most 8 items at a window of M >= 11 clones: a range at the IMU and one at the last clone, clone poses at
    clones 0, 2, .. 8, then a masked antenna fix and body velocity for the rest"""
    out = [("RANGE", 1, None), ("CLONE_RANGE", 1, -1)][:m]
    left = m - len(out)
    while left >= 6:
        out.append(("CLONE_POSE", 6, 2 * (len(out) - 2)))
        left -= 6
    if left > 3:
        out.append(("ANTENNA_POSITION", 3, None))
        left -= 3
    if left:
        out.append(("BODY_VELOCITY", left, None))
    return out


def fde_stack(M, m):
    if (M, m) in FDE_STACKS_AT:
        return FDE_STACKS_AT[(M, m)]
    return FDE_STACKS[m] if m in FDE_STACKS and M >= 2 else fde_fill(M, m)


def fde_faults(recipe):
    """[(name, faulty items, max_exclude)] of a recipe: none; the last item (warp 7 at 8 items); the first 6-row item; two items
    apart (the kept rows gathered around a hole) with max_exclude 2 and 1"""
    k = len(recipe)
    out = [("none", (), 2), ("last", (k - 1,), 1)]
    six = [i for i, (_, rows, _) in enumerate(recipe) if rows == 6 and i != k - 1]
    if six:
        out.append(("six", (six[0],), 1))
    if k >= 3:
        pair = (1, k - 1) if k >= 4 else (0, 2)
        out += [("pair", pair, 2), ("pair", pair, 1)]
    return out

# ---- k_nees: one CTA factors the (n + 1) x n bordered matrix in panels of 32
NEES_WINDOWS = (19, 24, 41, 95, 136, 191, 192)  # n mod 32 = 1, 31, 5, 9, 31, 9, 15
NEES_BREAK = (192, 150)  # window, clone whose block is made negative: first bad pivot 15 + 6 * 150 = 915, panel 28


# ---- mapped landmarks: the planned rows (ld, the workspace stride, from every observation) and the used rows m'
def lmk_rows(per_clone, groups=()):
    """sum over clones of min(2 a_k, 6) (a_k: observations of one-clone landmarks) plus over clone-set groups (c clones, o
    observations) min(2 o, 6 c).  With every observation: the host's ld; with the used ones: k_lmk_gain's m'."""
    return int(sum(min(2 * a, 6) for a in per_clone.values()) + sum(min(2 * o, 6 * c) for c, o in groups))


def spread(M, k):
    """k distinct clones of a window of M spread from 0 to M - 1"""
    return sorted({int(round(x)) for x in np.linspace(0, M - 1, k)}) if k > 1 else [M - 1]


def sweep_counts(M, rows):
    """clone -> observations with `rows` used rows: rows // 6 clones with 3 observations, one clone with 1 or 2 for the rest"""
    full, rest = divmod(rows, 6)
    clones = spread(M, full + (rest > 0))
    counts = {k: 3 for k in clones[:full]}
    if rest:
        counts[clones[full]] = rest // 2
    return counts


LMK_WINDOW = 192
LMK_SWEEP_ROWS = (30, 32, 34, 64, 66, 180, 1152)
LMK_WINDOWS = (91, 136, 191, 192)  # with clones 0, M // 2 and M - 1 observed
LMK_PER_CLONE = (255, 256)  # on clone 191 of a 192-clone window
LMK_FULL = {k: 256 for k in spread(192, 16)}  # 4096 observations: 16 clones x 256
# gating: (observations per clone, the clone whose every observation is gated): ld 36 -> m' 30 and ld 66 -> m' 60
LMK_GATE = ({k: 3 for k in spread(192, 6)}, {k: 3 for k in spread(192, 11)})
LMK_ITER_ROWS = (180, 1152)
# map uncertainty: (clone sets, landmarks per set); one-clone sets count per clone, the others per group
MAP_END = ([list(range(184, 192))] * 3 + [[191], [191], [0]])
MAP_FULL_SET = [list(range(184, 192))] * 32  # one group of 32 landmarks x 8 clones = 256 observations
MAP_SETS = [[k, k + 1] for k in range(191)] + [[k, k + 2] for k in range(65)]  # 256 clone-set groups of 2 clones
MAP_ROWS = [list(range(8 * g, 8 * g + 8)) for g in range(24) for _ in range(4)]  # 24 groups x 4 landmarks: 48 rows each
MAP_PAST = MAP_ROWS + [[0]]  # 2 rows more than kLmkMaxRows (planned rows are even: one row past cannot be asked for)


def map_rows(sets):
    """lmk_rows of landmarks with the given clone sets (one landmark per entry, every observation used)"""
    single, groups = {}, {}
    for cs in sets:
        if len(cs) == 1:
            single[cs[0]] = single.get(cs[0], 0) + 1
        else:
            groups[tuple(cs)] = groups.get(tuple(cs), 0) + len(cs)
    return lmk_rows(single, [(len(cs), o) for cs, o in groups.items()])


# ---- the consensus on map matches (consensus_kernels.cuh): k_lmk_hyp runs kConsWarps hypotheses (one warp each) per CTA;
# k_lmk_cons runs one CTA of kLmkThreads per member, strides the hypotheses by kLmkThreads, reduces them by shuffle in a warp
# and across the kLmkThreads / 32 warps in thread 0, and keeps kLmkMaxObs / kLmkThreads inlier bits per thread
CONS_WINDOWS = LMK_WINDOWS  # with clones 0, M // 2 and M - 1 observed
CONS_ALL = {k: 3 for k in range(192)}  # every clone of a 192-clone window touched: k_lmk_hyp's and k_lmk_cons's ps[kMaxKeep] full
CONS_PER_CLONE = LMK_PER_CLONE  # on clone 191
CONS_FULL = LMK_FULL  # 4096 observations: every inlier bit of a k_lmk_cons thread in use
CONS_HYP = (1, 7, 8, 9, 1023, 1024)  # around k_lmk_hyp's CTA edges, and the cap
CONS_FIRST = (0, 31, 32, 255, 256, 257, 1023)  # the first valid hypothesis: warp, CTA-stride and last-index edges of k_lmk_cons
CONS_TIE_OBS = 128  # observations of the tie cases (32 on each of 4 clones)
# map uncertainty: the clone-set shapes, and what the consensus excludes in each (a pattern a shape cannot hold is left out:
# MAP_FULL_SET's one clone set is the whole call)
CONS_MAP = {"full_set": MAP_FULL_SET, "sets": MAP_SETS, "rows": MAP_ROWS}
CONS_MAP_PATTERNS = ("one_observation", "landmark", "clone_set", "clone")
CONS_GATE = LMK_GATE  # the middle clone's observations all wrong: used rows 30 / 60 under a stride of 36 / 66
CONS_SWEEP_ROWS = LMK_SWEEP_ROWS  # used rows; wrong matches raise the planned rows past the next panel edge (1152: below it)
CONS_BATCH = 40  # members: two launch chunks of kBatchMembers and 8


def cons_sweep(M, rows):
    """(right, wrong) clone -> observations whose right ones use `rows` rows (sweep_counts) and whose wrong ones, excluded by
    the consensus, raise the planned rows by 2 on a clone no right match touches (by 0 at the cap: then one clone's 3 right
    matches become 2 right and 1 wrong, 2 used rows fewer)"""
    right = sweep_counts(M, rows)
    if rows + 2 <= K["kLmkMaxRows"]:
        return right, {next(k for k in range(M) if k not in right): 1}
    k = next(iter(right))
    right = dict(right)
    right[k] -= 1
    return right, {k: 1}


def lmk_tiles(n):
    """k_lmk_downdate's CTAs per member: the 32 x 32 tiles of P's lower triangle"""
    t = chunks(n, K["kLmkNB"])
    return t * (t + 1) // 2


# ---- the information form of the EKF update
def information_update(P, imu, poses, H, r, R_blocks):
    """the update of test_aid_gpu.numpy_update in information form, for a block-diagonal R = blkdiag(R_blocks [k, b, b]):
    b = H^T R^-1 r, P+ = (P^-1 + H^T R^-1 H)^-1, dx = P+ b, NIS = r^T R^-1 r - b^T P+ b; injection as numpy_update's.
    Costs n^3 and k b^2 n^2 instead of the Joseph form's (k b)^3."""
    from tests.landmark_map_reference import inject
    Rb = np.asarray(R_blocks, dtype=np.float64)
    k, bs = Rb.shape[0], Rb.shape[1]
    Ri = np.linalg.inv(Rb)
    RiH = np.einsum("kij,kjn->kin", Ri, H.reshape(k, bs, -1)).reshape(k * bs, -1)
    Rir = np.einsum("kij,kj->ki", Ri, r.reshape(k, bs)).ravel()
    b = H.T @ Rir
    Pn = np.linalg.inv(np.linalg.inv(P) + H.T @ RiH)
    Pn = 0.5 * (Pn + Pn.T)
    dx = Pn @ b
    imu, poses = inject(imu, poses, dx)
    return Pn, imu, poses, float(r @ Rir - b @ dx), float(np.linalg.norm(dx))
