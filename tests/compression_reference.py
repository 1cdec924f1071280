"""References of the compression stage (k_blockdiag, k_gram / k_gram_mma, k_assemble, k_rows; DESIGN.md 4.4) on its own: what
T'', R'', r'' must hold, from two independent sides, and the split-K plan the host picks for the Gram products.

The stage projects the stacked system (H_o, r_o, R_o = blkdiag A_j^T D_j A_j) on the basis Q'' = [E_15 | H_c] (m > n), or keeps
every row (m <= n):
    m > n :  T'' = Q''^T H_o,  r'' = Q''^T r_o,  R'' = Q''^T R_o Q''          (rows >= 15: Lambda = H_c^T H_c, beta = H_c^T r_o,
                                                                            Psi = sum_j H_c,j^T R_o,j H_c,j)
    m <= n:  T'' = [H_o; 0],   r'' = [r_o; 0],   R'' = blkdiag(R_o, 0).
  * basis_free: from tests/vision_reference.py's per-track H_o,j, r_o,j, A_j (fp64, msckf_numpy's own null-space basis).  Rows
    >= 15 do not depend on the basis (A_j A_j^T is the one projector onto H_f's left null space).  The explicit ("head") rows do:
    there each track's block is turned into the engine's basis A'_j by W_j = A_j^T A'_j.
  * same_operation: the operation the kernels perform, on the engine's own stage inputs (Z, Yq, U^T r, the block-diagonal terms,
    the Householder vectors), in extended precision (np.longdouble where it carries 64 mantissa bits, else fp64 with the
    bound widened by the reference's own rounding).  Every entry comes with its scale (the sum of the moduli of what the
    kernels add up) and its summation depth k, so that |engine - reference| <= gamma_k * scale is the rounding bound.
The split-K plan (split_plan) mirrors fill_args in engine.cu; the constants are parsed from the sources (parse_constants) and
checked against MIRROR by tests/test_compression_reference_cpu.py."""
import re
from pathlib import Path

import numpy as np

CSRC = Path(__file__).resolve().parent.parent / "msckf_mono_b200" / "csrc"
# name -> (source, regular expression of its definition, the value the grids of tests/test_compression_stage_gpu.py are built for)
MIRROR = {"GT": ("gram_kernels.cuh", r"constexpr\s+int\s+GT\s*=\s*(\d+);", 32),
          "GK": ("gram_kernels.cuh", r"constexpr\s+int\s+GK\s*=\s*(\d+);", 16),
          "kMaxSplit": ("gram_kernels.cuh", r"constexpr\s+int\s+kMaxSplit\s*=\s*(\d+);", 16),
          "kAsmRows": ("gram_kernels.cuh", r"constexpr\s+int\s+kAsmRows\s*=\s*(\d+);", 16),
          # K / kSplitRows splits before the cap (fill_args)
          "kSplitRows": ("engine.cu", r"std::min\(kMaxSplit,\s*a\.K\s*/\s*(\d+)\)", 96),
          # the Gram products run on the FP64 tensor cores (DMMA) from this many tracks (fill_args)
          "kDmmaTracks": ("engine.cu", r"gram_mma\s*&&\s*p\.N\s*>=\s*(\d+)", 200)}
K = {k: v for k, (_, _, v) in MIRROR.items()}
U64 = 2.0 ** -53  # unit roundoff of fp64: every sum of the stage is fp64, in both filter precisions
REF = np.longdouble if np.finfo(np.longdouble).eps < 1e-18 else np.float64
REF_DEPTH = REF is np.float64  # fp64 reference: its own rounding widens the bound by its depth


def parse_constants():
    out = {}
    for name, (fn, rx, _) in MIRROR.items():
        found = re.findall(rx, (CSRC / fn).read_text())
        assert len(found) == 1, (name, fn, found)
        out[name] = int(found[0])
    return out


def split_plan(N):
    """(nsplit, kchunk, depth of the last chunk) of the Gram products of N tracks (K = 3N rows of Z), as fill_args picks them"""
    Kr = 3 * N
    nsplit = max(1, min(K["kMaxSplit"], Kr // K["kSplitRows"]))
    kchunk = -(-Kr // nsplit)
    kchunk = max(K["GK"], -(-kchunk // K["GK"]) * K["GK"])
    nsplit = max(1, -(-Kr // kchunk))
    return nsplit, kchunk, Kr - (nsplit - 1) * kchunk


def dmma(N, option5=True):
    return bool(option5) and N >= K["kDmmaTracks"]


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U64 / (1 - k * U64)


# ------------------------------------------------------------------------------------------------------------ layouts
def dense_X(Xg, o0, L, idx, c, dt=np.float64):
    """X_j [2L, c] (clone columns only) from the engine's Xg [O, 2, 6]"""
    X = np.zeros((2 * L, c), dtype=dt)
    for i in range(L):
        k = int(idx[o0 + i])
        X[2 * i:2 * i + 2, 6 * k:6 * k + 6] = Xg[o0 + i].astype(dt)
    return X


def householder_q(V, taug, dt=REF):
    """(Q [2L, 2L], |V| |T| |V|^T) of the track's reflectors as k_rows forms them: Q = H_0 H_1 H_2 = I - V T V^T (compact WY,
    T upper triangular), H_k = I - tau_k v_k v_k^T with tau_k = 2 / v_k^T v_k (0 where the kernel stored tau = 0).  The second is
    the scale of the kernel's entries of Q, which it forms as 1 - (V T)_a . V_b"""
    V = V.astype(dt)
    tau = [dt(2) / (V[:, k] @ V[:, k]) if taug[k] != 0 else dt(0) for k in range(3)]
    s = V.T @ V
    T = np.diag(tau).astype(dt)
    T[0, 1] = -tau[1] * T[0, 0] * s[0, 1]
    T[0, 2] = -tau[2] * (T[0, 0] * s[0, 2] + T[0, 1] * s[1, 2])
    T[1, 2] = -tau[2] * T[1, 1] * s[1, 2]
    Va = np.abs(V).astype(np.float64)
    return np.eye(len(V), dtype=dt) - V @ T @ V.T, Va @ np.abs(T).astype(np.float64) @ Va.T


# ---------------------------------------------------------------------------------------------------- same operation
def same_operation(b, obs_off, clone_idx, u_var, v_var, M, nsplit):
    """T'', R'', r'' from the engine's stage buffers `b` (capi.Engine.stage_buffer names: Z, Yq, ur, D1, D2, bb, Xg, rg, Vg,
    taug, accept, row_off) in extended precision.  Returns dict T2, R2, r2 (REF), their scales sT, sR, sr and depths kT, kR, kr
    (fp64), head (bool [n, n]: the entries of the explicit rows and, when compressing, their R'' coupling columns), gram (bool
    [n, n]: Lambda / Psi, rows and columns >= 15 when compressing), head_rows / gram_rows (bool [n]: the same for r''), Q (track
    -> its Q [2L, 2L], for every head track)"""
    n, c = 15 + 6 * M, 6 * M
    N = len(obs_off) - 1
    m = int(b["row_off"][N])
    full = m <= n
    hcap = m if full else 15
    T2, R2, r2 = np.zeros((n, n), REF), np.zeros((n, n), REF), np.zeros(n, REF)
    sT, sR, sr = np.zeros((n, n)), np.zeros((n, n)), np.zeros(n)
    kT, kR, kr = np.ones((n, n)), np.ones((n, n)), np.ones(n)
    head, gram = np.zeros((n, n), bool), np.zeros((n, n), bool)
    head_rows, gram_rows = np.zeros(n, bool), np.zeros(n, bool)
    D = lambda L2: np.tile(np.array([u_var, v_var], REF), L2 // 2)  # noqa: E731
    Qs = {}
    Kr = 3 * N
    if not full and N:
        Z, Yq, ur = b["Z"].astype(REF), b["Yq"].astype(REF), b["ur"].astype(REF)
        aZ, aY = np.abs(b["Z"]), np.abs(b["Yq"])
        blk1, blk2 = np.zeros((c, c), REF), np.zeros((c, c), REF)
        for k in range(M):
            blk1[6 * k:6 * k + 6, 6 * k:6 * k + 6] = b["D1"][k]
            blk2[6 * k:6 * k + 6, 6 * k:6 * k + 6] = b["D2"][k]
        g = slice(15, n)
        T2[g, g] = blk1 - Z.T @ Z
        R2[g, g] = blk2 - (Z.T @ Yq + Yq.T @ Z)
        r2[g] = b["bb"].astype(REF).ravel() - Z.T @ ur
        sT[g, g] = np.abs(blk1).astype(np.float64) + aZ.T @ aZ
        sR[g, g] = np.abs(blk2).astype(np.float64) + aZ.T @ aY + aY.T @ aZ
        sr[g] = np.abs(b["bb"]).ravel() + aZ.T @ np.abs(b["ur"])
        # each partial sums its chunk's products (Psi: two per k), the splits are summed, then subtracted from the block term
        kT[g, g], kR[g, g], kr[g] = Kr + nsplit + 2, 2 * Kr + nsplit + 2, Kr + nsplit + 2
        gram[g, g], gram_rows[g] = True, True
    for j in range(N):
        h0 = int(b["row_off"][j])
        if not b["accept"][j] or h0 >= hcap:
            continue
        o0, L = int(obs_off[j]), int(obs_off[j + 1] - obs_off[j])
        L2, nh = 2 * L, min(2 * L - 3, hcap - h0)
        Q, mag = householder_q(b["Vg"][2 * o0:2 * o0 + L2], b["taug"][j])
        Qs[j] = Q
        Qa = np.eye(L2) + mag  # the scale of the entries of Q as the kernel forms them
        A, U, Aa, Ua = Q[:, 3:3 + nh], Q[:, :3], Qa[:, 3:3 + nh], Qa[:, :3]
        X = dense_X(b["Xg"], o0, L, clone_idx, c, REF)
        Xa = np.abs(X).astype(np.float64)
        r = b["rg"][o0:o0 + L].astype(REF).ravel()
        d = D(L2)
        da = d.astype(np.float64)
        rows = slice(h0, h0 + nh)
        T2[rows, 15:] = A.T @ X
        sT[rows, 15:] = Aa.T @ Xa
        r2[rows] = A.T @ r
        sr[rows] = Aa.T @ np.abs(r).astype(np.float64)
        R2[rows, rows] = A.T @ (d[:, None] * A)
        sR[rows, rows] = Aa.T @ (da[:, None] * Aa)
        # Q's entries rest on the 2L-term sums v_k^T v_l (T) and a 3-term product; r'' on the 2L-term s = sum r_a w_a; Q^T D Q on
        # the 2L-term W^T D W and a 9-term quadratic form
        kT[rows, :], kr[rows], kR[rows, rows] = 2 * L2 + 16, 2 * L2 + 16, 2 * L2 + 16
        head[rows, :], head_rows[rows] = True, True
        if not full:
            Z_j = b["Z"][3 * j:3 * j + 3].astype(REF)
            cpl = A.T @ (d[:, None] * X) - (A.T @ (d[:, None] * U)) @ Z_j
            scl = Aa.T @ (da[:, None] * Xa) + (Aa.T @ (da[:, None] * Ua)) @ np.abs(b["Z"][3 * j:3 * j + 3])
            R2[rows, 15:], R2[15:, rows] = cpl, cpl.T
            sR[rows, 15:], sR[15:, rows] = scl, scl.T
            kR[rows, 15:], kR[15:, rows] = 2 * L2 + 24, 2 * L2 + 24
            head[15:, rows] = True
    if REF_DEPTH:
        kT, kR, kr = 2 * kT, 2 * kR, 2 * kr
    return {"T2": T2, "R2": R2, "r2": r2, "sT": sT, "sR": sR, "sr": sr, "kT": kT, "kR": kR, "kr": kr, "head": head, "gram": gram,
            "head_rows": head_rows, "gram_rows": gram_rows, "Q": Qs, "m": m, "full": full}


def kappa(got, ref, scale, mask=None):
    """max |got - ref| / (u scale) over the entries of mask (scale 0: the entry must be exactly ref)"""
    d = np.abs(got.astype(REF) - ref).astype(np.float64)
    mask = np.ones(d.shape, bool) if mask is None else mask
    assert np.all(d[mask & (scale == 0)] == 0)
    sel = mask & (scale > 0)
    return float((d[sel] / (U64 * scale[sel])).max()) if sel.any() else 0.0


def within_gamma(got, ref, scale, depth):
    """the entries where |got - ref| exceeds gamma_depth * scale (empty: every entry within its rounding bound)"""
    d = np.abs(got.astype(REF) - ref).astype(np.float64)
    return np.argwhere(d > gamma(depth) * scale)


def orthonormal_null_basis(Q, Hf):
    """(|A^T A - I|, |A^T H_f|) of the trailing 2L - 3 columns A of Q"""
    A = Q[:, 3:].astype(np.float64)
    return float(np.abs(A.T @ A - np.eye(A.shape[1])).max()), float(np.abs(A.T @ Hf).max())


# ------------------------------------------------------------------------------------------------------------ basis free
def compress(H_o, r_o, Ro_blocks, n):
    """(T'', R'', r'') of the stacked system by the definition above; Ro_blocks in stacking order (R_o is never formed)"""
    m = H_o.shape[0]
    T2, R2, r2 = np.zeros((n, n)), np.zeros((n, n)), np.zeros(n)
    if m <= n:
        T2[:m], r2[:m] = H_o, r_o
        off = 0
        for Rb in Ro_blocks:
            R2[off:off + len(Rb), off:off + len(Rb)] = Rb
            off += len(Rb)
        return T2, R2, r2
    Qpp = np.hstack([np.eye(m, 15), H_o[:, 15:]])
    off = 0
    for Rb in Ro_blocks:
        Qb = Qpp[off:off + len(Rb)]
        R2 += Qb.T @ Rb @ Qb
        off += len(Rb)
    return Qpp.T @ H_o, R2, Qpp.T @ r_o


def basis_free(blocks, accepted, u_var, v_var, n, head_bases=None):
    """(T'', R'', r'', their scales) from vision_reference.project_tracks' per-track (H_o,j, r_o,j, A_j) of the accepted tracks;
    head_bases: track -> the engine's basis A'_j [2L, 2L - 3] for the tracks whose rows are explicit.  The scales are the same
    formula on the moduli (|Q''|^T |H_o|, ...): zero exactly where the entry is a structural zero"""
    Hs, rs, Rs, Ha, ra, Ra = [], [], [], [], [], []
    for j, (blk, a) in enumerate(zip(blocks, accepted)):
        if not a:
            continue
        H, r, A = blk
        if head_bases is not None and j in head_bases:
            W = A.T @ head_bases[j].astype(np.float64)
            H, r, A = W.T @ H, W.T @ r, A @ W
        d = np.tile([u_var, v_var], A.shape[0] // 2)
        Rb = A.T @ (d[:, None] * A)
        Hs.append(H); rs.append(r); Rs.append(Rb)
        Ha.append(np.abs(H)); ra.append(np.abs(r)); Ra.append(np.abs(A).T @ (d[:, None] * np.abs(A)))
    if not Hs:
        z = np.zeros((n, n))
        return z, z.copy(), np.zeros(n), z.copy(), z.copy(), np.zeros(n)
    ref = compress(np.vstack(Hs), np.concatenate(rs), Rs, n)
    scl = compress(np.vstack(Ha), np.concatenate(ra), Ra, n)
    return ref + scl
