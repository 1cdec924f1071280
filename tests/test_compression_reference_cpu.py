"""CPU checks of tests/compression_reference.py: on small random stacked systems with an explicit Householder basis per track,
both references equal the definition Q''^T H_o, Q''^T R_o Q'', Q''^T r_o (m > n) or the plain stacked system (m <= n); the
split-K plan mirror reproduces the plans the Gram kernels' edges depend on; the mirrored constants are the sources' own."""
import numpy as np
import pytest
import scipy.linalg as sla

from tests import compression_reference as cr


def householder(Hf):
    """(V [2L, 3] with unit diagonal and zeros above it, tau [3], Q = H_0 H_1 H_2) of an unpivoted Householder QR of H_f"""
    R = Hf.copy()
    L2 = len(R)
    V, tau = np.zeros((L2, 3)), np.zeros(3)
    for k in range(3):
        x = R[k:, k]
        beta = -np.copysign(np.linalg.norm(x), x[0])
        v = x.copy()
        v[0] -= beta
        v /= v[0]
        V[k:, k] = v
        tau[k] = 2.0 / (v @ v)
        R[k:] -= tau[k] * np.outer(v, v @ R[k:])
    Q = np.eye(L2)
    for k in range(3):
        Q = Q - tau[k] * np.outer(Q @ V[:, k], V[:, k])
    return V, tau, Q


def instance(rng, M, lengths, rejected=(), u_var=2.0e-5, v_var=5.0e-5):
    """a random stacked system over M clones: per track X_j (2 x 6 blocks at its clones), H_f, r_j and a Householder basis; the
    engine's stage buffers for it; and the definition's T'', R'', r''"""
    n, c = 15 + 6 * M, 6 * M
    off, idx, tracks = [0], [], []
    for L in lengths:
        k = np.sort(rng.choice(M, L, replace=False))
        idx += list(k)
        off.append(off[-1] + L)
        Hf = rng.normal(size=(2 * L, 3))
        V, tau, Q = householder(Hf)
        X = np.zeros((2 * L, c))
        Xg = rng.normal(size=(L, 2, 6))
        for i, kk in enumerate(k):
            X[2 * i:2 * i + 2, 6 * kk:6 * kk + 6] = Xg[i]
        tracks.append({"X": X, "Xg": Xg, "Hf": Hf, "r": rng.normal(size=2 * L), "V": V, "tau": tau, "Q": Q, "L": L})
    N, O = len(lengths), off[-1]
    acc = np.array([j not in rejected for j in range(N)], np.int32)
    rows = np.array([2 * t["L"] - 3 if a else 0 for t, a in zip(tracks, acc)])
    b = {"Z": np.zeros((3 * N, c)), "Yq": np.zeros((3 * N, c)), "ur": np.zeros(3 * N), "D1": np.zeros((M, 6, 6)),
         "D2": np.zeros((M, 6, 6)), "bb": np.zeros((M, 6)), "Xg": np.concatenate([t["Xg"] for t in tracks]),
         "rg": np.concatenate([t["r"].reshape(-1, 2) for t in tracks]), "Vg": np.concatenate([t["V"] for t in tracks]),
         "taug": np.array([t["tau"] for t in tracks]), "accept": acc, "row_off": np.concatenate([[0], np.cumsum(rows)])}
    Hs, rs, Rs = [], [], []
    for j, t in enumerate(tracks):
        if not acc[j]:
            continue
        d = np.tile([u_var, v_var], t["L"])
        U, A = t["Q"][:, :3], t["Q"][:, 3:]
        Zj = U.T @ t["X"]
        b["Z"][3 * j:3 * j + 3] = Zj
        b["Yq"][3 * j:3 * j + 3] = U.T @ (d[:, None] * t["X"]) - 0.5 * (U.T @ (d[:, None] * U)) @ Zj
        b["ur"][3 * j:3 * j + 3] = U.T @ t["r"]
        for i in range(t["L"]):
            kk = idx[off[j] + i]
            x0, x1 = t["Xg"][i]
            r0, r1 = t["r"][2 * i:2 * i + 2]
            b["D1"][kk] += np.outer(x0, x0) + np.outer(x1, x1)
            b["D2"][kk] += u_var * np.outer(x0, x0) + v_var * np.outer(x1, x1)
            b["bb"][kk] += x0 * r0 + x1 * r1
        Hs.append(np.hstack([np.zeros((2 * t["L"] - 3, 15)), A.T @ t["X"]]))
        rs.append(A.T @ t["r"])
        Rs.append(A.T @ (d[:, None] * A))
    H_o, r_o, R_o = np.vstack(Hs), np.concatenate(rs), sla.block_diag(*Rs)
    m = H_o.shape[0]
    if m > n:  # the definition: Q'' = [E_15 | H_c]
        Qpp = np.hstack([np.eye(m)[:, :15], H_o[:, 15:]])
        truth = (Qpp.T @ H_o, Qpp.T @ R_o @ Qpp, Qpp.T @ r_o)
    else:
        truth = (np.zeros((n, n)), np.zeros((n, n)), np.zeros(n))
        truth[0][:m], truth[1][:m, :m], truth[2][:m] = H_o, R_o, r_o
    return {"b": b, "off": np.array(off), "idx": np.array(idx), "tracks": tracks, "acc": acc, "truth": truth, "m": m, "n": n,
            "noise": (u_var, v_var)}


def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300))


CASES = {"compressed": (6, [3, 5, 2, 4, 6, 6, 5, 3, 2, 6, 4, 5], (3,)),  # m > n, the head rows straddle a track edge
         "compressed_edge": (3, [3] * 12, ()),  # 3-row tracks: row 15 on a track edge
         "plain": (8, [3, 5, 2, 4], (1,)),  # m <= n: every stacked row explicit
         "square": (4, [4] * 7 + [3, 2], ())}  # m = n = 39


@pytest.mark.parametrize("case", list(CASES))
def test_references_equal_the_definition(case):
    M, lengths, rejected = CASES[case]
    I = instance(np.random.default_rng(len(case)), M, lengths, rejected)
    assert (I["m"] > I["n"]) == case.startswith("compressed") and (case != "square" or I["m"] == I["n"])
    so = cr.same_operation(I["b"], I["off"], I["idx"], *I["noise"], M, nsplit=1)
    for got, want in zip((so["T2"], so["R2"], so["r2"]), I["truth"]):
        assert rel(got, want) <= 1e-13, case
    # the truth sits within the rounding bound of every entry of the same-operation reference, and at its structural zeros
    for got, want, s, k in zip(I["truth"], (so["T2"], so["R2"], so["r2"]), (so["sT"], so["sR"], so["sr"]), (so["kT"], so["kR"], so["kr"])):
        assert cr.within_gamma(got, want, s, k).size == 0, case
    # every head basis the reference rebuilds from (V, tau) is orthonormal and annihilates H_f
    for j, Q in so["Q"].items():
        orth, ann = cr.orthonormal_null_basis(Q, I["tracks"][j]["Hf"])
        assert orth <= 1e-14 and ann <= 1e-13 * np.abs(I["tracks"][j]["Hf"]).max(), (case, j, orth, ann)
    # basis-free: msckf_numpy-style blocks on another basis of each null space (from an SVD), turned into the Householder one
    blocks = []
    for t in I["tracks"]:
        A = sla.null_space(t["Hf"].T)
        H = np.hstack([np.zeros((A.shape[1], 15)), A.T @ t["X"]])
        blocks.append((H, A.T @ t["r"], A))
    bf = cr.basis_free(blocks, I["acc"], *I["noise"], I["n"], head_bases={j: Q[:, 3:] for j, Q in so["Q"].items()})
    for got, want in zip(bf[:3], I["truth"]):
        assert rel(got, want) <= 1e-13, case
    # its scales vanish exactly at the definition's structural zeros
    for s, want in zip(bf[3:], I["truth"]):
        assert np.all(want[s == 0] == 0), case
    # without the engine's bases only the rows >= 15 (compressed) agree: they do not depend on the basis
    if I["m"] > I["n"]:
        other = cr.basis_free(blocks, I["acc"], *I["noise"], I["n"])
        assert rel(other[0][15:], I["truth"][0][15:]) <= 1e-13 and rel(other[1][15:, 15:], I["truth"][1][15:, 15:]) <= 1e-13
        assert rel(other[2][15:], I["truth"][2][15:]) <= 1e-13


def test_kappa_and_the_rounding_bound_see_one_wrong_entry():
    I = instance(np.random.default_rng(7), 6, [3, 5, 2, 4, 6, 6, 5, 3, 2, 6, 4, 5])
    so = cr.same_operation(I["b"], I["off"], I["idx"], *I["noise"], 6, nsplit=1)
    T2 = so["T2"].astype(np.float64)
    assert cr.kappa(T2, so["T2"], so["sT"], so["gram"]) <= 1.0 and cr.within_gamma(T2, so["T2"], so["sT"], so["kT"]).size == 0
    i, j = np.unravel_index(np.argmax(so["sT"] * so["gram"]), T2.shape)
    T2[i, j] += 2 * cr.gamma(so["kT"][i, j]) * so["sT"][i, j]
    assert cr.within_gamma(T2, so["T2"], so["sT"], so["kT"]).tolist() == [[i, j]]
    assert cr.kappa(T2, so["T2"], so["sT"], so["gram"]) > 1.9 * so["kT"][i, j]


def test_split_plan_mirror():
    """the plans the Gram kernels' edges depend on (DESIGN.md 4.4)"""
    assert cr.split_plan(600) == (15, 128, 8)  # K = 1800: 16 splits recomputed to 15 at the cap, a last chunk 8 deep
    assert cr.split_plan(511)[0] == 14 and cr.split_plan(530)[0] == 15
    assert cr.split_plan(1) == (1, 16, 3) and cr.split_plan(31)[0] == 1 and cr.split_plan(32)[0] == 1 and cr.split_plan(64)[0] == 2
    assert cr.split_plan(512)[0] == 16 and cr.split_plan(200) == (6, 112, 40)
    for N in range(1, 2049):
        ns, kc, last = cr.split_plan(N)
        assert 1 <= ns <= cr.K["kMaxSplit"] and kc % cr.K["GK"] == 0 and 0 < last <= kc and (ns - 1) * kc + last == 3 * N, N
    assert not cr.dmma(199) and cr.dmma(200) and not cr.dmma(600, option5=False)
    # c = 6M, M = 1 .. 16: every even width of the last 32-tile
    assert {6 * M % cr.K["GT"] for M in range(1, 17)} == set(range(0, cr.K["GT"], 2))


def test_mirrored_constants_match_the_sources():
    assert cr.parse_constants() == cr.K
