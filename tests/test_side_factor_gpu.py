"""The mapped-landmark update when S = T P T^T + I is not positive definite (a clone block of P made strongly negative): status 1,
nothing applied, NIS NaN, and P, the state and the poses untouched bit for bit, for a single filter and for the one broken member
of a device batch whose other members equal single calls, at one and at eight linearisations."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from tests.test_aid_gpu import assert_unchanged, snapshot
from tests.test_batch_stream_gpu import Member
from tests.test_landmark_gpu import R_PIX, state_of
from tests.test_landmark_iter_gpu import KEYS, drifted_obs

pytestmark = pytest.mark.gpu
DTYPES = [np.float32, np.float64]
WINDOWS = ((3, 1), (12, 2), (40, 3))


def observed(M):
    """up to 8 clones (m' up to 48 rows): breaking the last one puts the bad pivot past the first 32-column panel"""
    return list(range(0, M, max(1, M // 8)))


def break_clone(m, k):
    P = m.e.covariance().astype(np.float64)
    b = slice(15 + 6 * k, 21 + 6 * k)
    P[b, b] = -1e3 * np.eye(6)
    m.e.set_covariance(P)


def spec(rng, m, max_iter):
    _, poses = state_of(m.e)
    clone, z, p_L = drifted_obs(rng, poses, observed(m.e.num_clones()), 6, 0.3)
    return {"clone": clone, "z": z, "p_L": p_L, "R": R_PIX, "max_iter": max_iter, "tol": 1e-10}


def assert_failed(r):
    assert r["status"] == 1 and r["applied"] == 0 and np.isnan(r["nis"]) and r["dx_norm"] == 0.0, r


@pytest.mark.parametrize("max_iter", [1, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_single_filter_writes_nothing(dtype, max_iter):
    rng = np.random.default_rng(71)
    for M, seed in WINDOWS:
        m = Member(dtype, M, seed=seed, max_clones=M + 2)
        s = spec(rng, m, max_iter)
        break_clone(m, observed(M)[-1])
        before = snapshot(m.e)
        r = m.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], max_iter=max_iter, tol=s["tol"])
        assert_failed(r)
        assert r["used"] == len(s["clone"]), M
        assert_unchanged(snapshot(m.e), before)


@pytest.mark.parametrize("max_iter", [1, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_broken_batch_member_writes_nothing(dtype, max_iter):
    rng = np.random.default_rng(73)
    mem = [Member(dtype, WINDOWS[i % 3][0], seed=90 + i, max_clones=WINDOWS[i % 3][0] + 2) for i in range(6)]
    specs = [spec(rng, m, max_iter) for m in mem]
    bad = 5  # 40 clones
    break_clone(mem[bad], observed(mem[bad].e.num_clones())[-1])
    twins = [m.twin(dtype, max_clones=m.e.num_clones() + 2) for m in mem]
    before = snapshot(mem[bad].e)
    single = [t.e.landmark_update(s["clone"], s["z"], s["p_L"], R=s["R"], max_iter=max_iter, tol=s["tol"]) for t, s in zip(twins, specs)]
    batch = capi.Batch([m.e for m in mem])
    got = batch.landmark_update(specs)
    batch.close()
    for i, (m, t) in enumerate(zip(mem, twins)):
        assert (got[i]["status"] == 1) == (i == bad), (i, got[i])
        for key in KEYS:
            assert np.array_equal(got[i][key], single[i][key], equal_nan=True), (i, key)
        assert np.array_equal(got[i]["gamma"], single[i]["gamma"], equal_nan=True) and np.array_equal(got[i]["flag"], single[i]["flag"])
        for x, y in zip(m.e.state() + (m.e.covariance(),), t.e.state() + (t.e.covariance(),)):
            assert np.array_equal(x, y), i
    assert_failed(got[bad])
    assert_unchanged(snapshot(mem[bad].e), before)
