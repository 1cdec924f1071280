"""The state kernels (k_propagate, k_augment, k_gather) at every window, Pade branch, reading count and batch shape they dispatch
on, against the dense fp64 reference of tests/state_reference.py applied to the engine's own fetched state: fetch, one call,
fetch again, compare, so that no error accumulates across calls.
  (a) propagate at windows of 0 .. 192 clones: P_IC in one register slot per thread (6M <= 256), two slots (<= 512) and
      global memory (> 512), and the windows of 137 .. 192 clones that only the update refuses;
  (b) one reading per Pade degree and squaring count of each dtype, and a reading whose LU exchanges rows, at 1 and 86 clones
      (the branch taken, its margin and the pivoting are asserted on the fetched state);
  (c) 1, 16, 17 and 33 readings in one call (16 per launch), a long reading inside a launch and first after a launch boundary;
  (d) augment at windows of 0 .. 191 clones (k_augment's column passes at n <= 256, <= 512, > 512), growth of the clone
      capacity up to the hard limit of 192, and augment at 192 refused for a filter and a batch with nothing written;
  (e) prune at windows of 1 .. 192 clones with six kinds of keep lists (k_gather's grid-stride loop from 41 kept clones);
  (f) augment and propagate right after prunes, with stale rows and columns past n in the swapped covariance buffer;
  (g) one device batch of 40 members of every kind above (two launches of 32 / 8 members).
Half of the propagate cases start right after an aided pose fix, where the null state differs from the current one.  The inputs
are nontrivial: nonzero biases, a dense SPD Q_imu at the EuRoC scales, a rotated attitude, the EuRoC extrinsics (a 6.5 cm lever
arm) and a dense random SPD covariance."""
import numpy as np
import pytest

from msckf_mono_b200 import capi
from oracle.msckf_numpy import quat_normalized, quat_to_rot
from tests import state_reference as sr
from tests.parity_cases import make_engine

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
HARD_MAX = 192
# worst differences to the reference over the cases of this file, measured on an H100 80GB HBM3 (700 W power limit); every case
# is asserted at 10 x these.  P (one reading / one call of up to 33 readings / augment): max |difference| / max |reference|;
# state: max |difference| of the IMU state (p, v, b_g, b_a, g, q) / max(1, max |reference|); pose: the same for the new clone.
MEASURED = {"float64": {"P": 3.2e-15, "P_n": 1.5e-15, "P_aug": 1.8e-16, "state": 2.2e-16, "state_n": 2.2e-16, "pose": 4.6e-17},
            "float32": {"P": 1.1e-6, "P_n": 4.6e-6, "P_aug": 8.1e-8, "state": 8.1e-8, "state_n": 1.8e-7, "pose": 2.2e-8}}
# ceilings that separate rounding from a wrong result, whatever was measured (a wrong Pade coefficient at degree 9 makes errors
# of order 1e-6, a missed row exchange of order 1)
CONTRACT = {"float64": {"P": 1e-11, "P_n": 1e-10, "P_aug": 1e-11, "state": 1e-11, "state_n": 1e-10, "pose": 1e-11},
            "float32": {"P": 1e-4, "P_n": 1e-3, "P_aug": 1e-4, "state": 1e-4, "state_n": 1e-3, "pose": 1e-4}}

_bases = {}


def rd(x, dtype):
    """x as an engine of dtype holds it, in fp64"""
    return np.asarray(x, dtype=dtype).astype(np.float64)


def new_engine(dtype, cap):
    """an initialised engine for `cap` clones (owned by a class filter it keeps alive)"""
    f = make_engine(dtype, max_clones=cap, max_tracks=8, max_obs=64)
    f.initialize(*sr.setup())
    e = capi.Engine(dtype, borrowed=f.engineHandle())
    e.filt = f
    return e


def coast(dtype):
    """one 10 ms reading that leaves the attitude, the velocity and the biases of IMU0 as they are (omega = b_g, a = b_a -
    C(q) g): the clones lie along the velocity, and every branch reading keeps the descriptor it has at IMU0"""
    s = sr.IMU0
    a = s["b_a"] - quat_to_rot(s["q_IG"]) @ s["g"]
    return np.concatenate([s["b_g"], a, [0.01]])[None, :]


def base(dtype, M):
    """the cached engine with M clones (one coasting reading apart) and a dense random SPD covariance"""
    key = (np.dtype(dtype).name, M)
    if key not in _bases:
        e = new_engine(dtype, max(M, 1))
        for _ in range(M):
            e.propagate_n(coast(dtype))
            e.augment()
        n = 15 + 6 * M
        B = np.random.default_rng(M).normal(size=(n, n))
        S = B @ B.T / n + 0.1 * np.eye(n)
        e.set_covariance((S + S.T) / 2)
        _bases[key] = e
    return _bases[key]


def twin(dtype, M, cap=None):
    """a fresh copy of the cached engine with M clones, in an engine created for `cap` clones (default M + 1, at most 192)"""
    e = new_engine(dtype, cap or min(M + 1, HARD_MAX))
    e.copy_state_from(base(dtype, M))
    return e


def fetch(e):
    imu, poses = e.state()
    return e.covariance().astype(np.float64), imu.astype(np.float64), poses.astype(np.float64)


def pose_fix(e):
    """an aided pose fix a few centimetres and degrees off the current pose: the null state stays behind"""
    _, imu, _ = fetch(e)
    z = np.concatenate([imu[0:3] + [0.04, -0.03, 0.05], quat_normalized(imu[15:19] + [0.01, -0.015, 0.02, 0.0])])
    res = e.aid_update(capi.AID_POSE, z, 0.01 * np.eye(6))
    assert res["applied"] == 1 and res["status"] == 0
    _, imu1, _ = fetch(e)
    assert np.abs(imu1[22:25] - imu1[3:6]).max() > 1e-4 and np.abs(imu1[25:29] - imu1[15:19]).max() > 1e-4


def prepared(dtype, M, fixed, cap=None):
    e = twin(dtype, M, cap)
    if fixed:
        pose_fix(e)
    return e


def bound(dtype, key, v, label):
    name = np.dtype(dtype).name
    print(f"{label}: {key} {v:.2e}")
    assert v <= CONTRACT[name][key], (label, key, v)
    assert v <= 10 * MEASURED[name][key], (label, key, v)


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def state_err(got, ref):
    return float(np.abs(got[0:19] - ref[0:19]).max() / max(1.0, np.abs(ref[0:19]).max()))


def check_propagate(e, before, rs, dtype, label):
    """the engine's state after propagating `rs` from `before` against the reference stepped reading by reading"""
    P0, imu0, poses0 = before
    P1, imu1, poses1 = fetch(e)
    Pr, imur = sr.propagate_n(P0, imu0, rd(rs, dtype), rd(sr.Q_IMU, dtype))
    assert np.array_equal(P1[15:, 15:], P0[15:, 15:]) and np.array_equal(poses1, poses0), label
    assert np.array_equal(imu1[6:15], imu0[6:15]), label  # b_g, b_a, g
    assert np.array_equal(imu1[19:22], imu1[0:3]) and np.array_equal(imu1[22:25], imu1[3:6]), label
    assert np.array_equal(imu1[25:29], imu1[15:19]), label
    assert np.array_equal(P1, P1.T), label
    sfx = "" if len(rs) == 1 else "_n"
    bound(dtype, "P" + sfx, rel(P1, Pr), label)
    bound(dtype, "state" + sfx, state_err(imu1, imur), label)


def check_augment(e, before, dtype, label):
    P0, imu0, poses0 = before
    P1, imu1, poses1 = fetch(e)
    n, M = P0.shape[0], len(poses0)
    assert P1.shape == (n + 6, n + 6) and len(poses1) == M + 1 and e.num_clones() == M + 1, label
    assert np.array_equal(P1[:n, :n], P0) and np.array_equal(poses1[:M], poses0) and np.array_equal(imu1, imu0), label
    assert np.array_equal(P1, P1.T), label
    cam = sr.CAMERA
    Pr, posesr = sr.augment(P0, imu0, poses0, rd(cam["q_CI"], dtype), rd(cam["p_C_I"], dtype))
    bound(dtype, "P_aug", rel(P1, Pr), label)
    bound(dtype, "pose", float(np.abs(poses1[M] - posesr[M]).max() / max(1.0, np.abs(posesr[M]).max())), label)


def check_prune(e, before, keep, label):
    P0, imu0, poses0 = before
    P1, imu1, poses1 = fetch(e)
    Pr, posesr = sr.prune(P0, poses0, keep)
    assert e.num_clones() == len(keep), label
    assert np.array_equal(P1, Pr) and np.array_equal(poses1, posesr) and np.array_equal(imu1, imu0), label


# --------------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [0, 1, 42, 43, 85, 86, 136, 137, 192])
def test_propagate_at_every_window(dtype, M):
    rng = np.random.default_rng(M)
    for fixed in (False, True):
        e = prepared(dtype, M, fixed)
        before = fetch(e)
        r = sr.reading(rng, 0.05)[None, :]
        e.propagate_n(r)
        check_propagate(e, before, r, dtype, f"{np.dtype(dtype).name} M={M} pose fix {fixed}")


# --------------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [1, 86])
def test_propagate_at_every_pade_branch(dtype, M):
    name = np.dtype(dtype).name
    seen, swaps = set(), 0
    for i, (deg, sq, r) in enumerate(sr.branch_readings(dtype)):
        e = prepared(dtype, M, fixed=bool(i % 2))
        before = fetch(e)
        d = sr.describe(before[1], r, dtype)
        assert (d["deg"], d["sq"]) == (deg, sq) and d["margin"] > 0.01, (deg, sq, d)
        seen.add((deg, min(sq, 3)))
        swaps += d["gap"] > 1.3
        e.propagate_n(r[None, :])
        check_propagate(e, before, r[None, :], dtype, f"{name} M={M} degree {deg} squarings {sq} dT {r[6]:.3g} "
                                                      f"pivot gap {d['gap']:.2f}")
    want = {(3, 0), (5, 0), (7, 0), (9, 0), (13, 0), (13, 1), (13, 3)} if name == "float64" else {(3, 0), (5, 0), (7, 0), (7, 2)}
    assert want <= seen and swaps >= 1


# --------------------------------------------------------------------------------------------------------------------- (c)
def long_readings(rng, k):
    """k readings of 5 ms, with a 0.5 s reading fifth (inside the first launch) and seventeenth (first of the second launch)"""
    rs = sr.readings(rng, k)
    for j in (4, 16):
        if j < k:
            rs[j, 6] = 0.5
    if k == 1:
        rs[0, 6] = 0.5
    return rs


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [42, 86])
@pytest.mark.parametrize("k", [1, 16, 17, 33])
def test_readings_across_launches(dtype, M, k):
    for fixed in (False, True):
        e = prepared(dtype, M, fixed)
        before = fetch(e)
        rs = long_readings(np.random.default_rng(k), k)
        n0 = e.launch_count()
        e.propagate_n(rs)
        assert e.launch_count() - n0 == (k + 15) // 16
        check_propagate(e, before, rs, dtype, f"{np.dtype(dtype).name} M={M} k={k} pose fix {fixed}")


# --------------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [0, 40, 41, 82, 83, 135, 191])
def test_augment_at_every_window(dtype, M):
    e = twin(dtype, M)
    before = fetch(e)
    e.augment()
    check_augment(e, before, dtype, f"{np.dtype(dtype).name} augment M={M}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_augment_grows_to_the_hard_limit_and_stops_there(dtype):
    """an engine created for 100 clones grows to the hard limit (new ldp, copied P) when its 101st clone arrives; filled up to
    192 clones, augment fails with ERR_CAPACITY alone and in a batch, and changes nothing"""
    name = np.dtype(dtype).name
    e = twin(dtype, 100, cap=100)
    before = fetch(e)
    e.augment()
    check_augment(e, before, dtype, f"{name} augment at capacity 100 (growth to 192)")
    for _ in range(HARD_MAX - 102):
        e.augment()
    before = fetch(e)
    e.augment()
    check_augment(e, before, dtype, f"{name} augment 191 -> 192 after growth")
    other = twin(dtype, 5)
    snap = lambda x: fetch(x) + (x.num_clones(), x.launch_count())  # noqa: E731
    was = [snap(e), snap(other)]
    with pytest.raises(RuntimeError, match="rc=-2"):
        e.augment()
    batch = capi.Batch([other, e])
    with pytest.raises(RuntimeError, match="rc=-2"):
        batch.augment()
    batch.close()
    for x, w in zip((e, other), was):
        for a, b in zip(snap(x), w):
            assert np.array_equal(a, b)


# --------------------------------------------------------------------------------------------------------------------- (e)
def keep_lists(M, rng):
    """none, one middle clone, all but the first, all but the last, every other, a random subset (duplicates dropped)"""
    ks = [[], [M // 2], list(range(1, M)), list(range(M - 1)), list(range(0, M, 2)),
          sorted(rng.choice(M, max(M // 3, 1), replace=False).tolist())]
    out = []
    for k in ks:
        if k not in out:
            out.append(k)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [1, 41, 86, 136, 192])
def test_prune_at_every_window(dtype, M):
    for keep in keep_lists(M, np.random.default_rng(M)):
        e = twin(dtype, M)
        before = fetch(e)
        e.prune(keep)
        check_prune(e, before, keep, f"{np.dtype(dtype).name} prune M={M} keep {len(keep)}")


# --------------------------------------------------------------------------------------------------------------------- (f)
@pytest.mark.parametrize("dtype", DTYPES)
def test_calls_after_prune_read_nothing_past_the_window(dtype):
    """136 -> 135 -> 3 clones: the second prune writes into the buffer that holds the 136-clone covariance, so every row and
    column past n = 33 of the live buffer is stale; augment and propagate must not read them"""
    name = np.dtype(dtype).name
    e = twin(dtype, 136)
    e.prune(list(range(1, 136)))
    e.prune([4, 70, 134])
    before = fetch(e)
    e.augment()
    check_augment(e, before, dtype, f"{name} augment after prune")
    before = fetch(e)
    r = sr.reading(np.random.default_rng(5), 0.05)[None, :]
    e.propagate_n(r)
    check_propagate(e, before, r, dtype, f"{name} propagate after prune")


# --------------------------------------------------------------------------------------------------------------------- (g)
BATCH_WINDOWS = [0, 1, 5, 42, 43, 85, 86, 136, 137, 192, 40, 41, 82, 83, 135, 191, 12, 20, 64, 100]
BATCH_COUNTS = [0, 1, 16, 17, 33, 3]


@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_device_batch(dtype):
    """40 members (two launches of 32 and 8): windows 0 .. 192, reading counts 0 .. 33 with every Pade branch somewhere,
    half after a pose fix, one member at its capacity whose augment grows it, the 192-clone members left out of augment, then
    every kind of keep list; each member after each call against the reference"""
    name = np.dtype(dtype).name
    rng = np.random.default_rng(40)
    branches = [r for _, _, r in sr.branch_readings(dtype)]
    Ms = [BATCH_WINDOWS[i % len(BATCH_WINDOWS)] for i in range(40)]
    mem = [prepared(dtype, M, fixed=bool(i % 2), cap=(M if i == 17 else None)) for i, M in enumerate(Ms)]
    batch = capi.Batch(mem)
    # propagate
    rss = []
    for i in range(40):
        k = BATCH_COUNTS[i % len(BATCH_COUNTS)]
        rs = sr.readings(rng, k)
        if k:
            rs[(7 * i) % k] = branches[i % len(branches)]
        rss.append(rs)
    before = [fetch(m) for m in mem]
    batch.propagate_n(rss)
    for i, (m, b, rs) in enumerate(zip(mem, before, rss)):
        label = f"{name} batch member {i} M={Ms[i]} k={len(rs)}"
        if len(rs):
            check_propagate(m, b, rs, dtype, label)
        else:
            assert all(np.array_equal(x, y) for x, y in zip(fetch(m), b)), label
    # augment (member 17 grows its capacity; the 192-clone members stay out)
    which = [M < HARD_MAX for M in Ms]
    assert Ms[17] == 20 and mem[17].num_clones() == 20
    before = [fetch(m) for m in mem]
    batch.augment(which)
    for i, (m, b, w) in enumerate(zip(mem, before, which)):
        if w:
            check_augment(m, b, dtype, f"{name} batch member {i} augment M={Ms[i]}")
        else:
            assert all(np.array_equal(x, y) for x, y in zip(fetch(m), b))
    # prune
    keeps = []
    for i, m in enumerate(mem):
        M = m.num_clones()
        ks = keep_lists(M, rng) if M else [[]]
        keeps.append(None if i % 7 == 6 else ks[i % len(ks)])
    before = [fetch(m) for m in mem]
    batch.prune(keeps)
    for i, (m, b, k) in enumerate(zip(mem, before, keeps)):
        if k is None:
            assert all(np.array_equal(x, y) for x, y in zip(fetch(m), b))
        else:
            check_prune(m, b, k, f"{name} batch member {i} prune")
    batch.close()
