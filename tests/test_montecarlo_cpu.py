"""Host side of the Monte-Carlo consistency runner (msckf_mono_b200/montecarlo.py) without a GPU: the trials' inputs, the
error-state convention, the chi^2 bounds of the summary, and the merge of per-rank summaries over gloo."""
import os
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy import stats

from msckf_mono_b200 import montecarlo as mc, shard

N_TRIALS, N_FRAMES = 6, 12


def test_trials_share_the_truths_ids_and_tracks():
    truth = mc.make_truth(n_frames=30, seq=8)
    for k in (0, 7):
        tr = mc.make_trial(truth, k)
        for ft, fk in zip(truth["frames"], tr["frames"]):
            assert ft["state_id"] == fk["state_id"] and ft["time"] == fk["time"] and len(ft["imu"]) == len(fk["imu"])
            for key in ("update", "add"):
                assert np.array_equal(ft[key][1], fk[key][1]) and ft[key][0].shape == fk[key][0].shape


def _chi2_ok(x, var):
    """sum of squares of zero-mean samples / var against chi^2_n at 99.9 % (two-sided)"""
    x = np.asarray(x).ravel()
    s = float(np.sum(x * x) / var)
    return stats.chi2.ppf(0.0005, x.size) <= s <= stats.chi2.ppf(0.9995, x.size)


def test_injected_noise_follows_the_filters_model():
    truth = mc.make_truth(n_frames=60, seq=8)
    nz = truth["noise"]
    Q = np.asarray(nz["Q_imu"])
    inj = mc.make_trial(truth, 2)["injected"]
    dT = inj["dT"][:, None]
    assert _chi2_ok(inj["pixel"][:, 0], nz["u_var_prime"]) and _chi2_ok(inj["pixel"][:, 1], nz["v_var_prime"])
    for key, i, scale in (("gyro", 0, np.sqrt(dT)), ("bias_g", 3, 1 / np.sqrt(dT)), ("accel", 6, np.sqrt(dT)), ("bias_a", 9, 1 / np.sqrt(dT))):
        for ax in range(3):
            assert _chi2_ok((inj[key] * scale)[:, ax], Q[i + ax, i + ax]), (key, ax)


def test_trial_inputs_do_not_depend_on_the_number_of_trials():
    truth = mc.make_truth(n_frames=10, seq=8)
    a = [mc.make_trial(truth, k, seed=3) for k in range(4)][3]
    b = [mc.make_trial(truth, k, seed=3) for k in range(16)][3]
    assert np.array_equal(a["e0"], b["e0"]) and np.array_equal(a["truth_bias"], b["truth_bias"])
    for fa, fb in zip(a["frames"], b["frames"]):
        assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(fa["imu"], fb["imu"]))
        assert np.array_equal(fa["update"][0], fb["update"][0]) and np.array_equal(fa["add"][0], fb["add"][0])
    assert not np.array_equal(a["e0"], mc.make_trial(truth, 2, seed=3)["e0"])


def test_error_state_round_trips():
    rng = np.random.default_rng(1)
    for M in (0, 4):
        q = rng.standard_normal(4)
        imu = np.concatenate([rng.standard_normal(15), q / np.linalg.norm(q)])
        poses = rng.standard_normal((M, 7))
        poses[:, 3:7] /= np.linalg.norm(poses[:, 3:7], axis=1, keepdims=True)
        base = {"imu": imu, "poses": poses}
        e = 0.1 * rng.standard_normal(15 + 6 * M)
        assert np.max(np.abs(mc.error_state(mc.perturb(base, e), base) - e)) < 1e-12
        assert np.max(np.abs(mc.error_state(base, mc.estimate_of(base, e)) - e)) < 1e-12
    # the sign convention: dq.w < 0 is the same rotation
    q = np.array([0.1, -0.2, 0.3, 0.9]); q /= np.linalg.norm(q)
    assert np.allclose(mc.quat_error(q, np.array([0.0, 0.0, 0.0, 1.0])), mc.quat_error(-q, np.array([0.0, 0.0, 0.0, 1.0])))


def _records(trials, seed=0):
    out = {}
    for k in trials:
        rng = np.random.default_rng([seed, k])
        rows = []
        for f in range(N_FRAMES):
            M = min(f, 5)
            rows.append({"orientation": rng.chisquare(3), "position": rng.chisquare(3), "pose": rng.chisquare(6),
                         "imu": rng.chisquare(15), "full": rng.chisquare(15 + 6 * M), "dim_full": 15 + 6 * M, "first_bad_pivot": -1})
        out[k] = mc.trial_record(rows, rng.random(N_FRAMES))
    return out


def test_summary_bounds_are_chi2_quantiles():
    s = mc.summarize(_records(range(N_TRIALS)))
    for c, d in (("orientation", 3), ("pose", 6), ("imu", 15)):
        v = s["components"][c]
        for f in range(N_FRAMES):
            assert v["lower"][f] == stats.chi2.ppf(0.025, N_TRIALS * d) / N_TRIALS
            assert v["upper"][f] == stats.chi2.ppf(0.975, N_TRIALS * d) / N_TRIALS
    v = s["components"]["full"]
    assert v["upper"][3] == stats.chi2.ppf(0.975, N_TRIALS * 33) / N_TRIALS
    assert len(s["pos_rmse"]) == N_FRAMES


def worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    merged = shard.gather_summaries(_records(shard.sequences_of_rank(N_TRIALS, rank, world)))
    if rank == 0:
        q.put(mc.summarize(merged))
    dist.destroy_process_group()


def test_two_rank_merge_equals_single_process():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert got == mc.summarize(_records(range(N_TRIALS)))
