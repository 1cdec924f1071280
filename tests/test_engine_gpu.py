"""GPU parity tests: the H100 engine behind the MSCKF<_S> surface (through the C view / C-ABI of
libmsckf_b200.so) against the CPU oracle on identical seeded inputs.

What is asserted:
  * integer bookkeeping (valid / accepted flags = zero accept/reject flips, clone ids, tracked ids, counters): bit-exact,
    inside every case (tests/parity_cases.py);
  * every floating-point difference against 10 x its committed measurement (tests/golden/parity_measured.json, written by
    scripts/measure_parity.py on the H100): no hand-picked loose bounds -- a regression of more than one decade fails;
  * on top of that the contract tolerances of SURVEY.md 8d where the path meets them: fp64 vs the oracle's implementation-
    independent part (exact-subspace mode) <= 1e-9 relative on small windows; trajectory RMS < 1e-4 m.
The oracle modes: `clean` = exact subspace (drop_null_rows), `faithful` = reference-literal compression (its rows from
numerically zero pivots are rounding noise, DESIGN.md 4.4-2), fp32 cases compare the fp32 engine with the fp32 oracle DIRECTLY.
"""
import numpy as np
import pytest

from tests import parity_cases as pc
from tests.common import make_oracle, rel, run_collect, synth
from tests.parity_cases import make_engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nf,nc,seq", pc.WINDOWS)
def test_window_fp64_vs_clean_oracle(oracle_lib, nf, nc, seq):
    name = f"f64_clean_{nf}x{nc}"
    got = pc.check(name, pc.run_case(name))
    assert got["rank_engine"] == got["rank_oracle"]  # same rank decision
    if nf <= 40:  # the contract tolerance of SURVEY 8d (fp64 <= 1e-9) holds outright on the small windows
        assert got["dx"] < 1e-9 and got["P"] < 1e-9 and got["gamma"] < 1e-9


@pytest.mark.parametrize("nf,nc,seq", pc.WINDOWS)
def test_window_fp64_vs_reference_faithful_oracle(oracle_lib, nf, nc, seq):
    name = f"f64_faithful_{nf}x{nc}"
    pc.check(name, pc.run_case(name))


@pytest.mark.parametrize("nf,nc,seq", pc.WINDOWS)
def test_window_fp32_engine_vs_fp32_oracle_direct(oracle_lib, nf, nc, seq):
    """the fp32 engine against the fp32 oracle on identical float32 inputs: flips = 0 (inside the case), dx / P / gamma / p_f_G"""
    name = f"f32_direct_{nf}x{nc}"
    pc.check(name, pc.run_case(name))


def test_isotropic_noise_makes_null_rows_irrelevant(oracle_lib):
    """f_u == f_v => R_n = sigma^2 I: any basis of the subspace gives the reference result to rounding."""
    got = pc.check("f64_iso_40x12", pc.run_case("f64_iso_40x12"))
    assert got["dx"] < 1e-9 and got["P"] < 1e-9


@pytest.mark.parametrize("nf,nc,seq", pc.WINDOWS)
def test_window_fp32_as_close_to_fp64_truth_as_fp32_oracle(oracle_lib, nf, nc, seq):
    """second view of the fp32 path: its distance to the fp64 truth is the fp32 oracle's own distance (factor 4)"""
    wl = synth.make_window_workload(n_features=nf, n_clones=nc, seq=seq)
    g = make_engine(np.float32)
    o32 = make_oracle(oracle_lib, np.float32)
    o64 = make_oracle(oracle_lib, np.float64, drop_null_rows=True)
    pc.f32_inputs(g, o32, o64)
    rg = run_collect(g, wl)
    r32 = run_collect(o32, wl)
    run_collect(o64, wl)
    assert np.array_equal(rg["valid"], r32["valid"]) and np.array_equal(rg["accepted"], r32["accepted"])
    e_g = rel(g.lastDeltaX(), o64.lastDeltaX())
    e_o = rel(o32.lastDeltaX(), o64.lastDeltaX())
    assert e_g < 4 * e_o + 1e-4, (e_g, e_o)
    P64 = o64.getCovariance()
    eP_g = np.abs(g.getCovariance() - P64).max() / np.abs(P64).max()
    eP_o = np.abs(o32.getCovariance() - P64).max() / np.abs(P64).max()
    assert eP_g < 4 * eP_o + 1e-5, (eP_g, eP_o)


@pytest.mark.parametrize("mode", ["clean", "faithful"])
def test_config_s_shape_500x60_fp64_vs_oracle_fixture(mode):
    """BASELINE config-S shape (n = 375: the non-fused tail kernel, the fp64 k_jac without the single-warp gate copy) against
    the committed outputs of the oracle (which needs a minute of CPU here): zero flips, numbers vs measurement."""
    name = f"stress_f64_500x60_{mode}"
    got = pc.check(name, pc.run_case(name))
    assert got["m"] == 500 * 117
    if mode == "clean":
        assert got["rank_engine"] == got["rank_oracle"]


@pytest.mark.parametrize("mode", ["clean", "faithful"])
def test_config_s_full_2000x60_fp64_vs_oracle_fixture(mode):
    """the full BASELINE config S (2000 features x 60 clones, fp64; the oracle needs 4 minutes of CPU: committed fixture)"""
    name = f"stress_f64_2000x60_{mode}"
    got = pc.check(name, pc.run_case(name))
    assert got["m"] == 2000 * 117 and got["flips"] == 0


@pytest.mark.parametrize("mode", ["clean", "faithful"])
def test_config_b_fp32_vs_oracle_fixture(mode):
    name = f"configB_f32_300x30_{mode}"
    got = pc.check(name, pc.run_case(name))
    assert got["m"] == 300 * 57 and got["flips"] == 0


@pytest.mark.parametrize("name", ["win_f64_8x6_clean", "win_f64_40x12_clean", "win_f64_iso_40x12", "win_f64_3x4", "stream_f64_60"])
def test_engine_matches_numpy_golden(name):
    """engine vs the committed fixtures of the independent NumPy/LAPACK restatement (no oracle involved)."""
    pc.check(f"numpy_{name}", pc.run_case(f"numpy_{name}"))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stream_bookkeeping_bit_exact(oracle_lib, dtype):
    name = f"stream150_{np.dtype(dtype).name}"
    pc.check(name, pc.run_case(name))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stream_trajectory_rms_vs_oracle(oracle_lib, dtype):
    """north-star trajectory bar: RMS position difference engine vs oracle < 1e-4 m over the sequence (fp64 and fp32)"""
    name = f"traj200_{np.dtype(dtype).name}"
    got = pc.check(name, pc.run_case(name))
    assert got["rms_m"] < 1e-4, got
    assert got["rms_vs_truth_m"] < 0.1


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_prune_redundant_states(oracle_lib, dtype):
    """pruneRedundantStates (msckf.h:453-682): TRIANGULATE + RESIDUALIZE entry points and the covariance gather."""
    name = f"prune_redundant_{np.dtype(dtype).name}"
    pc.check(name, pc.run_case(name))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_rejections_and_pfg_index_quirk(oracle_lib, dtype):
    """outliers (LM cost / cheirality / chi-square gate) and checkMotion rejections, including the reference's
    p_f_G_vec mis-indexing after a checkMotion rejection (msckf.h:357 vs :374 vs :419, SURVEY.md 7-5)."""
    name = f"rejections_{np.dtype(dtype).name}"
    pc.check(name, pc.run_case(name))


def test_no_accepted_track_leaves_state_untouched(oracle_lib):
    wl = synth.make_window_workload(n_features=12, n_clones=6, seq=13)
    for fr in wl["frames"][1:]:
        fr["update"][0][:] += np.random.default_rng(5).normal(0, 0.2, fr["update"][0].shape)  # garbage tracks
    g = make_engine(np.float64)
    synth.drive(g, wl, marginalize_last=False)
    P0, s0 = g.getCovariance(), g.getImuState()
    g.marginalize()
    assert g.lastReport()["accepted"].sum() == 0
    assert np.array_equal(g.getCovariance(), P0)
    assert all(np.array_equal(g.getImuState()[k], s0[k]) for k in s0)
    assert g.counters()["n_updates"] == 0


def test_finish_residualises_remaining_tracks(oracle_lib):
    pc.check("finish", pc.run_case("finish"))


def test_handles_are_independent():
    wl_a = synth.make_window_workload(n_features=30, n_clones=8, seq=20)
    wl_b = synth.make_window_workload(n_features=25, n_clones=9, seq=21)
    solo = make_engine(np.float32)
    synth.drive(solo, wl_a)
    a, b = make_engine(np.float32), make_engine(np.float32)
    a.initialize(wl_a["camera"], wl_a["noise"], wl_a["params"], wl_a["imu_state"])
    b.initialize(wl_b["camera"], wl_b["noise"], wl_b["params"], wl_b["imu_state"])
    for k in range(9):
        for f, wl in ((a, wl_a), (b, wl_b)):
            if k >= len(wl["frames"]):
                continue
            fr = wl["frames"][k]
            for (w, acc, dT) in fr["imu"]:
                f.propagate(w, acc, dT)
            f.augmentState(fr["state_id"], fr["time"])
            if fr["update"] is not None:
                f.update(*fr["update"])
            if fr["add"] is not None:
                f.addFeatures(*fr["add"])
            f.marginalize()
            f.pruneEmptyStates()
    assert np.array_equal(a.getCovariance(), solo.getCovariance())  # bit-identical: deterministic kernels
    assert np.array_equal(a.getImuState()["p_I_G"], solo.getImuState()["p_I_G"])


@pytest.mark.parametrize("nf,nc,seq", [(40, 12, 4), (300, 30, 0)])
def test_fused_and_separate_substitution_agree(nf, nc, seq):
    """The tail kernel runs the forward substitution either fused into the blocked Cholesky (default where the window
    fits) or as a separate sweep (large windows; engine option 3 = 0): same factor, same results up to rounding."""
    name = f"fused_vs_separate_{nf}x{nc}"
    pc.check(name, pc.run_case(name))


def test_gram_on_fp64_tensor_cores_matches_simt_tiles():
    """engine option 5: the compression's Gram products as DMMA (mma.sync m8n8k4 f64) vs SIMT DFMA tiles -- same rank, same flags"""
    pc.check("gram_mma_vs_simt_300x30", pc.run_case("gram_mma_vs_simt_300x30"))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_track_group_sizes_of_the_feature_kernel_are_bit_identical(dtype):
    """engine option 6: k_jac works on a track with a group of 128 (one filter), 64 or 32 threads (device batches).  The
    floating-point sums are dealt to 128 virtual threads whatever the group, so all three give the same bits -- which is
    what lets a batch reproduce the filter run alone.  Config B (60 rows per track: more than one virtual warp)."""
    from msckf_mono_b200 import capi
    wl = synth.make_window_workload(n_features=300, n_clones=30, seq=1)
    out = []
    for g in (128, 64, 32):
        f = make_engine(dtype, max_clones=40, max_tracks=512, max_obs=512 * 30)
        synth.drive(f, wl, marginalize_last=False)
        capi.Engine(dtype, borrowed=f.engineHandle()).set_option(6, float(g))
        f.marginalize()
        rep = f.lastReport()
        out.append((f.getCovariance(), rep["gamma"].copy(), rep["accepted"].copy(), f.getImuState()["p_I_G"].copy()))
    assert out[0][2].sum() > 250
    for o in out[1:]:
        for a, b in zip(out[0], o):
            assert np.array_equal(a, b)


def test_tail_with_one_and_two_chain_ctas_agree_and_rank_pivots_show_the_gap():
    """engine option 7: the tail's chains of diagonal blocks on two CTAs of a 9-CTA cluster (default where the device accepts
    that cluster size) or on one CTA of an 8-CTA cluster (the fallback): same rank, same flags, results equal to rounding.
    `msckf_b200_rank_pivots` shows what the rank decision saw: n - rank pivots at rounding-noise level, far below the
    threshold, and every kept pivot far above it."""
    from msckf_mono_b200 import capi
    wl = synth.make_window_workload(n_features=300, n_clones=30, seq=0)
    out = []
    for chains in (2, 1):
        f = make_engine(np.float64, max_clones=40, max_tracks=512, max_obs=512 * 30)
        synth.drive(f, wl, marginalize_last=False)
        e = capi.Engine(np.float64, borrowed=f.engineHandle())
        e.set_option(7, float(chains))
        f.marginalize()
        pv = e.rank_pivots()
        out.append((f.getCovariance(), f.lastReport()["accepted"].copy(), f.counters()["rows_kept"], pv))
    (Pa, acca, ra, pva), (Pb, accb, rb, pvb) = out
    assert ra == rb and np.array_equal(acca, accb)
    assert np.max(np.abs(Pa - Pb)) <= 1e-7 * np.max(np.abs(Pa))
    for pv, r in ((pva, ra), (pvb, rb)):
        n = pv.size
        assert n == 15 + 6 * 30
        dropped = np.sort(pv)[: n - r]
        kept = np.sort(pv)[n - r:]
        assert np.all(np.abs(dropped) < 1e-10) and np.all(kept > 1e-6), (dropped, kept[:3])


def test_batched_entry_point_matches_individual_updates():
    """`msckf_mono_marginalize_batch` (host work on several threads, one stream per filter) gives bit-identical filters to
    calling marginalize() one by one."""
    from msckf_mono_b200.cview import marginalize_batch
    wls = [synth.make_window_workload(n_features=40 + 7 * i, n_clones=10 + i, seq=20 + i) for i in range(6)]
    one, many = [], []
    for wl in wls:
        a, b = make_engine(np.float32), make_engine(np.float32)
        synth.drive(a, wl, marginalize_last=False)
        synth.drive(b, wl, marginalize_last=False)
        one.append(a); many.append(b)
    for a in one:
        a.marginalize()
    marginalize_batch(many, threads=3)
    for a, b in zip(one, many):
        assert np.array_equal(a.getCovariance(), b.getCovariance())
        assert np.array_equal(a.getImuState()["p_I_G"], b.getImuState()["p_I_G"])
        ra, rb = a.lastReport(), b.lastReport()
        assert np.array_equal(ra["accepted"], rb["accepted"]) and np.array_equal(ra["gamma"], rb["gamma"])
        assert a.counters() == b.counters()


def test_persistent_batch_over_a_stream_is_bit_identical():
    """msckf_mono::MSCKFBatch (persistent device batch; the filters share its stream): four filters streamed in lockstep with
    propagate / augment / update / addFeatures per filter and ONE batched marginalize per frame -- including frames where some
    members have nothing queued -- end bit-identical to the same filters run alone."""
    from msckf_mono_b200.cview import FilterBatch
    wls = [synth.make_stream_workload(n_frames=40, seq=50 + i, max_features=25 + 5 * i, max_track_length=8 + 2 * i, max_cam_states=8 + i) for i in range(4)]
    solo, grp = [], []
    for wl in wls:
        a, b = make_engine(np.float32), make_engine(np.float32)
        for f in (a, b):
            f.initialize(wl["camera"], wl["noise"], wl["params"], wl["imu_state"])
        solo.append(a); grp.append(b)
    fb = FilterBatch(grp, threads=2)
    for k in range(40):
        for i, wl in enumerate(wls):
            fr = wl["frames"][k]
            for f in (solo[i], grp[i]):
                for (w, acc, dT) in fr["imu"]:
                    f.propagate(w, acc, dT)
                f.augmentState(fr["state_id"], fr["time"])
                f.update(*fr["update"])
                f.addFeatures(*fr["add"])
            solo[i].marginalize()
        fb.marginalize()
        for i in range(4):
            ra, rb = solo[i].lastReport(), grp[i].lastReport()
            assert np.array_equal(ra["accepted"], rb["accepted"]) and np.array_equal(ra["gamma"], rb["gamma"]), (k, i)
            solo[i].pruneEmptyStates(); grp[i].pruneEmptyStates()
    for a, b in zip(solo, grp):
        assert a.counters()["n_updates"] > 10 and a.counters() == b.counters()
        assert np.array_equal(a.getCovariance(), b.getCovariance())
        assert np.array_equal(a.getImuState()["p_I_G"], b.getImuState()["p_I_G"])
    fb.close()
    # after the batch is gone the filters run on their own streams again
    grp[0].marginalize()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bench_dump_is_what_the_class_getters_return(tmp_path, dtype):
    """bench.py --dump-outputs reads the corrected state through capi.Engine.state() / covariance() / delta_x(); the
    arrays must be the filters' own state as the drop-in class reports it, and past the size budget a seeded subset."""
    import bench
    from msckf_mono_b200 import capi
    filts, engs, reps = [], [], []
    for seq in (3, 4, 5):
        f = make_engine(dtype, max_clones=20, max_tracks=64, max_obs=64 * 12)
        synth.drive(f, synth.make_window_workload(n_features=40, n_clones=12, seq=seq))
        c = f.counters()
        filts.append(f)
        engs.append(capi.Engine(dtype, borrowed=f.engineHandle()))
        reps.append({"accepted": f.lastReport()["accepted"].copy(), "m": c["m"], "rank": c["rows_kept"]})
    n = 15 + 6 * filts[0].getNumCamStates()
    per_filter = 4 * (len(reps[0]["accepted"]) + 29 + 7 * filts[0].getNumCamStates() + n * n) + 8 * (2 + n)
    for max_bytes, count in ((64 << 20, 3), (2 * per_filter, 2)):
        out = tmp_path / str(count)
        bench.dump_outputs(out, engs, reps, max_bytes=max_bytes)
        d = {p.stem: np.load(p) for p in out.glob("*.npy")}
        idx = d["filter_index"].astype(int)
        assert len(idx) == count and len(set(idx)) == count
        assert sum(a.nbytes for k, a in d.items() if k != "filter_index") <= max_bytes
        for row, i in enumerate(idx):
            f, s, cs = filts[i], filts[i].getImuState(), filts[i].getCamStates()
            imu = np.concatenate([s[k] for k in ("p_I_G", "v_I_G", "b_g", "b_a", "g", "q_IG", "p_I_G_null", "v_I_G_null", "q_IG_null")])
            np.testing.assert_array_equal(d["imu_state"][row], imu.astype(dtype).astype(np.float32))
            np.testing.assert_array_equal(d["clone_poses"][row], np.hstack([cs["p_C_G"], cs["q_CG"]]).astype(dtype).astype(np.float32))
            np.testing.assert_array_equal(d["covariance"][row], f.getCovariance().astype(dtype).astype(np.float32))
            np.testing.assert_array_equal(d["accepted"][row], reps[i]["accepted"])
            np.testing.assert_array_equal(d["m_rank"][row], [reps[i]["m"], reps[i]["rank"]])
            assert np.isfinite(d["delta_x"][row]).all() and d["delta_x"].shape[1] == n


def test_window_growth_and_single_observation_tracks():
    """Capacities are initial sizes (the reference's window and track lists are unbounded std::vectors): a filter created
    for 6 clones / 8 tracks grows through 14 clones and 40 tracks and matches a filter that was created large.  A track
    with one observation (min_track_length = 1) is reported as rejected instead of failing the batch."""
    wl = synth.make_window_workload(n_features=40, n_clones=14, seq=4)
    small = make_engine(np.float64, max_clones=6, max_tracks=8, max_obs=16)
    big = make_engine(np.float64, max_clones=40, max_tracks=512, max_obs=512 * 30)
    synth.drive(small, wl)
    synth.drive(big, wl)
    assert np.array_equal(small.getCovariance(), big.getCovariance())
    assert np.array_equal(small.lastReport()["accepted"], big.lastReport()["accepted"])
    from msckf_mono_b200 import capi
    e = capi.Engine(np.float64, borrowed=big.engineHandle())
    M = e.num_clones()
    off = np.array([0, 1, 4], dtype=np.int32)          # track 0: one observation; track 1: three
    idx = np.array([0, 0, 1, 2], dtype=np.int32)
    obs = np.zeros(8)
    rep = e.update(capi.MARGINALIZE, capi.TrackBatch(off, obs, idx, np.float64))
    assert M >= 3 and rep["accepted"][0] == 0


def test_c_abi_update_batch_matches_separate_updates():
    """`msckf_b200_update_batch` on the raw C-ABI: engines whose state was copied from driven filters, the queued batches
    replayed through the batched entry point -> same m, rank, accept flags and bit-identical covariance as one-by-one."""
    from msckf_mono_b200 import capi
    wls = [synth.make_window_workload(n_features=30 + 9 * i, n_clones=9 + i, seq=40 + i) for i in range(5)]
    engines, batches, ref = [], [], []
    for wl in wls:
        f = make_engine(np.float64, max_clones=40, max_tracks=512, max_obs=512 * 30)  # same capacities as capi.Engine's defaults
        synth.drive(f, wl, marginalize_last=False)
        off, obs, idx = f.packQueued()
        src = capi.Engine(np.float64, borrowed=f.engineHandle())
        e = capi.Engine(np.float64)
        e.copy_state_from(src)
        engines.append(e)
        batches.append(capi.TrackBatch(off, obs, idx, np.float64))
        f.marginalize()
        rep = f.lastReport()
        ref.append((f.getCovariance(), rep["accepted"].copy(), f.counters()))
    reps = capi.update_batch(engines, capi.MARGINALIZE, batches, threads=4)
    for e, r, (P, acc, cnt) in zip(engines, reps, ref):
        assert np.array_equal(r["accepted"].astype(bool), acc.astype(bool))
        assert r["m"] == cnt["m"] and r["rank"] == cnt["rows_kept"]
        assert np.array_equal(e.covariance(), P)


def test_maximum_track_length_98_fp64(oracle_lib):
    """The reference's chi-square table has 99 entries (msckf.h:91), so 98 observations per track is the longest track it
    can gate.  98 clones -> n = 603: the large-window tail kernel (blocks of 16) and the CTA-wide gate -- paths the other
    tests do not reach."""
    got = pc.check("l98_f64", pc.run_case("l98_f64"))
    # 7 gauge directions; one of them is only nearly null at this geometry, and the two implementations' thresholds
    # (pivot of the basis Gram matrix vs. a pivoted QR) land on either side of it -- with no effect on the result above
    assert got["rank_oracle"] in (603 - 7, 603 - 6) and got["rank_engine"] in (603 - 7, 603 - 6)


def test_engine_update_is_invariant_to_track_order():
    """Same property as tests/test_oracle.py::test_update_is_invariant_to_track_order, on the engine alone (isotropic
    pixel noise): permuting the features permutes the per-track outputs and leaves the update unchanged."""
    pc.check("order_invariance", pc.run_case("order_invariance"))


def test_non_finite_update_is_reported_not_hidden():
    """MSCKF_B200_ERR_NUMERIC: a covariance poisoned with NaN makes the update non-finite; the engine applies it like the
    reference would (msckf.h:1369-1418 has no check) and says so through the fetch status."""
    from msckf_mono_b200 import capi
    wl = synth.make_window_workload(n_features=12, n_clones=6, seq=13)
    f = make_engine(np.float64)
    synth.drive(f, wl, marginalize_last=False)
    off, obs, idx = f.packQueued()
    e = capi.Engine(np.float64, borrowed=f.engineHandle())
    ok = capi.Engine(np.float64)
    ok.copy_state_from(e)
    assert ok.update(capi.MARGINALIZE, capi.TrackBatch(off, obs, idx, np.float64))["m"] > 0
    bad = capi.Engine(np.float64)
    bad.copy_state_from(e)
    bad.poison_covariance()
    with pytest.raises(RuntimeError, match="non-finite"):
        bad.update(capi.MARGINALIZE, capi.TrackBatch(off, obs, idx, np.float64))


def test_full_size_properties_stress_fp64():
    """BASELINE config S (2000 features x 60 clones, fp64): size-independent properties: exact symmetry, positive
    semi-definiteness, information gain, rank = n - 7 gauge directions, every track accepted (the oracle's flags: fixture)."""
    wl = synth.make_window_workload(n_features=2000, n_clones=60, seq=30)
    g = make_engine(np.float64, max_clones=64, max_tracks=2048, max_obs=2048 * 60)
    synth.drive(g, wl, marginalize_last=False)
    P0 = g.getCovariance()
    g.marginalize()
    rep = g.lastReport()
    assert rep["valid"].all() and rep["accepted"].all()  # = the oracle's flags (tests/golden/stress_f64_2000x60_*.npz): zero flips
    P1 = g.getCovariance()
    n = P1.shape[0]
    assert n == 15 + 6 * 60 and np.isfinite(P1).all()
    assert np.array_equal(P1, P1.T)
    w = np.linalg.eigvalsh(P1)
    assert w.min() > -1e-9 * w.max()
    d = np.linalg.eigvalsh(P0 - P1)
    assert d.min() > -1e-9 * np.abs(d).max()
    assert np.trace(P1) < 0.9 * np.trace(P0)
    c = g.counters()
    assert c["m"] == int(rep["rows"].sum()) and c["rows_kept"] in (n - 7, n - 6)  # 7 gauge directions (one is only nearly null)


def test_config_b_all_accepted_fp32():
    """BASELINE config B (300 x 30 fp32): every track is accepted so m = 300 * 57 exactly (SURVEY.md 8d)."""
    wl = synth.make_window_workload(n_features=300, n_clones=30, seq=0)
    g = make_engine(np.float32)
    synth.drive(g, wl)
    rep = g.lastReport()
    assert rep["accepted"].all() and g.counters()["m"] == 300 * 57
    P = g.getCovariance()
    assert np.array_equal(P, P.T) and np.isfinite(P).all()
