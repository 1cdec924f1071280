"""Occupancy of the feature kernel in a device batch: k_jac<float, 32> (a warp per track, two tracks per CTA) must hold 10 CTAs
= 20 tracks per SM at config B (300 tracks x 30 clones, fp32), so that a batch of 8 filters (2 400 tracks) runs in one wave on
the H100's 132 SMs (2 640 resident tracks).  Shared memory sets that figure: a few hundred bytes more per CTA give 9 CTAs and a
second wave (DESIGN.md 4.2)."""
import numpy as np
import pytest

from tests.common import synth

pytestmark = pytest.mark.gpu


def test_feature_kernel_holds_ten_ctas_per_sm_at_config_b():
    from msckf_mono_b200 import capi, engine_filter
    caps = dict(max_clones=38, max_tracks=512, max_obs=512 * 30)
    tmpl, batches, work = [], [], []
    for seq in (0, 1):
        f = engine_filter(np.float32, **caps)
        synth.drive(f, synth.make_window_workload(n_features=300, n_clones=30, seq=seq), marginalize_last=False)
        off, obs, idx = f.packQueued()
        batches.append(capi.TrackBatch(off, obs, idx, np.float32))
        tmpl.append(f)
        work.append(capi.Engine(np.float32, **caps))
        work[-1].copy_state_from(capi.Engine(np.float32, borrowed=f.engineHandle()))
    b = capi.Batch(work)
    try:
        assert b.jac_occupancy() == 0  # nothing launched yet
        b.stage(capi.MARGINALIZE, batches)
        b.launch()
        reps = b.fetch(batches)
        assert all(r["m"] == 300 * 57 for r in reps)  # the bench shape: every track accepted, L = 30 throughout
        assert b.jac_occupancy() >= 10
    finally:
        b.close()
