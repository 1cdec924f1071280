"""The ROS-free ASL player (C++ host over the drop-in class shim, `msckf_mono_b200/asl/asl_player.cpp`) on an H100:
the same on-disk sequence is played by the compiled player through `msckf_mono::MSCKF<_S>` and, for the check, by the
CPU oracle driven from Python with the reference's call order.  Bar (BASELINE north star): trajectories agree to
< 1e-4 m RMS; the clone-window size per frame (pruning bookkeeping) is identical."""
import numpy as np
import pytest

from msckf_mono_b200 import asl, synth
from tests.common import make_oracle

pytestmark = pytest.mark.gpu


def _oracle_trajectory(oracle_lib, wl, dtype):
    o = make_oracle(oracle_lib, dtype, drop_null_rows=True)
    pos, ncl = [], []

    def grab(k, f):
        pos.append(np.array(f.getImuState()["p_I_G"], float))
        ncl.append(f.getNumCamStates())

    synth.drive(o, wl, prune_redundant=True, on_frame=grab)
    return np.array(pos), np.array(ncl)


@pytest.mark.parametrize("dtype,name,tol", [(np.float64, "f64", 1e-4), (np.float32, "f32", 2e-3)])
def test_player_trajectory_matches_oracle(oracle_lib, tmp_path, dtype, name, tol):
    wl = synth.make_stream_workload(n_frames=120, seq=1, max_features=60)
    mav0 = asl.write_mav0(wl, str(tmp_path))
    out = str(tmp_path / f"traj_{name}.csv")
    summary = asl.run_player(mav0, dtype=name, out=out, state_id="frame")
    assert summary["frames"] == 120 and summary["gt_matched"] == 120
    tr = asl.read_trajectory(out)
    pos_o, ncl_o = _oracle_trajectory(oracle_lib, wl, dtype)
    rms = float(np.sqrt(np.mean(np.sum((tr["p"] - pos_o) ** 2, axis=1))))
    print(f"asl_player {name}: RMS vs oracle {rms:.3e} m, RMSE vs ground truth {summary['position_rmse_m']:.3e} m, "
          f"{summary['frames_per_s']:.0f} frames/s")
    assert np.array_equal(tr["n_clones"], ncl_o)  # window bookkeeping (pruneRedundantStates / pruneEmptyStates): exact
    # fp64: the BASELINE bar (1e-4 m).  fp32: two fp32 implementations of a 120-frame dead-reckoning + update stream differ
    # by accumulated rounding; the bound is a few times what the fp32 oracle itself is away from the fp64 oracle.
    assert rms < tol, rms
    assert np.isfinite(summary["position_rmse_m"]) and summary["position_rmse_m"] < 1.0
