"""The drop-in boundary compiles for a reference-shaped caller (VERDICT r01 item 3).

`tests/stub/caller_shaped.cpp` uses every boundary symbol the reference's two callers use (datasets/asl_msckf.cpp,
src/ros_interface.cpp): the type aliases of msckf_mono/types.h, msckf_mono/matrix_utils.h, the class surface with the
reference's signatures, a const filter, a container of filters.  It is compiled and run (over the recording stub of the
C-ABI, no GPU) in both configurations of types.h: the Eigen-free stand-ins, and the Eigen branch against a mock of the
Eigen names (this image has no Eigen; tests/stub/mini_eigen says what that does and does not prove)."""
import re
import subprocess

import pytest

from tests.common import ROOT
from tests.fake_engine import build_program

SRC = ROOT / "tests" / "stub" / "caller_shaped.cpp"


def build_and_run(tmp_path, name, extra):
    exe = build_program(tmp_path / name, [SRC], flags=["-Wall", "-Werror=return-type", *extra])
    return subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout


def test_caller_shaped_tu_compiles_and_runs_with_pod_types(tmp_path):
    out = build_and_run(tmp_path, "caller_pod", ["-DMSCKF_B200_NO_EIGEN"])
    m = re.search(r"clones (\d+) tracked (\d+) pruned (\d+)", out)
    assert m and int(m.group(1)) >= 1 and int(m.group(3)) > 0, out
    assert "moved clones" in out and "skew -0.3 omega -0.1" in out


def test_eigen_branch_of_the_headers_compiles_against_the_mock(tmp_path):
    out_pod = build_and_run(tmp_path, "caller_pod", ["-DMSCKF_B200_NO_EIGEN"])
    out_eig = build_and_run(tmp_path, "caller_eigen", [f"-I{ROOT / 'tests' / 'stub' / 'mini_eigen'}"])
    assert out_eig == out_pod  # same bookkeeping through either branch of types.h


def test_every_reference_boundary_symbol_is_declared():
    """reference include/msckf_mono/types.h:8-126 and matrix_utils.h:8-87, name for name (listed in INTEGRATION.md)"""
    types = (ROOT / "include" / "msckf_mono" / "types.h").read_text()
    for name in ["Quaternion", "Matrix3", "Matrix4", "MatrixX", "RowVector3", "Vector2", "Vector3", "Vector4", "VectorX", "Point", "GyroscopeReading",
                 "AccelerometerReading", "Isometry3"]:
        assert len(re.findall(rf"using {name} =", types)) == 2, name  # Eigen branch and POD branch
    for name in ["Camera", "camState", "imuState", "imuReading", "noiseParams", "MSCKFParams", "featureTrackToResidualize", "featureTrack"]:
        assert re.search(rf"struct {name} {{", types), name
    assert "std::vector<camState<_Scalar>> cam_states;" in types  # featureTrackToResidualize::cam_states (types.h:107)
    utils = (ROOT / "include" / "msckf_mono" / "matrix_utils.h").read_text()
    for name in ["vectorToSkewSymmetric", "omegaMat", "skewSymmetricToVector", "cond", "square_slice", "column_slice"]:
        assert re.search(rf"\b{name}\(", utils), name
    shim = (ROOT / "include" / "msckf_mono" / "msckf.h").read_text()
    for sig in ["void initialize(const Camera<_S>& camera, const noiseParams<_S>& noise_params, const MSCKFParams<_S>& msckf_params,",
                "void propagate(imuReading<_S>& measurement_)", "void augmentState(const int& state_id, const _S& time)",
                "void update(const aligned_vector<Vector2<_S>>& measurements, const std::vector<size_t>& feature_ids)",
                "void addFeatures(const aligned_vector<Vector2<_S>>& features, const std::vector<size_t>& feature_ids)", "void marginalize()",
                "void pruneRedundantStates()", "void pruneEmptyStates()", "void finish()", "inline size_t getNumCamStates()",
                "inline imuState<_S> getImuState()", "inline aligned_vector<Vector3<_S>> getMap()", "inline Camera<_S> getCamera()",
                "inline camState<_S> getCamState(size_t i)", "inline std::vector<camState<_S>> getCamStates() const",
                "inline std::vector<camState<_S>> getPrunedStates()"]:
        assert sig in shim, sig
