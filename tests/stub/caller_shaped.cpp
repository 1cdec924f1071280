// tests/stub/caller_shaped.cpp -- TEST INFRASTRUCTURE ONLY.
// A translation unit shaped like the reference's two callers of msckf_mono::MSCKF<float> -- the ASL dataset driver
// (/root/reference/datasets/asl_msckf.cpp:57-160 set-up, :229-298 per-reading / per-image loop, :339-409 getters) and the
// ROS node's set-up (/root/reference/src/ros_interface.cpp:250-262 Matrix4 T_cam_imu, :92-116 frame loop) -- written against
// the drop-in headers of THIS repo.  It touches every boundary symbol those callers use: the type aliases of types.h
// (Matrix4, Matrix3, Vector3, Quaternion, aligned vectors of Vector2), matrix_utils.h, the class surface with the
// reference's exact signatures, a const filter, a container of filters.  Linked against the recording fake of the C-ABI
// (tests/stub/stub_*.cpp, no GPU) it runs a few frames and prints a checksum of the integer bookkeeping.  Compiled twice by
// tests/test_dropin_boundary_cpu.py: with the POD stand-ins (MSCKF_B200_NO_EIGEN) and through the Eigen branch against
// tests/stub/mini_eigen (a mock of the Eigen names, since this image has no Eigen).
#include <cstdio>
#include <iostream>
#include <vector>

#include <msckf_mono/matrix_utils.h>
#include <msckf_mono/msckf.h>

using namespace msckf_mono;
#ifdef MSCKF_B200_HAVE_EIGEN
template <class T> using ref_vector = std::vector<T, Eigen::aligned_allocator<T>>;  // spelled like the reference's callers
#else
template <class T> using ref_vector = aligned_vector<T>;
#endif

static size_t count_tracked(const MSCKF<float>& filter) {  // getCamStates() is const in the reference (msckf.h:835)
  size_t n = 0;
  for (const auto& cs : filter.getCamStates()) n += cs.tracked_feature_ids.size();
  return n;
}

int main() {
  // ---- ros_interface.cpp:250-262: extrinsics from a 4x4
  Matrix4<float> T_cam_imu;
  T_cam_imu.setZero();
  for (int i = 0; i < 4; ++i) T_cam_imu(i, i) = 1.f;
  T_cam_imu(0, 3) = 0.02f; T_cam_imu(1, 3) = -0.05f;
  Matrix3<float> R_cam_imu = T_cam_imu.block<3, 3>(0, 0);
  Vector3<float> p_cam_imu = T_cam_imu.block<3, 1>(0, 3);
  Matrix3<float> R_imu_cam = R_cam_imu.transpose();
  Vector3<float> p_imu_cam = R_imu_cam * (-1.f * p_cam_imu);
  (void)p_imu_cam;

  Camera<float> camera;
  camera.f_u = 458.654f; camera.f_v = 457.296f; camera.c_u = 367.215f; camera.c_v = 248.375f; camera.b = 0;
  camera.q_CI = Quaternion<float>(R_cam_imu).inverse();
  camera.p_C_I = p_cam_imu;
  const auto q_CI = camera.q_CI;
  std::cout << "q_CI " << q_CI.x() << "," << q_CI.y() << "," << q_CI.z() << "," << q_CI.w() << " p_C_I " << camera.p_C_I.transpose() << std::endl;

  // ---- asl_msckf.cpp:73-125: noise and filter parameters
  const float feature_cov = 7;
  noiseParams<float> noise_params;
  noise_params.u_var_prime = std::pow(feature_cov / camera.f_u, 2);
  noise_params.v_var_prime = std::pow(feature_cov / camera.f_v, 2);
  FixedMatrix<float, 12, 1> Q_imu_vars;
  const float w_var = 1e-5f, dbg_var = 3.6733e-5f, a_var = 1e-3f, dba_var = 7e-4f;
  Q_imu_vars << w_var, w_var, w_var, dbg_var, dbg_var, dbg_var, a_var, a_var, a_var, dba_var, dba_var, dba_var;
  noise_params.Q_imu = Q_imu_vars.asDiagonal();
  FixedMatrix<float, 15, 1> IMUCovar_vars;
  IMUCovar_vars << 1e-5f, 1e-5f, 1e-5f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-12f, 1e-12f, 1e-12f;
  noise_params.initial_imu_covar = IMUCovar_vars.asDiagonal();
  MSCKFParams<float> msckf_params;
  msckf_params.max_gn_cost_norm = std::pow(11.f / camera.f_u, 2);
  msckf_params.translation_threshold = 0.05f;
  msckf_params.min_rcond = 3e-12f;
  msckf_params.redundancy_angle_thresh = 0.005f;
  msckf_params.redundancy_distance_thresh = 0.05f;
  msckf_params.max_track_length = 1000;  // the reference's default: "wait for features to go out of view"
  msckf_params.min_track_length = 3;
  msckf_params.max_cam_states = 20;

  imuState<float> firstImuState;
  firstImuState.b_a = Vector3<float>();
  firstImuState.b_g = Vector3<float>();
  firstImuState.g << 0.0, 0.0, -9.81;
  firstImuState.q_IG = Quaternion<float>(1, 0, 0, 0);
  firstImuState.p_I_G = Vector3<float>();
  firstImuState.v_I_G = Vector3<float>();

  std::vector<MSCKF<float>> filters;  // a container of filters (movable, like any value type)
  filters.emplace_back();
  MSCKF<float>& msckf = filters.back();
  msckf.initialize(camera, noise_params, msckf_params, firstImuState);
  imuState<float> imu_state = msckf.getImuState();
  auto q = imu_state.q_IG;
  std::cout << "p_I_G " << imu_state.p_I_G.transpose() << " q_IG " << q.w() << "," << q.x() << "," << q.y() << "," << q.z()
            << " world_adjusted_a " << (q.toRotationMatrix().transpose() * (Vector3<float>() - imu_state.b_a)).transpose() << std::endl;

  // matrix_utils.h (reached by the reference's front end through corner_detector.h:24)
  Vector3<float> w; w << 0.1f, -0.2f, 0.3f;
  const Matrix3<float> sk = vectorToSkewSymmetric(w);
  const Matrix4<float> Om = omegaMat(w);
  MatrixX<float> big(4, 4), sub;
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) big(i, j) = Om(i, j);
  IndexVector inds(2); inds(0) = 0; inds(1) = 3;
  square_slice(big, inds, sub);
  FixedMatrix<float, 3, DynamicSize> cols(3, 4), csub;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) cols(i, j) = (float)(10 * i + j);
  column_slice<float, 3>(cols, inds, csub);
  std::printf("skew %g omega %g slice %g %g cols %g\n", sk(0, 1), Om(3, 0), sub(0, 1), sub(1, 0), csub(2, 1));

  // ---- asl_msckf.cpp:229-298: per reading propagate (+ getImuState before it), per image the update sequence
  int state_k = 0;
  size_t next_id = 1;
  std::vector<size_t> live;
  for (int frame = 0; frame < 30; ++frame) {
    for (int k = 0; k < 10; ++k) {
      state_k++;
      imuReading<float> imu_data;
      imu_data.omega << 0.01f, 0.0f, 0.02f;
      imu_data.a << 0.f, 0.f, 9.81f;
      imu_data.dT = 0.005f;
      imuState<float> prev_imu_state = msckf.getImuState();
      Quaternion<float> prev_rotation = prev_imu_state.q_IG;
      (void)prev_rotation;
      msckf.propagate(imu_data);
      Vector3<float> cam_frame_av = (camera.q_CI.inverse() * (imu_data.omega - prev_imu_state.b_g));
      (void)cam_frame_av;
    }
    ref_vector<Vector2<float>> cur_features, new_features;
    std::vector<size_t> cur_ids, new_ids;
    for (size_t id : live)
      if ((id + frame) % 7 != 0) { Vector2<float> z; z << 0.01f * (float)(id % 13), -0.02f * (float)(id % 5); cur_features.push_back(z); cur_ids.push_back(id); }
    for (int k = 0; k < 4; ++k) { Vector2<float> z; z << 0.1f * k, 0.05f; new_features.push_back(z); new_ids.push_back(next_id++); }
    msckf.augmentState(state_k, 0.05f * frame);
    msckf.update(cur_features, cur_ids);
    msckf.addFeatures(new_features, new_ids);
    msckf.marginalize();
    msckf.pruneRedundantStates();
    msckf.pruneEmptyStates();
    live = cur_ids;
    live.insert(live.end(), new_ids.begin(), new_ids.end());
    // ---- asl_msckf.cpp:300-409: what the publishers read
    auto st = msckf.getImuState();
    Quaternion<float> q_out = st.q_IG.inverse();
    (void)q_out;
    ref_vector<Vector3<float>> map = msckf.getMap();
    for (auto& point : map) (void)point(0);
    for (auto& cs : msckf.getCamStates()) { (void)cs.p_C_G[0]; (void)cs.q_CG.inverse(); (void)cs.time; (void)cs.state_id; }
    for (auto ci : msckf.getPrunedStates()) (void)ci.p_C_G[2];
  }
  msckf.finish();
  const MSCKF<float>& cref = msckf;
  std::printf("clones %zu tracked %zu pruned %zu camera_fu %g\n", msckf.getNumCamStates(), count_tracked(cref), msckf.getPrunedStates().size(),
              msckf.getCamera().f_u);
  MSCKF<float> moved = std::move(filters.back());  // move construction keeps the engine alive in the new object
  std::printf("moved clones %zu state0 %d\n", moved.getNumCamStates(), moved.getNumCamStates() ? moved.getCamState(0).state_id : -1);
  return 0;
}
