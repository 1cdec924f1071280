// msckf_mono_b200/asl/asl_player.cpp
// ROS-free ASL / EuRoC player + trajectory evaluator (SURVEY.md 8f-3): drives msckf_mono::MSCKF<_S> -- the drop-in shim
// over the H100 engine -- with the call order of the reference's dataset front end
// (/root/reference/datasets/asl_msckf.cpp:206-296: per IMU reading propagate(); per image augmentState, update,
// addFeatures, marginalize, pruneRedundantStates, pruneEmptyStates), from a mav0 folder with PRE-EXTRACTED feature tracks
// (cam0/tracks.csv; the FAST/KLT image front end is out of scope, SURVEY.md 8f-4).  Deliberately NOT copied: the
// reference drops frames when its wall clock falls behind the dataset clock (asl_msckf.cpp:262-264), which makes its
// output non-deterministic.  The filter starts from the ground-truth row of the first image, like the reference.
//
//   asl_player --mav0 DIR [--dtype f32|f64] [--out traj.csv] [--max-frames N] [--prune-redundant 0|1]
//              [--state-id imu|frame] [--device K] [--dry-run]
// prints one JSON line: frames, imu readings, updates, position RMSE vs ground truth, wall time.
#include <chrono>
#include <cstring>
#include <set>
#include <string>

#include "asl_io.hpp"
#include <msckf_mono/msckf.h>

namespace asl = msckf_b200::asl;

struct Options {
  std::string mav0, out;
  std::string dtype = "f32", state_id = "imu";
  int max_frames = -1, device = 0;
  bool prune_redundant = true, dry_run = false;
};

template <class S>
static int run(const Options& o) {
  using namespace msckf_mono;
  const auto imu = asl::read_imu(o.mav0);
  const auto gt = asl::read_groundtruth(o.mav0);
  const auto tracks = asl::read_tracks(o.mav0);
  const auto frames = asl::read_frame_times(o.mav0);
  const auto cam = asl::read_camera(o.mav0);
  const auto fc = asl::read_filter_config(o.mav0);
  if (frames.empty()) throw std::runtime_error("cam0/data.csv has no frames");
  if (o.dry_run) {  // parse-only mode: counts and checksums of what was read (no GPU involved)
    double cs_imu = 0, cs_tr = 0;
    for (const auto& r : imu) cs_imu += r.w[0] + r.w[1] + r.w[2] + r.a[0] + r.a[1] + r.a[2];
    unsigned long long cs_id = 0;
    for (const auto& r : tracks) { cs_tr += r.x + r.y; cs_id += r.id; }
    std::printf("{\"dry_run\": true, \"frames\": %zu, \"imu\": %zu, \"groundtruth\": %zu, \"track_rows\": %zu, \"imu_checksum\": %.17g, "
                "\"track_checksum\": %.17g, \"id_checksum\": %llu, \"fu\": %.17g, \"fv\": %.17g, \"T_BS_03\": %.17g, "
                "\"max_track_length\": %d, \"feature_cov\": %.17g}\n",
                frames.size(), imu.size(), gt.size(), tracks.size(), cs_imu, cs_tr, cs_id, cam.fu, cam.fv, cam.T_BS[3],
                fc.max_track_length, fc.feature_cov);
    return 0;
  }
  // ---- camera: q_CI rotates IMU -> camera = inverse of R_BS; p_C_I = p_BS (asl_readers.cpp:27-33)
  Camera<S> camera;
  camera.f_u = (S)cam.fu; camera.f_v = (S)cam.fv; camera.c_u = (S)cam.cu; camera.c_v = (S)cam.cv; camera.b = S(0);
  {
    const double R_BS[9] = {cam.T_BS[0], cam.T_BS[1], cam.T_BS[2], cam.T_BS[4], cam.T_BS[5], cam.T_BS[6], cam.T_BS[8], cam.T_BS[9], cam.T_BS[10]};
    const double R_CI[9] = {R_BS[0], R_BS[3], R_BS[6], R_BS[1], R_BS[4], R_BS[7], R_BS[2], R_BS[5], R_BS[8]};
    double q[4];
    asl::rot_to_quat(R_CI, q);
    camera.q_CI = Quaternion<S>((S)q[0], (S)q[1], (S)q[2], (S)q[3]);
    camera.p_C_I(0) = (S)cam.T_BS[3]; camera.p_C_I(1) = (S)cam.T_BS[7]; camera.p_C_I(2) = (S)cam.T_BS[11];
  }
  // ---- noise and parameters (asl_msckf.cpp:73-125)
  noiseParams<S> noise;
  noise.u_var_prime = (S)std::pow(fc.feature_cov / cam.fu, 2);
  noise.v_var_prime = (S)std::pow(fc.feature_cov / cam.fv, 2);
  noise.Q_imu.setZero();
  noise.initial_imu_covar.setZero();
  for (int i = 0; i < 3; ++i) {
    noise.Q_imu(i, i) = (S)fc.w_var; noise.Q_imu(3 + i, 3 + i) = (S)fc.dbg_var;
    noise.Q_imu(6 + i, 6 + i) = (S)fc.a_var; noise.Q_imu(9 + i, 9 + i) = (S)fc.dba_var;
    noise.initial_imu_covar(i, i) = (S)fc.q_var_init; noise.initial_imu_covar(3 + i, 3 + i) = (S)fc.bg_var_init;
    noise.initial_imu_covar(6 + i, 6 + i) = (S)fc.v_var_init; noise.initial_imu_covar(9 + i, 9 + i) = (S)fc.ba_var_init;
    noise.initial_imu_covar(12 + i, 12 + i) = (S)fc.p_var_init;
  }
  MSCKFParams<S> params;
  params.max_gn_cost_norm = (S)std::pow(fc.max_gn_cost_norm / cam.fu, 2);
  params.min_rcond = (S)fc.min_rcond;
  params.translation_threshold = (S)fc.translation_threshold;
  params.redundancy_angle_thresh = (S)fc.redundancy_angle_thresh;
  params.redundancy_distance_thresh = (S)fc.redundancy_distance_thresh;
  params.min_track_length = fc.min_track_length;
  params.max_track_length = fc.max_track_length;
  params.max_cam_states = fc.max_cam_states;
  // ---- initial state: the ground-truth row at (or the last one before) the first image
  const asl::GtRow* g0 = nullptr;
  for (const auto& g : gt) { if (g.t_ns <= frames[0]) g0 = &g; else break; }
  if (!g0) { if (gt.empty()) throw std::runtime_error("no ground truth to start from"); g0 = &gt[0]; }
  imuState<S> x0;
  for (int i = 0; i < 3; ++i) {
    x0.p_I_G(i) = (S)g0->p[i]; x0.v_I_G(i) = (S)g0->v[i]; x0.b_g(i) = (S)g0->bw[i]; x0.b_a(i) = (S)g0->ba[i]; x0.g(i) = (S)fc.gravity[i];
  }
  x0.q_IG = Quaternion<S>((S)g0->q_wxyz[0], (S)-g0->q_wxyz[1], (S)-g0->q_wxyz[2], (S)-g0->q_wxyz[3]);  // q_IG = conj(q_RS)

  MSCKF<S> msckf;
  msckf.setEngineOptions(o.device);
  msckf.initialize(camera, noise, params, x0);

  std::vector<asl::PoseRow> traj;
  std::set<uint64_t> seen;
  size_t ii = 0, ti = 0;
  while (ii < imu.size() && imu[ii].t_ns <= frames[0]) ++ii;  // readings up to the first image only set the previous time
  int64_t t_prev_imu = (ii > 0) ? imu[ii - 1].t_ns : frames[0];
  int state_k = 0;
  long n_imu = 0, n_frames = 0;
  const auto wall0 = std::chrono::steady_clock::now();
  for (size_t fi = 0; fi < frames.size(); ++fi) {
    if (o.max_frames >= 0 && (int)fi >= o.max_frames) break;
    const int64_t tf = frames[fi];
    for (; ii < imu.size() && imu[ii].t_ns <= tf; ++ii) {  // asl_msckf.cpp:233-246
      imuReading<S> m;
      for (int i = 0; i < 3; ++i) { m.omega(i) = (S)imu[ii].w[i]; m.a(i) = (S)imu[ii].a[i]; }
      m.dT = (S)((double)(imu[ii].t_ns - t_prev_imu) / 1e9);
      t_prev_imu = imu[ii].t_ns;
      msckf.propagate(m);
      ++state_k;
      ++n_imu;
    }
    aligned_vector<Vector2<S>> cur, fresh;
    std::vector<size_t> cur_ids, fresh_ids;
    while (ti < tracks.size() && tracks[ti].t_ns < tf) ++ti;
    for (; ti < tracks.size() && tracks[ti].t_ns == tf; ++ti) {
      Vector2<S> z;
      z(0) = (S)tracks[ti].x; z(1) = (S)tracks[ti].y;
      if (seen.insert(tracks[ti].id).second) { fresh.push_back(z); fresh_ids.push_back((size_t)tracks[ti].id); }
      else { cur.push_back(z); cur_ids.push_back((size_t)tracks[ti].id); }
    }
    msckf.augmentState(o.state_id == "frame" ? (int)fi : state_k, (S)((double)tf / 1e9));  // asl_msckf.cpp:270
    msckf.update(cur, cur_ids);
    msckf.addFeatures(fresh, fresh_ids);
    msckf.marginalize();
    if (o.prune_redundant) msckf.pruneRedundantStates();
    msckf.pruneEmptyStates();
    const auto s = msckf.getImuState();
    asl::PoseRow r;
    r.t_ns = tf;
    for (int i = 0; i < 3; ++i) r.p[i] = (double)s.p_I_G(i);
    r.q_wxyz[0] = (double)s.q_IG.w(); r.q_wxyz[1] = -(double)s.q_IG.x(); r.q_wxyz[2] = -(double)s.q_IG.y(); r.q_wxyz[3] = -(double)s.q_IG.z();
    r.n_clones = (int)msckf.getNumCamStates();
    r.n_tracks_residualized = 0;
    traj.push_back(r);
    ++n_frames;
  }
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - wall0).count();
  if (!o.out.empty()) asl::write_trajectory(o.out, traj);
  int matched = 0;
  const double rmse = asl::position_rmse(traj, gt, &matched);
  std::printf("{\"frames\": %ld, \"imu_readings\": %ld, \"dtype\": \"%s\", \"position_rmse_m\": %.9g, \"gt_matched\": %d, "
              "\"wall_s\": %.6f, \"frames_per_s\": %.3f, \"final_clones\": %d}\n",
              n_frames, n_imu, o.dtype.c_str(), rmse, matched, wall, n_frames / wall, traj.empty() ? 0 : traj.back().n_clones);
  return 0;
}

int main(int argc, char** argv) {
  Options o;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto need = [&](const char* name) -> std::string {
      if (i + 1 >= argc) { std::fprintf(stderr, "%s needs a value\n", name); std::exit(2); }
      return argv[++i];
    };
    if (a == "--mav0") o.mav0 = need("--mav0");
    else if (a == "--out") o.out = need("--out");
    else if (a == "--dtype") o.dtype = need("--dtype");
    else if (a == "--max-frames") o.max_frames = std::stoi(need("--max-frames"));
    else if (a == "--prune-redundant") o.prune_redundant = std::stoi(need("--prune-redundant")) != 0;
    else if (a == "--state-id") o.state_id = need("--state-id");
    else if (a == "--device") o.device = std::stoi(need("--device"));
    else if (a == "--dry-run") o.dry_run = true;
    else { std::fprintf(stderr, "unknown argument %s\n", a.c_str()); return 2; }
  }
  if (o.mav0.empty()) { std::fprintf(stderr, "usage: asl_player --mav0 DIR [--dtype f32|f64] [--out traj.csv] [--max-frames N] "
                                              "[--prune-redundant 0|1] [--state-id imu|frame] [--device K] [--dry-run]\n"); return 2; }
  try {
    if (o.dtype == "f32") return run<float>(o);
    if (o.dtype == "f64") return run<double>(o);
    std::fprintf(stderr, "bad --dtype %s\n", o.dtype.c_str());
    return 2;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "asl_player: %s\n", e.what());
    return 1;
  }
}
