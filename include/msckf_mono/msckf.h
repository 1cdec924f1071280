// include/msckf_mono/msckf.h -- drop-in replacement of the reference's msckf_mono::MSCKF<_S>
// (/root/reference/include/msckf_mono/msckf.h:31-1512; "ref :N" below = line N of that file).
//
// Same namespace, class name, template parameter and public member functions.  All integer bookkeeping
// (feature tracks, clone ids, residualisation and pruning decisions) runs on the host exactly as in the
// reference; all floating-point work goes through the C-ABI of libmsckf_b200.so (include/msckf_b200.h)
// into hand-written sm_90a kernels, with the covariance, clone poses and IMU state device resident.
// There is no CPU fallback: a failed device call throws std::runtime_error.
//
// Call-order contract (same as the reference's drivers, src/ros_interface.cpp:92-116,
// datasets/asl_msckf.cpp:233-294): per image propagate()* -> augmentState -> update -> addFeatures ->
// marginalize -> [pruneRedundantStates] -> pruneEmptyStates.  marginalize() residualises the tracks queued
// by the preceding update()/finish() at the clone poses current at that time (the reference snapshots
// copies of the clones in update(); the two coincide unless a measurement update is inserted between
// update() and marginalize(), which this class rejects loudly).
#ifndef MSCKF_HPP_
#define MSCKF_HPP_

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <iostream>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

#include <msckf_b200.h>
#include <msckf_mono/types.h>

namespace msckf_mono {

template <typename _S> class MSCKFBatch;

// An image observation of a landmark whose position is known (a prior map, a surveyed marker, a relocalisation match; not in
// the reference): normalised image coordinates z of the landmark at p_L_G, seen from the image whose clone has id state_id.
struct landmarkObservation {
  int state_id;
  double z[2];
  double p_L_G[3];
};
// A map landmark with position uncertainty (not in the reference): its map position p_L_G and the lower triangle xx, yx, yy,
// zx, zy, zz of its 3 x 3 covariance.  mapObservation: normalised image coordinates z of landmark `landmark` (an index into
// the landmark list of the call) seen from the image whose clone has id state_id.
struct mapLandmark {
  double p_L_G[3];
  double Sigma[6];
};
struct mapObservation {
  int state_id;
  int landmark;
  double z[2];
};

template <typename _S>
class MSCKF {
  friend class MSCKFBatch<_S>;

 public:
  MSCKF_B200_ALIGNED_NEW
  MSCKF() {}
  ~MSCKF() { if (engine_) msckf_b200_destroy(engine_); }
  // The filter owns device memory: it moves (so that filters can live in containers and be returned by value) but does not
  // copy -- the reference's implicit copy duplicated a few KB of host state, here it would have to duplicate a device-resident
  // covariance behind the caller's back (use msckf_b200_copy_state on engine() for an explicit checkpoint).
  MSCKF(const MSCKF&) = delete;
  MSCKF& operator=(const MSCKF&) = delete;
  MSCKF(MSCKF&& o) noexcept { moveFrom(o); }
  MSCKF& operator=(MSCKF&& o) noexcept {
    if (this != &o) {
      if (engine_) msckf_b200_destroy(engine_);
      engine_ = nullptr;
      moveFrom(o);
    }
    return *this;
  }

  // Engine capacities (call before initialize; 0 = derive from MSCKFParams).
  void setEngineOptions(int device, int max_clones = 0, int max_tracks = 0, int max_obs = 0) {
    device_ = device; cap_clones_ = max_clones; cap_tracks_ = max_tracks; cap_obs_ = max_obs;
  }

  // ref :72-97
  void initialize(const Camera<_S>& camera, const noiseParams<_S>& noise_params, const MSCKFParams<_S>& msckf_params,
                  const imuState<_S>& imu_state) {
    camera_ = camera;
    noise_params_ = noise_params;
    msckf_params_ = msckf_params;
    imu_state_ = imu_state;
    imu_state_.p_I_G_null = imu_state_.p_I_G;
    imu_state_.v_I_G_null = imu_state_.v_I_G;
    imu_state_.q_IG_null = imu_state_.q_IG;
    last_feature_id_ = 0;
    feature_tracks_.clear(); tracked_feature_ids_.clear(); feature_tracks_to_residualize_.clear();
    tracks_to_remove_.clear(); cam_states_.clear(); pruned_states_.clear(); map_.clear();
    if (engine_) { msckf_b200_destroy(engine_); engine_ = nullptr; }
    msckf_b200_config cfg;
    cfg.dtype = sizeof(_S) == 4 ? MSCKF_B200_F32 : MSCKF_B200_F64;
    cfg.device = device_;
    const int lcap = std::min(std::max(msckf_params.max_track_length, 2), 98);  // chi-square table has 99 entries (ref :91)
    // initial sizes only: like the reference's std::vectors, the engine grows on demand (window, tracks, observations)
    cfg.max_clones = cap_clones_ > 0 ? cap_clones_ : std::min(std::max(msckf_params.max_cam_states + 8, 32), 104);
    cfg.max_tracks = cap_tracks_ > 0 ? cap_tracks_ : 512;
    cfg.max_obs = cap_obs_ > 0 ? cap_obs_ : cfg.max_tracks * std::min(lcap, 32);
    check(msckf_b200_create(&cfg, &engine_), "msckf_b200_create");
    _S cam[7] = {camera.q_CI.x(), camera.q_CI.y(), camera.q_CI.z(), camera.q_CI.w(), camera.p_C_I(0), camera.p_C_I(1), camera.p_C_I(2)};
    std::vector<_S> nz(2 + 144 + 225);
    nz[0] = noise_params.u_var_prime; nz[1] = noise_params.v_var_prime;
    for (int i = 0; i < 12; ++i) for (int j = 0; j < 12; ++j) nz[2 + 12 * i + j] = noise_params.Q_imu(i, j);
    for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) nz[146 + 15 * i + j] = noise_params.initial_imu_covar(i, j);
    _S pr[2] = {msckf_params.max_gn_cost_norm, msckf_params.translation_threshold};
    _S im[19];
    for (int i = 0; i < 3; ++i) {
      im[i] = imu_state.p_I_G(i); im[3 + i] = imu_state.v_I_G(i); im[6 + i] = imu_state.b_g(i);
      im[9 + i] = imu_state.b_a(i); im[12 + i] = imu_state.g(i);
    }
    im[15] = imu_state.q_IG.x(); im[16] = imu_state.q_IG.y(); im[17] = imu_state.q_IG.z(); im[18] = imu_state.q_IG.w();
    check(msckf_b200_initialize(engine_, cam, nz.data(), pr, im), "msckf_b200_initialize");
    state_dirty_ = false;
    imu_queue_.clear();
    epoch_ = 0; epoch_at_queue_ = 0;
  }

  // ref :101-145.  The reading is queued on the host; the queue is handed to the device in one call
  // (msckf_b200_propagate_n: one kernel launch for up to 16 readings, same arithmetic reading by reading) by whichever
  // member function next needs the device state -- augmentState() in the reference's ROS loop (src/ros_interface.cpp:92-108),
  // getImuState() in its ASL loop (datasets/asl_msckf.cpp:229-234, one reading per call there).
  void propagate(imuReading<_S>& measurement_) {
    const _S r[7] = {measurement_.omega(0), measurement_.omega(1), measurement_.omega(2), measurement_.a(0), measurement_.a(1),
                     measurement_.a(2), measurement_.dT};
    imu_queue_.insert(imu_queue_.end(), r, r + 7);
    state_dirty_ = true;
  }

  // ref :148-212
  void augmentState(const int& state_id, const _S& time) {
    check(msckf_b200_augment(eng()), "msckf_b200_augment");
    augmentAbsorb(state_id, time);
  }
  // host part of augmentState, after the device appended the clone
  void augmentAbsorb(const int& state_id, const _S& time) {
    map_.clear();
    camState<_S> cam_state;
    cam_state.last_correlated_id = -1;
    cam_state.time = time;
    cam_state.state_id = state_id;
    cam_states_.push_back(cam_state);  // pose filled lazily from the device (refreshState)
    state_dirty_ = true;
  }

  // ref :215-299
  void update(const aligned_vector<Vector2<_S>>& measurements, const std::vector<size_t>& feature_ids) {
    feature_tracks_to_residualize_.clear();
    tracks_to_remove_.clear();
    int id_iter = 0;
    for (auto feature_id : tracked_feature_ids_) {
      auto input_it = std::find(feature_ids.begin(), feature_ids.end(), feature_id);
      const bool is_valid = (input_it != feature_ids.end());
      auto track = feature_tracks_.begin() + id_iter;
      if (is_valid) {
        const size_t d = std::distance(feature_ids.begin(), input_it);
        track->observations.push_back(measurements[d]);
        auto cam_state_iter = cam_states_.end() - 1;
        cam_state_iter->tracked_feature_ids.push_back(feature_id);
        track->cam_state_indices.push_back(cam_state_iter->state_id);
      }
      if (!is_valid || (track->observations.size() >= (size_t)msckf_params_.max_track_length)) {
        featureTrackToResidualize<_S> ttr;
        removeTrackedFeature(feature_id, ttr.cam_state_indices);
        if (ttr.cam_state_indices.size() >= (size_t)msckf_params_.min_track_length) {
          ttr.feature_id = track->feature_id;
          ttr.observations = track->observations;
          ttr.initialized = track->initialized;
          if (track->initialized) ttr.p_f_G = track->p_f_G;
          feature_tracks_to_residualize_.push_back(ttr);
        }
        tracks_to_remove_.push_back(feature_id);
      }
      id_iter++;
    }
    for (auto feature_id : tracks_to_remove_) {
      auto track_iter = feature_tracks_.begin();
      while (track_iter != feature_tracks_.end()) {
        if (track_iter->feature_id == feature_id) {
          const size_t last_id = track_iter->cam_state_indices.back();
          for (size_t index : track_iter->cam_state_indices)
            for (auto& camstate : cam_states_)
              if (!camstate.tracked_feature_ids.size() && (size_t)camstate.state_id == index) camstate.last_correlated_id = (int)last_id;
          track_iter = feature_tracks_.erase(track_iter);
          break;
        } else
          track_iter++;
      }
      auto cid = std::find(tracked_feature_ids_.begin(), tracked_feature_ids_.end(), feature_id);
      if (cid != tracked_feature_ids_.end()) tracked_feature_ids_.erase(cid);
    }
    epoch_at_queue_ = epoch_;
  }

  // ref :302-332
  void addFeatures(const aligned_vector<Vector2<_S>>& features, const std::vector<size_t>& feature_ids) {
    for (size_t i = 0; i < features.size(); i++) {
      const size_t id = feature_ids[i];
      if (std::find(tracked_feature_ids_.begin(), tracked_feature_ids_.end(), id) == tracked_feature_ids_.end()) {
        featureTrack<_S> track;
        track.feature_id = feature_ids[i];
        track.observations.push_back(features[i]);
        auto cam_state_last = cam_states_.end() - 1;
        cam_state_last->tracked_feature_ids.push_back(feature_ids[i]);
        track.cam_state_indices.push_back(cam_state_last->state_id);
        feature_tracks_.push_back(track);
        tracked_feature_ids_.push_back(feature_ids[i]);
      } else {
        std::cout << "Error, added new feature that was already being tracked" << std::endl;
        return;
      }
    }
  }

  // ref :336-449.  Loop A, loop B, gating, compression and the Kalman update all run on the device.
  void marginalize() {
    marginalizeLaunch();
    marginalizeCollect();
  }

  // ref :453-682.  Phases (shared with MSCKFBatch): triangulate the uninitialised features seen by the redundant clones,
  // residualise the observations those clones made, delete the clones.
  void pruneRedundantStates() {
    if (!redundantPruneWanted()) return;
    refreshState();
    msckf_b200_tracks tr;
    msckf_b200_report rep = {};
    if (redundantTriangulatePrepare(tr, rep, true)) {
      check(msckf_b200_update(eng(), MSCKF_B200_TRIANGULATE, &tr, &rep), "msckf_b200_update(TRIANGULATE)");
      redundantTriangulateAbsorb();
    }
    if (redundantResidualizePrepare(tr, true)) {
      rep = msckf_b200_report();
      checkNumeric(msckf_b200_update(eng(), MSCKF_B200_RESIDUALIZE, &tr, &rep), "msckf_b200_update(RESIDUALIZE)");
      redundantResidualizeAbsorb(rep);
    }
    refreshState();
    std::vector<int> keep;
    if (redundantDeletePrepare(keep)) check(msckf_b200_prune(eng(), keep.data(), (int)keep.size()), "msckf_b200_prune");
  }

  // ref :685-761.  Phases (shared with MSCKFBatch): how many leading clones go, then (with the poses refreshed) the bookkeeping.
  void pruneEmptyStates() {
    const int ndel = emptyStatesToDelete();
    if (ndel <= 0) return;
    refreshState();
    std::vector<int> keep;
    emptyStatesDelete(ndel, keep);
    check(msckf_b200_prune(eng(), keep.data(), (int)keep.size()), "msckf_b200_prune");
  }

  // ref :765-807
  void finish() {
    finishQueue();
    marginalize();
  }
  // the queueing half of finish(): every remaining track joins the residualisation queue
  void finishQueue() {
    for (size_t i = 0; i < tracked_feature_ids_.size(); i++) {
      std::vector<size_t> camStateIndices;
      removeTrackedFeature(tracked_feature_ids_[i], camStateIndices);
      if (camStateIndices.size() >= (size_t)msckf_params_.min_track_length) {
        featureTrackToResidualize<_S> track;
        const featureTrack<_S>* src = &feature_tracks_[i];
        if (src->feature_id != tracked_feature_ids_[i])
          for (auto& ft : feature_tracks_)
            if (ft.feature_id == tracked_feature_ids_[i]) { src = &ft; break; }
        track.feature_id = src->feature_id;
        track.observations = src->observations;
        track.initialized = src->initialized;
        if (src->initialized) track.p_f_G = src->p_f_G;
        track.cam_state_indices = camStateIndices;
        feature_tracks_to_residualize_.push_back(track);
      }
      tracks_to_remove_.push_back(tracked_feature_ids_[i]);
    }
    epoch_at_queue_ = epoch_;
  }

  // ---- getters (ref :810-848), all by value like the reference
  inline size_t getNumCamStates() { return cam_states_.size(); }
  inline imuState<_S> getImuState() { refreshState(); return imu_state_; }
  inline aligned_vector<Vector3<_S>> getMap() { return map_; }
  inline Camera<_S> getCamera() { return camera_; }
  inline camState<_S> getCamState(size_t i) { refreshState(); return cam_states_[i]; }
  inline std::vector<camState<_S>> getCamStates() const { refreshState(); return cam_states_; }  // const like ref :835
  inline std::vector<camState<_S>> getPrunedStates() {
    std::sort(pruned_states_.begin(), pruned_states_.end(), [](const camState<_S>& a, const camState<_S>& b) { return a.state_id < b.state_id; });
    return pruned_states_;
  }

  // ---- extras (not in the reference): diagnostics used by the parity tests and the bench
  struct TrackReport { int cm_ok = 0, tri_ok = 0, valid = 0, accepted = 0, rows = 0; _S gamma = 0; Vector3<_S> p_f_G; };
  const std::vector<TrackReport>& lastReport() const { return last_report_; }
  int lastStackedRows() const { return last_m_; }
  int lastRank() const { return last_rank_; }
  const std::vector<size_t>& trackedFeatureIds() const { return tracked_feature_ids_; }
  const std::vector<featureTrackToResidualize<_S>>& tracksToResidualize() const { return feature_tracks_to_residualize_; }
  msckf_b200_engine* engine() { return eng(); }  // (queued IMU readings are handed over first)
  // full (15+6M)^2 covariance, row-major (the reference keeps it private in three blocks, ref :52-54)
  std::vector<_S> getCovariance() {
    const size_t n = 15 + 6 * cam_states_.size();
    std::vector<_S> P(n * n);
    check(msckf_b200_get_covariance(eng(), P.data()) < 0 ? -1 : 0, "msckf_b200_get_covariance");
    return P;
  }
  // consistency against ground truth: NEES = e^T P^-1 e of the orientation, position, IMU pose, IMU state and (with one truth
  // pose per clone, in window order) the whole state, computed on the device (msckf_b200_nees).  Queued IMU readings are
  // applied first, like the getters do; nothing of the filter changes.
  msckf_b200_nees_result nees(const imuState<double>& truth, const std::vector<camState<double>>* truth_cams = nullptr) {
    std::vector<double> im, poses;
    neesPack(truth, truth_cams, im, poses);
    msckf_b200_nees_result r;
    check(msckf_b200_nees(eng(), im.data(), truth_cams ? poses.data() : nullptr, &r), "msckf_b200_nees");
    return r;
  }
  // a truth in the C-ABI's layouts: imu 19 doubles (p, v, b_g, b_a, g, q_IG xyzw), poses 7 per clone (p_C_G, q_CG xyzw)
  void neesPack(const imuState<double>& truth, const std::vector<camState<double>>* truth_cams, std::vector<double>& im,
                std::vector<double>& poses) const {
    if (truth_cams && truth_cams->size() != cam_states_.size())
      throw std::invalid_argument("MSCKF::nees: one truth pose per clone of the window, in window order");
    im.assign(19, 0.0);
    for (int i = 0; i < 3; ++i) {
      im[i] = truth.p_I_G(i); im[3 + i] = truth.v_I_G(i); im[6 + i] = truth.b_g(i); im[9 + i] = truth.b_a(i); im[12 + i] = truth.g(i);
    }
    im[15] = truth.q_IG.x(); im[16] = truth.q_IG.y(); im[17] = truth.q_IG.z(); im[18] = truth.q_IG.w();
    poses.assign(7 * std::max<size_t>(truth_cams ? truth_cams->size() : 0, 1), 0.0);
    if (truth_cams)
      for (size_t k = 0; k < truth_cams->size(); ++k) {
        const camState<double>& c = (*truth_cams)[k];
        for (int i = 0; i < 3; ++i) poses[7 * k + i] = c.p_C_G(i);
        poses[7 * k + 3] = c.q_CG.x(); poses[7 * k + 4] = c.q_CG.y(); poses[7 * k + 5] = c.q_CG.z(); poses[7 * k + 6] = c.q_CG.w();
      }
  }
  // aided measurements (not in the reference): one EKF update of P and the state on the device (msckf_b200_aid_update) --
  // a position or pose fix, a zero-velocity update, a clone pose prior or a caller-linearised measurement.  Queued IMU
  // readings are applied first; the host mirror of the state is refreshed from the device on the next getter.  An applied
  // update between update() and marginalize() makes marginalize() refuse the queued tracks, as after a vision update.
  msckf_b200_aid_result aidedUpdate(const msckf_b200_aid& aid) {
    msckf_b200_aid_result r = {};
    checkNumeric(msckf_b200_aid_update(eng(), &aid, &r), "msckf_b200_aid_update");
    aidAbsorb(r);
    return r;
  }
  // VELOCITY with z = 0: the caller knows the platform stands still
  msckf_b200_aid_result zeroVelocityUpdate(const Matrix3<double>& R, double chi2_max = 0) {
    const double z[3] = {0.0, 0.0, 0.0};
    return aidedUpdate(aidModel(MSCKF_B200_AID_VELOCITY, 0, 3, z, R, chi2_max));
  }
  msckf_b200_aid_result positionUpdate(const Vector3<double>& p_I_G, const Matrix3<double>& R, double chi2_max = 0) {
    const double z[3] = {p_I_G(0), p_I_G(1), p_I_G(2)};
    return aidedUpdate(aidModel(MSCKF_B200_AID_POSITION, 0, 3, z, R, chi2_max));
  }
  // R: 6 x 6 over [dtheta, dp]
  msckf_b200_aid_result poseUpdate(const Vector3<double>& p_I_G, const Quaternion<double>& q_IG, const FixedMatrix<double, 6, 6>& R,
                                   double chi2_max = 0) {
    const double z[7] = {p_I_G(0), p_I_G(1), p_I_G(2), q_IG.x(), q_IG.y(), q_IG.z(), q_IG.w()};
    return aidedUpdate(aidModel(MSCKF_B200_AID_POSE, 0, 6, z, R, chi2_max));
  }
  // clone k of the window (window order)
  msckf_b200_aid_result clonePoseUpdate(size_t k, const Vector3<double>& p_C_G, const Quaternion<double>& q_CG,
                                        const FixedMatrix<double, 6, 6>& R, double chi2_max = 0) {
    const double z[7] = {p_C_G(0), p_C_G(1), p_C_G(2), q_CG.x(), q_CG.y(), q_CG.z(), q_CG.w()};
    return aidedUpdate(aidModel(MSCKF_B200_AID_CLONE_POSE, (int)k, 6, z, R, chi2_max));
  }
  // H: m x (15 + 6M) in the engine's error-state order, r: m, R: m x m (m <= 32)
  msckf_b200_aid_result linearUpdate(const MatrixX<double>& H, const VectorX<double>& r, const MatrixX<double>& R, double chi2_max = 0) {
    const int m = (int)H.rows(), n = (int)H.cols();
    if ((int)r.rows() != m || (int)R.rows() != m || (int)R.cols() != m) throw std::invalid_argument("MSCKF::linearUpdate: H, r and R differ in rows");
    std::vector<double> h((size_t)m * n), z(m);
    for (int i = 0; i < m; ++i) {
      z[i] = r(i);
      for (int j = 0; j < n; ++j) h[(size_t)i * n + j] = H(i, j);
    }
    msckf_b200_aid a = aidModel(MSCKF_B200_AID_LINEAR, 0, m, z.data(), R, chi2_max);
    a.n = n;
    a.H = h.data();
    return aidedUpdate(a);
  }
  // stacked aided updates (not in the reference; msckf_b200_aid_stack_update): up to 8 items -- odometry (BODY_VELOCITY,
  // RELATIVE_POSE), GNSS antenna positions and headings, radio ranges and rangefinder distances (at the IMU or at a clone) and the fixes above -- fused as ONE update with R block-diagonal across items, one NIS over all rows and one
  // chi2_max gate.  Items name clones by window position.  Bookkeeping as aidedUpdate(const msckf_b200_aid&).
  msckf_b200_aid_result aidedUpdate(const std::vector<msckf_b200_aid_item>& items, double chi2_max = 0) {
    msckf_b200_aid_result r = {};
    checkNumeric(msckf_b200_aid_stack_update(eng(), items.data(), (int)items.size(), chi2_max, &r), "msckf_b200_aid_stack_update");
    aidAbsorb(r);
    return r;
  }
  // the same stack with fault detection and exclusion over its items (msckf_b200_aid_stack_update_fde): degenerate items are
  // dropped, and up to fde.max_exclude items failing the block w-test are excluded before the rest is applied.  A thresholds
  // table or max_exclude the C-ABI would refuse throws std::invalid_argument.  Bookkeeping as aidedUpdate(items).
  msckf_b200_aid_fde_result aidedUpdate(const std::vector<msckf_b200_aid_item>& items, const msckf_b200_aid_fde& fde) {
    checkFde(fde);
    msckf_b200_aid_fde_result r = {};
    checkNumeric(msckf_b200_aid_stack_update_fde(eng(), items.data(), (int)items.size(), &fde, &r), "msckf_b200_aid_stack_update_fde");
    aidAbsorb(r.stack);
    return r;
  }
  static void checkFde(const msckf_b200_aid_fde& fde) {
    for (int d = 0; d < 32; ++d)
      if (!(std::isfinite(fde.chi2[d]) && fde.chi2[d] > 0.0)) throw std::invalid_argument("MSCKF::aidedUpdate: fde.chi2 must be finite and > 0");
    if (fde.max_exclude < 0 || fde.max_exclude > 7) throw std::invalid_argument("MSCKF::aidedUpdate: fde.max_exclude outside 0..7");
  }
  // the iterated stacks (msckf_b200_aid_stack_update_iter / _fde_iter): the stack relinearised about its own update, up to
  // iter.max_iter linearisations (0 or 1: the call above bit for bit), for the first range or GNSS epoch after drift; iter_out
  // receives the linearisations applied, whether the step converged to iter.tol, and the last step.  An iter the C-ABI would
  // refuse throws std::invalid_argument.  Bookkeeping as aidedUpdate(items).
  msckf_b200_aid_result aidedUpdate(const std::vector<msckf_b200_aid_item>& items, double chi2_max, const msckf_b200_aid_iter& iter,
                                    msckf_b200_aid_iter_result& iter_out) {
    checkIter(iter);
    msckf_b200_aid_result r = {};
    checkNumeric(msckf_b200_aid_stack_update_iter(eng(), items.data(), (int)items.size(), chi2_max, &iter, &r, &iter_out),
                 "msckf_b200_aid_stack_update_iter");
    aidAbsorb(r);
    return r;
  }
  msckf_b200_aid_fde_result aidedUpdate(const std::vector<msckf_b200_aid_item>& items, const msckf_b200_aid_fde& fde,
                                        const msckf_b200_aid_iter& iter, msckf_b200_aid_iter_result& iter_out) {
    checkFde(fde);
    checkIter(iter);
    msckf_b200_aid_fde_result r = {};
    checkNumeric(msckf_b200_aid_stack_update_fde_iter(eng(), items.data(), (int)items.size(), &fde, &iter, &r, &iter_out),
                 "msckf_b200_aid_stack_update_fde_iter");
    aidAbsorb(r.stack);
    return r;
  }
  static void checkIter(const msckf_b200_aid_iter& iter) {
    if (iter.max_iter < 0 || iter.max_iter > 16) throw std::invalid_argument("MSCKF::aidedUpdate: iter.max_iter outside 0..16");
    if (!(std::isfinite(iter.tol) && iter.tol >= 0.0)) throw std::invalid_argument("MSCKF::aidedUpdate: iter.tol must be finite and >= 0");
  }
  // v_I: the IMU's velocity in its own frame (wheel or leg odometry); mask bits 0..2 select the rows used, R is popcount(mask)
  // square over them.  mask 0b110 with v_I = 0 is the non-holonomic constraint v_y = v_z = 0.
  msckf_b200_aid_result bodyVelocityUpdate(const Vector3<double>& v_I, const MatrixX<double>& R, int mask = 7, double chi2_max = 0) {
    if (mask < 1 || mask > 7) throw std::invalid_argument("MSCKF::bodyVelocityUpdate: the mask must select rows 0..2");
    const double z[3] = {v_I(0), v_I(1), v_I(2)};
    const int m = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_BODY_VELOCITY, mask, 0, m, z, R)}, chi2_max);
  }
  // the pose of image state_id_b relative to image state_id_a in camera frames: p = C_a (p_C_G,b - p_C_G,a), q of C_b C_a^T;
  // R 6 x 6 over [dtheta, dp].  An id that is not in the window throws std::invalid_argument before any device call.
  msckf_b200_aid_result relativePoseUpdate(int state_id_a, int state_id_b, const Vector3<double>& p, const Quaternion<double>& q,
                                           const FixedMatrix<double, 6, 6>& R, double chi2_max = 0) {
    const int a = windowPosition(state_id_a, "MSCKF::relativePoseUpdate"), b = windowPosition(state_id_b, "MSCKF::relativePoseUpdate");
    const double z[7] = {p(0), p(1), p(2), q.x(), q.y(), q.z(), q.w()};
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_RELATIVE_POSE, a, b, 6, z, R)}, chi2_max);
  }
  // a GNSS antenna position p_A_G = p_I_G + C(q_IG)^T lever, the lever arm in the IMU frame; mask bits 0..2 select the rows
  // used (0b100 with a zero lever: an altitude, 0b011: a horizontal fix), R is popcount(mask) square over them
  msckf_b200_aid_result antennaPositionUpdate(const Vector3<double>& p_A_G, const Vector3<double>& lever, const MatrixX<double>& R,
                                              int mask = 7, double chi2_max = 0) {
    if (mask < 1 || mask > 7) throw std::invalid_argument("MSCKF::antennaPositionUpdate: the mask must select rows 0..2");
    const double z[6] = {p_A_G(0), p_A_G(1), p_A_G(2), lever(0), lever(1), lever(2)};
    const int m = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_ANTENNA_POSITION, mask, 0, m, z, R)}, chi2_max);
  }
  // the same at the clone of image state_id (a delayed fix: the image of the fix's epoch), the lever arm in that clone's camera
  // frame (l_C = C(q_CI) (l_I - p_C_I)).  An id that is not in the window throws std::invalid_argument before any device call.
  msckf_b200_aid_result cloneAntennaPositionUpdate(int state_id, const Vector3<double>& p_A_G, const Vector3<double>& lever,
                                                   const MatrixX<double>& R, int mask = 7, double chi2_max = 0) {
    const int k = windowPosition(state_id, "MSCKF::cloneAntennaPositionUpdate");
    if (mask < 1 || mask > 7) throw std::invalid_argument("MSCKF::cloneAntennaPositionUpdate: the mask must select rows 0..2");
    const double z[6] = {p_A_G(0), p_A_G(1), p_A_G(2), lever(0), lever(1), lever(2)};
    const int m = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_CLONE_ANTENNA_POSITION, k, mask, m, z, R)}, chi2_max);
  }
  // a heading psi (rad): the yaw atan2(d_y, d_x) in G of d = C(q_IG)^T axis, the axis in the IMU frame (a dual-antenna baseline,
  // a compass's forward axis); var is its variance.  An axis within ~1e-3 rad of vertical gives status 2 and changes nothing.
  msckf_b200_aid_result headingUpdate(double psi, const Vector3<double>& axis, double var, double chi2_max = 0) {
    const double z[4] = {psi, axis(0), axis(1), axis(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_HEADING, 0, 0, 1, z, R)}, chi2_max);
  }
  // the same at the clone of image state_id, the axis in that clone's camera frame (f_C = C(q_CI) f_I)
  msckf_b200_aid_result cloneHeadingUpdate(int state_id, double psi, const Vector3<double>& axis, double var, double chi2_max = 0) {
    const int k = windowPosition(state_id, "MSCKF::cloneHeadingUpdate");
    const double z[4] = {psi, axis(0), axis(1), axis(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_CLONE_HEADING, k, 0, 1, z, R)}, chi2_max);
  }
  // a radio range (UWB two-way ranging, an acoustic or radio beacon) |p_I_G + C(q_IG)^T lever - anchor| from an antenna on the
  // body, the lever arm in the IMU frame, to an anchor at a surveyed position in G; var is its variance.  An antenna within 1e-6 m
  // of its anchor gives status 2 and changes nothing.
  msckf_b200_aid_result rangeUpdate(double range, const Vector3<double>& anchor, const Vector3<double>& lever, double var,
                                    double chi2_max = 0) {
    const double z[7] = {range, anchor(0), anchor(1), anchor(2), lever(0), lever(1), lever(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_RANGE, 0, 0, 1, z, R)}, chi2_max);
  }
  // the same at the clone of image state_id (a delayed range: the image of its epoch), the lever arm in that clone's camera frame
  msckf_b200_aid_result cloneRangeUpdate(int state_id, double range, const Vector3<double>& anchor, const Vector3<double>& lever,
                                         double var, double chi2_max = 0) {
    const int k = windowPosition(state_id, "MSCKF::cloneRangeUpdate");
    const double z[7] = {range, anchor(0), anchor(1), anchor(2), lever(0), lever(1), lever(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_CLONE_RANGE, k, 0, 1, z, R)}, chi2_max);
  }
  // a rangefinder (laser, sonar) distance along the beam axis, from a sensor at lever (both in the IMU frame), to the level plane
  // {x : x_z = h} in G (the ground below, a ceiling above); var is its variance.  A beam within ~1e-3 rad of parallel to the
  // plane, or a plane behind the sensor, gives status 2 and changes nothing.
  msckf_b200_aid_result planeRangeUpdate(double range, double h, const Vector3<double>& lever, const Vector3<double>& axis, double var,
                                         double chi2_max = 0) {
    const double z[8] = {range, h, lever(0), lever(1), lever(2), axis(0), axis(1), axis(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_PLANE_RANGE, 0, 0, 1, z, R)}, chi2_max);
  }
  // the same at the clone of image state_id, the lever arm and the axis in that clone's camera frame
  msckf_b200_aid_result clonePlaneRangeUpdate(int state_id, double range, double h, const Vector3<double>& lever,
                                              const Vector3<double>& axis, double var, double chi2_max = 0) {
    const int k = windowPosition(state_id, "MSCKF::clonePlaneRangeUpdate");
    const double z[8] = {range, h, lever(0), lever(1), lever(2), axis(0), axis(1), axis(2)};
    MatrixX<double> R(1, 1);
    R(0, 0) = var;
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_CLONE_PLANE_RANGE, k, 0, 1, z, R)}, chi2_max);
  }
  // the at-rest items on their own (stacks of GYRO_AT_REST / ACCEL_AT_REST): the mean gyro reading, or the mean specific force,
  // of IMU readings taken at rest, R 3 x 3 (standstillUpdate forms both from the readings)
  msckf_b200_aid_result gyroAtRestUpdate(const Vector3<double>& omega_mean, const MatrixX<double>& R, double chi2_max = 0) {
    const double z[3] = {omega_mean(0), omega_mean(1), omega_mean(2)};
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_GYRO_AT_REST, 0, 0, 3, z, R)}, chi2_max);
  }
  msckf_b200_aid_result accelAtRestUpdate(const Vector3<double>& a_mean, const MatrixX<double>& R, double chi2_max = 0) {
    const double z[3] = {a_mean(0), a_mean(1), a_mean(2)};
    return aidedUpdate(std::vector<msckf_b200_aid_item>{aidItem(MSCKF_B200_AID_ACCEL_AT_REST, 0, 0, 3, z, R)}, chi2_max);
  }
  // standstill (not in the reference; msckf_b200_standstill_update: statistics, gate and outcomes there): the IMU readings
  // propagated since the previous image are tested for rest on their scatter about their mean and, at rest, fused as one
  // zero-velocity, gyro-bias and specific-force update.  The class only reports: on outcome 0 the caller skips the frame's
  // augmentState / update / marginalize / prune and keeps propagating (INTEGRATION.md).  Queued readings are handed over
  // first; readings or a cfg the C-ABI would refuse throw std::invalid_argument before any device call.  Bookkeeping as
  // aidedUpdate(items).
  msckf_b200_standstill_result standstillUpdate(const std::vector<imuReading<_S>>& readings, const msckf_b200_standstill& cfg) {
    std::vector<_S> r;
    packStandstill(readings, cfg, r, "MSCKF::standstillUpdate");
    msckf_b200_standstill_result o = {};
    checkNumeric(msckf_b200_standstill_update(eng(), r.data(), (int)readings.size(), &cfg, &o), "msckf_b200_standstill_update");
    aidAbsorb(o.stack);
    return o;
  }
  // readings in msckf_b200_propagate_n's layout, after the checks of msckf_b200_standstill_update (std::invalid_argument)
  static void packStandstill(const std::vector<imuReading<_S>>& readings, const msckf_b200_standstill& cfg, std::vector<_S>& r,
                             const std::string& what) {
    if (readings.size() < 2 || readings.size() > 4096) throw std::invalid_argument(what + ": 2 to 4096 readings");
    if (!(std::isfinite(cfg.noise_scale) && cfg.noise_scale >= 1.0)) throw std::invalid_argument(what + ": noise_scale must be finite and >= 1");
    if (!(std::isfinite(cfg.sigma_v) && cfg.sigma_v > 0.0)) throw std::invalid_argument(what + ": sigma_v must be finite and > 0");
    if (!(std::isfinite(cfg.scatter_max) && cfg.scatter_max > 0.0)) throw std::invalid_argument(what + ": scatter_max must be finite and > 0");
    if (!(std::isfinite(cfg.chi2_max) && cfg.chi2_max > 0.0)) throw std::invalid_argument(what + ": chi2_max must be finite and > 0");
    r.clear();
    for (const auto& m : readings) {
      const _S v[7] = {m.omega(0), m.omega(1), m.omega(2), m.a(0), m.a(1), m.a(2), m.dT};
      for (int i = 0; i < 7; ++i)
        if (!std::isfinite((double)v[i])) throw std::invalid_argument(what + ": non-finite reading");
      if (!(m.dT > 0)) throw std::invalid_argument(what + ": dT must be > 0");
      r.insert(r.end(), v, v + 7);
    }
  }
  // the window position of the clone of image state_id (std::invalid_argument when it is not in the window)
  int windowPosition(int state_id, const char* what) const {
    for (size_t pos = 0; pos < cam_states_.size(); ++pos)
      if (cam_states_[pos].state_id == state_id) return (int)pos;
    throw std::invalid_argument(std::string(what) + ": state_id " + std::to_string(state_id) + " is not in the window");
  }
  // host bookkeeping after an aided update: the mirror is stale, and an applied update moves the state the queued tracks saw
  void aidAbsorb(const msckf_b200_aid_result& r) {
    state_dirty_ = true;
    if (r.applied) epoch_++;
  }
  // mapped landmarks (not in the reference): one EKF update with image observations of landmarks whose position is known,
  // fused on the device (msckf_b200_landmark_update; model, gate and outcomes there).  R: 2 x 2 pixel noise in normalised
  // coordinates (NULL: diag(u_var', v_var')); chi2_obs > 0 gates every observation on its own.  gamma / flag (optional) receive
  // one entry per observation.  An observation of an image that is not in the window throws std::invalid_argument before any
  // device call.  Queued IMU readings are applied first, the host mirror is refreshed on the next getter, and an applied update
  // between update() and marginalize() makes marginalize() refuse the queued tracks, as after aidedUpdate().  max_iter >= 2
  // iterates the update (an iterated EKF: relinearise at the updated clone poses until max |delta_{i+1} - delta_i| <= tol, at
  // most max_iter linearisations), for relocalisation after drift; the default is the single linearisation.
  msckf_b200_landmark_result landmarkUpdate(const std::vector<landmarkObservation>& obs, const FixedMatrix<double, 2, 2>* R = nullptr,
                                            double chi2_obs = 0, std::vector<double>* gamma = nullptr, std::vector<int>* flag = nullptr,
                                            int max_iter = 1, double tol = 1e-10) {
    msckf_b200_landmarks lm{};
    landmarkPack(obs, R, chi2_obs, gamma, flag, lm);
    lm.max_iter = max_iter; lm.tol = tol;
    msckf_b200_landmark_result r = {};
    checkNumeric(msckf_b200_landmark_update(eng(), &lm, &r), "msckf_b200_landmark_update");
    landmarkAbsorb(r);
    return r;
  }
  // mapped landmarks with map uncertainty (not in the reference; msckf_b200_map_landmark_update: model, gate, caps there): each
  // landmark's position error, N(0, Sigma), is marginalised over all its observations in the call.  An observation of an
  // image that is not in the window, or of a landmark outside `landmarks`, throws std::invalid_argument before any device
  // call; otherwise as the landmarkUpdate above.
  msckf_b200_landmark_result landmarkUpdate(const std::vector<mapObservation>& obs, const std::vector<mapLandmark>& landmarks,
                                            const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                            std::vector<double>* gamma = nullptr, std::vector<int>* flag = nullptr, int max_iter = 1,
                                            double tol = 1e-10) {
    msckf_b200_landmarks lm{};
    msckf_b200_landmark_map map{};
    mapPack(obs, landmarks, R, chi2_obs, gamma, flag, lm, map);
    lm.max_iter = max_iter; lm.tol = tol;
    msckf_b200_landmark_result r = {};
    checkNumeric(msckf_b200_map_landmark_update(eng(), &lm, &map, &r), "msckf_b200_map_landmark_update");
    landmarkAbsorb(r);
    return r;
  }
  // the same updates with a consensus on the matches (msckf_b200_landmark_update_consensus: model, sampling, selection and flag 3
  // there): the outliers of the best 4-dof correction are excluded before the update; cons_out receives the consensus result.
  // An invalid consensus (hypotheses outside 0 .. 1024, or with hypotheses > 0 a thresh that is not finite and > 0 or
  // min_inliers < 2) throws std::invalid_argument before any device call; otherwise as the landmarkUpdate forms above.
  msckf_b200_landmark_result landmarkUpdate(const std::vector<landmarkObservation>& obs, const msckf_b200_landmark_consensus& cons,
                                            msckf_b200_landmark_consensus_result& cons_out, const FixedMatrix<double, 2, 2>* R = nullptr,
                                            double chi2_obs = 0, std::vector<double>* gamma = nullptr, std::vector<int>* flag = nullptr,
                                            int max_iter = 1, double tol = 1e-10) {
    checkConsensus(cons);
    msckf_b200_landmarks lm{};
    landmarkPack(obs, R, chi2_obs, gamma, flag, lm);
    lm.max_iter = max_iter; lm.tol = tol;
    msckf_b200_landmark_result r = {};
    checkNumeric(msckf_b200_landmark_update_consensus(eng(), &lm, nullptr, &cons, &r, &cons_out), "msckf_b200_landmark_update_consensus");
    landmarkAbsorb(r);
    return r;
  }
  msckf_b200_landmark_result landmarkUpdate(const std::vector<mapObservation>& obs, const std::vector<mapLandmark>& landmarks,
                                            const msckf_b200_landmark_consensus& cons, msckf_b200_landmark_consensus_result& cons_out,
                                            const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                            std::vector<double>* gamma = nullptr, std::vector<int>* flag = nullptr, int max_iter = 1,
                                            double tol = 1e-10) {
    checkConsensus(cons);
    msckf_b200_landmarks lm{};
    msckf_b200_landmark_map map{};
    mapPack(obs, landmarks, R, chi2_obs, gamma, flag, lm, map);
    lm.max_iter = max_iter; lm.tol = tol;
    msckf_b200_landmark_result r = {};
    checkNumeric(msckf_b200_landmark_update_consensus(eng(), &lm, &map, &cons, &r, &cons_out), "msckf_b200_landmark_update_consensus");
    landmarkAbsorb(r);
    return r;
  }
  // the consensus settings the C-ABI accepts
  static void checkConsensus(const msckf_b200_landmark_consensus& c) {
    if (c.hypotheses < 0 || c.hypotheses > 1024) throw std::invalid_argument("landmarkUpdate: hypotheses outside 0 .. 1024");
    if (c.hypotheses > 0 && !(std::isfinite(c.thresh) && c.thresh > 0.0))
      throw std::invalid_argument("landmarkUpdate: consensus thresh is not finite and > 0");
    if (c.hypotheses > 0 && c.min_inliers < 2) throw std::invalid_argument("landmarkUpdate: consensus min_inliers < 2");
  }
  // landmarkPack of the observations' map positions, and the map (landmark ids, Sigma) in this object's buffers
  void mapPack(const std::vector<mapObservation>& obs, const std::vector<mapLandmark>& landmarks, const FixedMatrix<double, 2, 2>* R,
               double chi2_obs, std::vector<double>* gamma, std::vector<int>* flag, msckf_b200_landmarks& lm,
               msckf_b200_landmark_map& map) {
    std::vector<landmarkObservation> o(obs.size());
    lmk_id_.resize(obs.size());
    for (size_t i = 0; i < obs.size(); ++i) {
      if (obs[i].landmark < 0 || obs[i].landmark >= (int)landmarks.size())
        throw std::invalid_argument("MSCKF::landmarkUpdate: landmark " + std::to_string(obs[i].landmark) + " is not in the map");
      o[i].state_id = obs[i].state_id;
      o[i].z[0] = obs[i].z[0]; o[i].z[1] = obs[i].z[1];
      for (int c = 0; c < 3; ++c) o[i].p_L_G[c] = landmarks[obs[i].landmark].p_L_G[c];
      lmk_id_[i] = obs[i].landmark;
    }
    landmarkPack(o, R, chi2_obs, gamma, flag, lm);
    lmk_sig_.resize(6 * landmarks.size());
    for (size_t l = 0; l < landmarks.size(); ++l)
      for (int c = 0; c < 6; ++c) lmk_sig_[6 * l + c] = landmarks[l].Sigma[c];
    map.landmark = lmk_id_.data(); map.Sigma_L = lmk_sig_.data(); map.n_landmarks = (int)landmarks.size();
  }
  // a msckf_b200_landmarks of obs with window positions from the clone list (pointers into this object's buffers)
  void landmarkPack(const std::vector<landmarkObservation>& obs, const FixedMatrix<double, 2, 2>* R, double chi2_obs,
                    std::vector<double>* gamma, std::vector<int>* flag, msckf_b200_landmarks& lm) {
    const size_t n = obs.size();
    lmk_clone_.resize(n); lmk_z_.resize(2 * n); lmk_p_.resize(3 * n);
    for (size_t i = 0; i < n; ++i) {
      size_t pos = 0;
      while (pos < cam_states_.size() && cam_states_[pos].state_id != obs[i].state_id) ++pos;
      if (pos == cam_states_.size())
        throw std::invalid_argument("MSCKF::landmarkUpdate: state_id " + std::to_string(obs[i].state_id) + " is not in the window");
      lmk_clone_[i] = (int)pos;
      lmk_z_[2 * i] = obs[i].z[0]; lmk_z_[2 * i + 1] = obs[i].z[1];
      for (int c = 0; c < 3; ++c) lmk_p_[3 * i + c] = obs[i].p_L_G[c];
    }
    if (R) { lmk_R_[0] = (*R)(0, 0); lmk_R_[1] = (*R)(1, 0); lmk_R_[2] = (*R)(1, 1); }
    if (gamma) gamma->assign(n, 0.0);
    if (flag) flag->assign(n, 0);
    lm.n_obs = (int)n; lm.clone = lmk_clone_.data(); lm.z = lmk_z_.data(); lm.p_L_G = lmk_p_.data();
    lm.R = R ? lmk_R_ : nullptr; lm.chi2_obs = chi2_obs;
    lm.gamma = gamma ? gamma->data() : nullptr; lm.flag = flag ? flag->data() : nullptr;
  }
  // host bookkeeping after a landmark update (the same as after an aided update)
  void landmarkAbsorb(const msckf_b200_landmark_result& r) {
    state_dirty_ = true;
    if (r.applied) epoch_++;
  }
  // marginalize() = launch + collect (kept separate for pipelining and for batches of filters, MSCKFBatch below).
  void marginalizeLaunch() {
    msckf_b200_tracks tr;
    if (!marginalizePrepare(tr, true)) return;
    check(msckf_b200_update_async(eng(), MSCKF_B200_MARGINALIZE, &tr), "msckf_b200_update_async");
    launch_pending_ = true;
  }
  void marginalizeCollect() {
    if (!launch_pending_) return;
    launch_pending_ = false;
    msckf_b200_report rep;
    marginalizeReport(rep);
    checkNumeric(msckf_b200_fetch(engine_, &rep), "msckf_b200_fetch");
    marginalizeAbsorb(rep);
  }
  // pieces of marginalize() for a caller that runs the device part of several filters as one batch (MSCKFBatch):
  // Prepare packs the queued tracks (false: nothing queued), Report points a report at this filter's buffers, Absorb
  // folds the fetched report back into the host bookkeeping (ref :368-372).
  bool marginalizePrepare(msckf_b200_tracks& tr, bool in_engine_buffer) {
    last_report_.clear();
    launch_pending_ = false;
    if (feature_tracks_to_residualize_.empty()) return false;
    if (epoch_at_queue_ != epoch_)
      throw std::logic_error("msckf_mono::MSCKF::marginalize: a measurement update was applied between update()/finish() and "
                             "marginalize(); the queued tracks' clone snapshots (ref :250) would differ from the device state");
    packTracks(feature_tracks_to_residualize_, nullptr, tr, in_engine_buffer);
    return true;
  }
  void marginalizeReport(msckf_b200_report& rep) {
    const int N = (int)feature_tracks_to_residualize_.size();
    rp_cm_.resize(N); rp_tri_.resize(N); rp_valid_.resize(N); rp_acc_.resize(N); rp_gamma_.resize(N); rp_pfg_.resize(3 * (size_t)N);
    rep.cm_ok = rp_cm_.data(); rep.tri_ok = rp_tri_.data(); rep.valid = rp_valid_.data(); rep.accepted = rp_acc_.data();
    rep.gamma = rp_gamma_.data(); rep.p_f_G = rp_pfg_.data(); rep.m = 0; rep.rank = 0;
  }
  void marginalizeAbsorb(const msckf_b200_report& rep) {
    const int N = (int)feature_tracks_to_residualize_.size();
    last_report_.resize(N);
    for (int t = 0; t < N; ++t) {
      auto& track = feature_tracks_to_residualize_[t];
      TrackReport& r = last_report_[t];
      r.cm_ok = rp_cm_[t]; r.tri_ok = rp_tri_[t]; r.valid = rp_valid_[t]; r.accepted = rp_acc_[t]; r.gamma = rp_gamma_[t];
      for (int k = 0; k < 3; ++k) r.p_f_G(k) = rp_pfg_[3 * (size_t)t + k];
      r.rows = r.accepted ? (2 * (int)track.observations.size() - 3) : 0;
      if (r.valid) { track.initialized = true; track.p_f_G = r.p_f_G; map_.push_back(r.p_f_G); }  // ref :368-372
    }
    last_m_ = rep.m; last_rank_ = rep.rank;
    if (rep.m > 0) epoch_++;
    state_dirty_ = true;
  }
  // pieces of pruneRedundantStates() (ref :453-682).  The clone poses must be current (refreshState) before the first
  // Prepare and before DeletePrepare.  A Prepare returning false has nothing for the device.
  bool redundantPruneWanted() const { return cam_states_.size() >= 20; }
  // ref :464-534, first loop: drop single observations, queue the uninitialised features for checkMotion + initializePosition
  bool redundantTriangulatePrepare(msckf_b200_tracks& tr, msckf_b200_report& rep, bool in_engine_buffer) {
    rm_cam_state_ids_.clear();
    tri_feat_.clear(); tri_involved_.clear(); tri_batch_.clear();
    findRedundantCamStates(rm_cam_state_ids_);
    const auto& rm_cam_state_ids = rm_cam_state_ids_;
    for (size_t fi = 0; fi < feature_tracks_.size(); ++fi) {
      auto& feature = feature_tracks_[fi];
      std::vector<size_t> involved;
      size_t obs_id = 0;
      for (const auto& cam_id : rm_cam_state_ids) {
        auto it = std::find(feature.cam_state_indices.begin(), feature.cam_state_indices.end(), cam_id);
        if (it != feature.cam_state_indices.end()) { involved.push_back(cam_id); obs_id = std::distance(feature.cam_state_indices.begin(), it); }
      }
      if (involved.size() == 0) continue;
      if (involved.size() == 1) {
        feature.observations.erase(feature.observations.begin() + obs_id);
        feature.cam_state_indices.erase(feature.cam_state_indices.begin() + obs_id);
        continue;
      }
      if (!feature.initialized) {
        featureTrackToResidualize<_S> q;
        q.feature_id = feature.feature_id;
        q.observations = feature.observations;
        for (size_t pos = 0; pos < cam_states_.size(); ++pos)
          if (std::find(feature.cam_state_indices.begin(), feature.cam_state_indices.end(), (size_t)cam_states_[pos].state_id) !=
              feature.cam_state_indices.end())
            q.cam_state_indices.push_back(pos);
        if (q.cam_state_indices.size() != q.observations.size())
          throw std::logic_error("pruneRedundantStates: observations and associated clones differ in number");
        tri_feat_.push_back(fi);
        tri_involved_.push_back(involved);
        tri_batch_.push_back(q);
      }
    }
    if (tri_batch_.empty()) return false;
    packTracks(tri_batch_, nullptr, tr, in_engine_buffer);
    const int N = (int)tri_batch_.size();
    rp_cm_.resize(N); rp_tri_.resize(N); rp_pfg_.resize(3 * (size_t)N);
    rep = msckf_b200_report();
    rep.cm_ok = rp_cm_.data(); rep.tri_ok = rp_tri_.data(); rep.p_f_G = rp_pfg_.data();
    return true;
  }
  void redundantTriangulateAbsorb() {
    for (size_t k = 0; k < tri_batch_.size(); ++k) {
      auto& feature = feature_tracks_[tri_feat_[k]];
      // checkMotion on fewer than two clones is false (ref :982-984)
      const bool cm = tri_batch_[k].cam_state_indices.size() >= 2 && rp_cm_[k];
      if (!cm || !rp_tri_[k]) {
        for (const auto& cam_id : tri_involved_[k]) {
          auto it = std::find(feature.cam_state_indices.begin(), feature.cam_state_indices.end(), cam_id);
          if (it != feature.cam_state_indices.end()) {
            const size_t oi = std::distance(feature.cam_state_indices.begin(), it);
            feature.cam_state_indices.erase(it);
            feature.observations.erase(feature.observations.begin() + oi);
          }
        }
      } else {
        feature.initialized = true;
        for (int c = 0; c < 3; ++c) feature.p_f_G(c) = rp_pfg_[3 * k + c];
        map_.push_back(feature.p_f_G);
      }
    }
  }
  // ref :545-607, second loop: residualise the observations of the redundant clones
  bool redundantResidualizePrepare(msckf_b200_tracks& tr, bool in_engine_buffer) {
    const auto& rm_cam_state_ids = rm_cam_state_ids_;
    res_batch_.clear();
    for (auto& feature : feature_tracks_) {
      std::vector<size_t> involved;
      aligned_vector<Vector2<_S>> involved_obs;
      for (const auto& cam_id : rm_cam_state_ids) {
        auto it = std::find(feature.cam_state_indices.begin(), feature.cam_state_indices.end(), cam_id);
        if (it != feature.cam_state_indices.end()) {
          involved.push_back(cam_id);
          involved_obs.push_back(feature.observations[std::distance(feature.cam_state_indices.begin(), it)]);
        }
      }
      if (involved.size() == 0) continue;
      featureTrackToResidualize<_S> q;
      q.feature_id = feature.feature_id;
      q.observations = involved_obs;
      for (size_t pos = 0; pos < cam_states_.size(); ++pos)
        if (std::find(involved.begin(), involved.end(), (size_t)cam_states_[pos].state_id) != involved.end()) q.cam_state_indices.push_back(pos);
      q.initialized = true;
      q.p_f_G = feature.p_f_G;
      if (q.cam_state_indices.size() != q.observations.size())
        throw std::logic_error("pruneRedundantStates: involved observations and clones differ in number");
      res_batch_.push_back(q);
      for (const auto& cam_id : involved) {
        auto it = std::find(feature.cam_state_indices.begin(), feature.cam_state_indices.end(), cam_id);
        if (it != feature.cam_state_indices.end()) {
          const size_t oi = std::distance(feature.cam_state_indices.begin(), it);
          feature.cam_state_indices.erase(it);
          feature.observations.erase(feature.observations.begin() + oi);
        }
      }
    }
    if (res_batch_.empty()) return false;
    packTracks(res_batch_, &res_batch_, tr, in_engine_buffer);
    return true;
  }
  void redundantResidualizeAbsorb(const msckf_b200_report& rep) {
    if (rep.m > 0) epoch_++;
    state_dirty_ = true;
  }
  // ref :616-681: the bookkeeping of deleting the redundant clones; keep = surviving positions (false: none is deleted)
  bool redundantDeletePrepare(std::vector<int>& keep) {
    keep.clear();
    std::vector<camState<_S>> kept;
    for (size_t pos = 0; pos < cam_states_.size(); ++pos) {
      if (std::find(rm_cam_state_ids_.begin(), rm_cam_state_ids_.end(), (size_t)cam_states_[pos].state_id) != rm_cam_state_ids_.end())
        pruned_states_.push_back(cam_states_[pos]);
      else { keep.push_back((int)pos); kept.push_back(cam_states_[pos]); }
    }
    if (keep.size() == cam_states_.size()) return false;
    cam_states_.swap(kept);
    return true;
  }
  // pieces of pruneEmptyStates() (ref :685-761): the number of leading clones to delete (<= 0: none), and the bookkeeping
  // of deleting them (the poses must be current), which gives the positions that survive
  int emptyStatesToDelete() const {
    const int max_states = msckf_params_.max_cam_states;
    if ((int)cam_states_.size() < max_states) return 0;
    const int num_cam_states = (int)cam_states_.size();
    int last_to_remove = num_cam_states - max_states - 1;
    if (cam_states_.front().tracked_feature_ids.size()) return 0;
    for (int i = 1; i < num_cam_states - max_states; i++)
      if (cam_states_[i].tracked_feature_ids.size()) { last_to_remove = i - 1; break; }
    return last_to_remove + 1;
  }
  void emptyStatesDelete(int ndel, std::vector<int>& keep) {
    const int num_cam_states = (int)cam_states_.size();
    for (int i = 0; i < ndel; ++i) pruned_states_.push_back(cam_states_[i]);
    cam_states_.erase(cam_states_.begin(), cam_states_.begin() + ndel);
    keep.clear();
    for (int i = ndel; i < num_cam_states; ++i) keep.push_back(i);
  }

 private:
  Camera<_S> camera_;
  noiseParams<_S> noise_params_;
  MSCKFParams<_S> msckf_params_;
  std::vector<featureTrack<_S>> feature_tracks_;
  std::vector<size_t> tracked_feature_ids_;
  std::vector<featureTrackToResidualize<_S>> feature_tracks_to_residualize_;
  std::vector<size_t> tracks_to_remove_;
  size_t last_feature_id_ = 0;
  mutable imuState<_S> imu_state_;             // host mirror of the device state (refreshState)
  mutable std::vector<camState<_S>> cam_states_;  // bookkeeping on host; poses mirrored from the device
  std::vector<camState<_S>> pruned_states_;
  aligned_vector<Vector3<_S>> map_;
  msckf_b200_engine* engine_ = nullptr;
  int device_ = 0, cap_clones_ = 0, cap_tracks_ = 0, cap_obs_ = 0;
  mutable bool state_dirty_ = false;
  bool launch_pending_ = false;
  mutable std::vector<_S> imu_queue_;  // IMU readings not yet handed to the device (7 scalars each)
  unsigned long long epoch_ = 0, epoch_at_queue_ = 0;
  std::vector<TrackReport> last_report_;
  int last_m_ = 0, last_rank_ = 0;
  std::vector<int> pk_off_, pk_idx_, rp_cm_, rp_tri_, rp_valid_, rp_acc_;
  std::vector<_S> pk_obs_, pk_pfg_, rp_gamma_, rp_pfg_;
  // pruneRedundantStates() between its phases
  std::vector<size_t> rm_cam_state_ids_, tri_feat_;
  std::vector<std::vector<size_t>> tri_involved_;
  std::vector<featureTrackToResidualize<_S>> tri_batch_, res_batch_;
  std::vector<double> aid_R_;  // R of the last convenience-form aided update, row-major
  std::vector<int> lmk_clone_;  // the last landmark update's observations in the C-ABI's layout (landmarkPack)
  std::vector<int> lmk_id_;       // ... and the landmark of each, with every landmark's Sigma (mapPack)
  std::vector<double> lmk_sig_;
  std::vector<double> lmk_z_, lmk_p_;
  double lmk_R_[3] = {0.0, 0.0, 0.0};

  // a msckf_b200_aid of one of the convenience forms (z must outlive the call; R is copied row-major into aid_R_)
  template <class Mat>
  msckf_b200_aid aidModel(int model, int clone, int m, const double* z, const Mat& R, double chi2_max) {
    if ((int)R.rows() != m || (int)R.cols() != m) throw std::invalid_argument("MSCKF: aided update R has the wrong shape");
    aid_R_.resize((size_t)m * m);
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < m; ++j) aid_R_[(size_t)i * m + j] = R(i, j);
    msckf_b200_aid a = {};
    a.model = model; a.clone = clone; a.m = m; a.n = 0;
    a.z = z; a.H = nullptr; a.R = aid_R_.data(); a.chi2_max = chi2_max;
    return a;
  }
  // a msckf_b200_aid_item of one of the single-item forms (z must outlive the call; R is copied into aid_R_ as by aidModel)
  template <class Mat>
  msckf_b200_aid_item aidItem(int model, int a, int b, int m, const double* z, const Mat& R) {
    const msckf_b200_aid q = aidModel(model, 0, m, z, R, 0.0);
    msckf_b200_aid_item it = {};
    it.model = model; it.a = a; it.b = b; it.z = z; it.R = q.R;
    return it;
  }

  static void check(int rc, const char* what) {
    if (rc != 0) throw std::runtime_error(std::string(what) + " failed (" + std::to_string(rc) + "): " + msckf_b200_last_error());
  }
  // a non-finite update is not an error in the reference: its only anomaly handling is a print (ref :1405-1409)
  static void checkNumeric(int rc, const char* what) {
    if (rc == MSCKF_B200_ERR_NUMERIC) { std::cout << "[msckf_b200] " << what << ": " << msckf_b200_last_error() << std::endl; return; }
    check(rc, what);
  }
  void moveFrom(MSCKF& o) {
    camera_ = o.camera_; noise_params_ = o.noise_params_; msckf_params_ = o.msckf_params_;
    feature_tracks_ = std::move(o.feature_tracks_); tracked_feature_ids_ = std::move(o.tracked_feature_ids_);
    feature_tracks_to_residualize_ = std::move(o.feature_tracks_to_residualize_); tracks_to_remove_ = std::move(o.tracks_to_remove_);
    last_feature_id_ = o.last_feature_id_; imu_state_ = o.imu_state_; cam_states_ = std::move(o.cam_states_);
    pruned_states_ = std::move(o.pruned_states_); map_ = std::move(o.map_);
    engine_ = o.engine_; o.engine_ = nullptr;
    device_ = o.device_; cap_clones_ = o.cap_clones_; cap_tracks_ = o.cap_tracks_; cap_obs_ = o.cap_obs_;
    state_dirty_ = o.state_dirty_; launch_pending_ = o.launch_pending_; imu_queue_ = std::move(o.imu_queue_);
    epoch_ = o.epoch_; epoch_at_queue_ = o.epoch_at_queue_; last_report_ = std::move(o.last_report_);
    last_m_ = o.last_m_; last_rank_ = o.last_rank_;
  }
  // the engine handle for a call that needs the device state: queued IMU readings are applied first
  msckf_b200_engine* eng() const {
    if (!imu_queue_.empty()) {
      const int k = (int)(imu_queue_.size() / 7);
      const int rc = msckf_b200_propagate_n(engine_, imu_queue_.data(), k);
      imu_queue_.clear();
      check(rc, "msckf_b200_propagate_n");
    }
    return engine_;
  }

  // Flat SoA form of a track batch.  in_engine_buffer: packed straight into the engine's pinned input block
  // (msckf_b200_input_buffer: no second copy on the way to the device); otherwise into this object's own vectors.
  // with_pfg: the tracks' positions ride along (RESIDUALIZE).
  void packTracks(const std::vector<featureTrackToResidualize<_S>>& tracks, const std::vector<featureTrackToResidualize<_S>>* with_pfg,
                  msckf_b200_tracks& tr, bool in_engine_buffer = true) {
    const size_t N = tracks.size();
    size_t tot = 0;
    for (size_t t = 0; t < N; ++t) tot += tracks[t].observations.size();
    int* off; int* idx; _S* obs; _S* pfg = nullptr;
    if (in_engine_buffer) {
      check(msckf_b200_input_buffer(eng(), (int)N, (int)tot, &tr), "msckf_b200_input_buffer");
      off = const_cast<int*>(tr.obs_offset); idx = const_cast<int*>(tr.clone_index);
      obs = static_cast<_S*>(const_cast<void*>(tr.obs)); pfg = static_cast<_S*>(const_cast<void*>(tr.p_f_G));
    } else {
      pk_off_.resize(N + 1); pk_obs_.resize(2 * tot); pk_idx_.resize(tot); pk_pfg_.resize(3 * N);
      off = pk_off_.data(); idx = pk_idx_.data(); obs = pk_obs_.data(); pfg = pk_pfg_.data();
      tr.n_tracks = (int)N; tr.obs_offset = off; tr.obs = obs; tr.clone_index = idx; tr.p_f_G = pfg;
    }
    if (!with_pfg) tr.p_f_G = nullptr;
    tot = 0;
    for (size_t t = 0; t < N; ++t) { off[t] = (int)tot; tot += tracks[t].observations.size(); }
    off[N] = (int)tot;
    for (size_t t = 0; t < N; ++t) {
      const auto& trk = tracks[t];
      if (trk.cam_state_indices.size() != trk.observations.size())
        throw std::logic_error("track observations and clone indices differ in number");
      // the reference clears the queue in update() only (:218): finish() after a marginalize() would re-residualise the
      // last update's tracks with their old positional indices (undefined behaviour there once clones were pruned)
      for (size_t ci : trk.cam_state_indices)
        if (ci >= cam_states_.size()) throw std::logic_error("stale residualisation queue: clone index out of range (reference: undefined behaviour)");
      for (size_t i = 0; i < trk.observations.size(); ++i) {
        obs[2 * (off[t] + i)] = trk.observations[i](0);
        obs[2 * (off[t] + i) + 1] = trk.observations[i](1);
        idx[off[t] + i] = (int)trk.cam_state_indices[i];
      }
      if (with_pfg) for (int c = 0; c < 3; ++c) pfg[3 * t + c] = (*with_pfg)[t].p_f_G(c);
    }
  }

  // pull the IMU state and clone poses back from the device when something changed them
  void refreshState() const {
    if (!state_dirty_ || !engine_) return;
    _S im[29];
    std::vector<_S> poses(7 * std::max<size_t>(cam_states_.size(), 1));
    check(msckf_b200_get_state(eng(), im, poses.data()), "msckf_b200_get_state");
    refreshAbsorb(im, poses.data());
  }
  // the host mirror from msckf_b200_get_state's layouts (imu: 29 scalars, poses: 7 per clone)
  void refreshAbsorb(const _S* im, const _S* poses) const {
    for (int i = 0; i < 3; ++i) {
      imu_state_.p_I_G(i) = im[i]; imu_state_.v_I_G(i) = im[3 + i]; imu_state_.b_g(i) = im[6 + i]; imu_state_.b_a(i) = im[9 + i];
      imu_state_.g(i) = im[12 + i]; imu_state_.p_I_G_null(i) = im[19 + i]; imu_state_.v_I_G_null(i) = im[22 + i];
    }
    imu_state_.q_IG = Quaternion<_S>(im[18], im[15], im[16], im[17]);
    imu_state_.q_IG_null = Quaternion<_S>(im[28], im[25], im[26], im[27]);
    for (size_t k = 0; k < cam_states_.size(); ++k) {
      for (int i = 0; i < 3; ++i) cam_states_[k].p_C_G(i) = poses[7 * k + i];
      cam_states_[k].q_CG = Quaternion<_S>(poses[7 * k + 6], poses[7 * k + 3], poses[7 * k + 4], poses[7 * k + 5]);
    }
    state_dirty_ = false;
  }

  // ref :1469-1485 (positions only: the clone copies are the device-resident poses)
  void removeTrackedFeature(const size_t featureID, std::vector<size_t>& camStateIndices) {
    camStateIndices.clear();
    for (size_t c_i = 0; c_i < cam_states_.size(); c_i++) {
      auto it = std::find(cam_states_[c_i].tracked_feature_ids.begin(), cam_states_[c_i].tracked_feature_ids.end(), featureID);
      if (it != cam_states_[c_i].tracked_feature_ids.end()) {
        cam_states_[c_i].tracked_feature_ids.erase(it);
        camStateIndices.push_back(c_i);
      }
    }
  }

  static _S angularDistance(const Quaternion<_S>& a, const Quaternion<_S>& b) {  // Eigen 3.3 semantics
    const _S bx = -b.x(), by = -b.y(), bz = -b.z(), bw = b.w();
    const _S dw = a.w() * bw - a.x() * bx - a.y() * by - a.z() * bz;
    const _S dx = a.w() * bx + a.x() * bw + a.y() * bz - a.z() * by;
    const _S dy = a.w() * by + a.y() * bw + a.z() * bx - a.x() * bz;
    const _S dz = a.w() * bz + a.z() * bw + a.x() * by - a.y() * bx;
    return _S(2) * std::atan2(std::sqrt(dx * dx + dy * dy + dz * dz), std::abs(dw));
  }

  // ref :1049-1098 (host: integer logic + two norms per clone)
  void findRedundantCamStates(std::vector<size_t>& rm_cam_state_ids) {
    if (cam_states_.size() < 5) return;
    const _S dist_thresh = msckf_params_.redundancy_distance_thresh;
    const _S angle_thresh = msckf_params_.redundancy_angle_thresh;
    size_t kf = 0;
    size_t next = 1;
    const size_t prot = cam_states_.size() - 3;
    while (next != prot) {
      _S d2 = 0;
      for (int i = 0; i < 3; ++i) { const _S d = cam_states_[next].p_C_G(i) - cam_states_[kf].p_C_G(i); d2 += d * d; }
      const _S distance = std::sqrt(d2);
      const _S angle = angularDistance(cam_states_[kf].q_CG, cam_states_[next].q_CG);
      if (distance < dist_thresh && angle < angle_thresh) rm_cam_state_ids.push_back(cam_states_[next].state_id);
      else kf = next;
      ++next;
      const int num_remaining = (int)(cam_states_.size() - rm_cam_state_ids.size());
      if (num_remaining <= msckf_params_.max_cam_states) break;
    }
    const int num_over_max = (int)(cam_states_.size() - rm_cam_state_ids.size()) - msckf_params_.max_cam_states;
    for (int i = 0; i < num_over_max; i++)
      if (rm_cam_state_ids.end() == std::find(rm_cam_state_ids.begin(), rm_cam_state_ids.end(), (size_t)cam_states_[i].state_id))
        rm_cam_state_ids.push_back(cam_states_[i].state_id);
    if (rm_cam_state_ids.size() < 2) rm_cam_state_ids.clear();
    std::sort(rm_cam_state_ids.begin(), rm_cam_state_ids.end());
  }
};

// Not in the reference: the per-image step of several independent filters (sequences, Monte-Carlo trials) as ONE device
// batch -- one launch per kernel with the filter index in the block index, one packed copy each way (msckf_b200_batch_* in
// include/msckf_b200.h).  The member functions below mean what MSCKF's members of the same name mean, applied to every
// filter; each filter ends bit-identical to calling them filter by filter.  The IMU readings queued by propagate() (here or
// on the filters themselves) go to the device in one call before any batched device call.  update() and addFeatures() are
// host bookkeeping only and stay per filter.  While the object lives the filters share its CUDA stream; all their own member
// functions stay usable.
template <typename _S>
class MSCKFBatch {
 public:
  explicit MSCKFBatch(const std::vector<MSCKF<_S>*>& filters, int host_threads = 1) : filters_(filters), threads_(host_threads) {
    std::vector<msckf_b200_engine*> es;
    for (auto* f : filters_) es.push_back(f->engine());
    if (msckf_b200_batch_create(es.data(), (int)es.size(), &batch_) != 0)
      throw std::runtime_error(std::string("msckf_b200_batch_create failed: ") + msckf_b200_last_error());
  }
  ~MSCKFBatch() { if (batch_) msckf_b200_batch_destroy(batch_); }
  MSCKFBatch(const MSCKFBatch&) = delete;
  MSCKFBatch& operator=(const MSCKFBatch&) = delete;
  size_t size() const { return filters_.size(); }
  const std::vector<MSCKF<_S>*>& filters() const { return filters_; }

  // MSCKF::propagate of filter i (queued on the host like there)
  void propagate(size_t i, imuReading<_S>& reading) { filters_.at(i)->propagate(reading); }
  // MSCKF::augmentState of every filter: state_ids[i] / times[i] for filter i
  void augmentState(const std::vector<int>& state_ids, const std::vector<_S>& times) {
    if (state_ids.size() != size() || times.size() != size()) throw std::invalid_argument("MSCKFBatch::augmentState: one state id and time per filter");
    flushImu();
    MSCKF<_S>::check(msckf_b200_batch_augment(batch_, nullptr), "msckf_b200_batch_augment");
    for (size_t i = 0; i < size(); ++i) filters_[i]->augmentAbsorb(state_ids[i], times[i]);
  }
  void marginalize() {
    const size_t n = size();
    flushImu();
    resetUpdate();
    bool any = false;
    for (size_t i = 0; i < n; ++i) {
      active_[i] = filters_[i]->marginalizePrepare(tracks_[i], false) ? 1 : 0;
      if (active_[i]) { filters_[i]->marginalizeReport(reports_[i]); any = true; }
    }
    if (!any) return;
    runUpdate(MSCKF_B200_MARGINALIZE);
    for (size_t i = 0; i < n; ++i)
      if (active_[i]) filters_[i]->marginalizeAbsorb(reports_[i]);
  }
  void pruneRedundantStates() {
    const size_t n = size();
    std::vector<char> wanted(n, 0);
    bool any = false;
    for (size_t i = 0; i < n; ++i) any |= (wanted[i] = filters_[i]->redundantPruneWanted() ? 1 : 0) != 0;
    if (!any) return;
    flushImu();
    refresh(wanted);
    resetUpdate();
    any = false;
    for (size_t i = 0; i < n; ++i)
      if (wanted[i]) any |= (active_[i] = filters_[i]->redundantTriangulatePrepare(tracks_[i], reports_[i], false) ? 1 : 0) != 0;
    if (any) {
      runUpdate(MSCKF_B200_TRIANGULATE);
      for (size_t i = 0; i < n; ++i) if (active_[i]) filters_[i]->redundantTriangulateAbsorb();
    }
    resetUpdate();
    any = false;
    for (size_t i = 0; i < n; ++i)
      if (wanted[i]) any |= (active_[i] = filters_[i]->redundantResidualizePrepare(tracks_[i], false) ? 1 : 0) != 0;
    if (any) {
      runUpdate(MSCKF_B200_RESIDUALIZE);
      for (size_t i = 0; i < n; ++i) if (active_[i]) filters_[i]->redundantResidualizeAbsorb(reports_[i]);
    }
    refresh(wanted);
    keep_.assign(n, std::vector<int>());
    std::vector<int> n_keep(n, -1);
    any = false;
    for (size_t i = 0; i < n; ++i)
      if (wanted[i] && filters_[i]->redundantDeletePrepare(keep_[i])) { n_keep[i] = (int)keep_[i].size(); any = true; }
    if (any) prune(n_keep);
  }
  void pruneEmptyStates() {
    const size_t n = size();
    std::vector<int> ndel(n, 0);
    std::vector<char> wanted(n, 0);
    bool any = false;
    for (size_t i = 0; i < n; ++i) any |= (wanted[i] = (ndel[i] = filters_[i]->emptyStatesToDelete()) > 0 ? 1 : 0) != 0;
    if (!any) return;
    flushImu();
    refresh(wanted);
    keep_.assign(n, std::vector<int>());
    std::vector<int> n_keep(n, -1);
    for (size_t i = 0; i < n; ++i)
      if (wanted[i]) { filters_[i]->emptyStatesDelete(ndel[i], keep_[i]); n_keep[i] = (int)keep_[i].size(); }
    prune(n_keep);
  }
  void finish() {
    for (auto* f : filters_) f->finishQueue();
    marginalize();
  }
  // brings every filter's host mirror of the IMU state and clone poses up to date with one synchronisation, so that the
  // getters after a batched step do not synchronise filter by filter
  void refreshState() {
    flushImu();
    refresh(std::vector<char>(size(), 1));
  }
  // MSCKF::nees of every filter (truth_cams empty, or truth_cams[i] == nullptr: no truth poses for filter i), as one
  // msckf_b200_batch_nees: one launch per 32 filters and one synchronisation
  std::vector<msckf_b200_nees_result> nees(const std::vector<imuState<double>>& truth,
                                           const std::vector<const std::vector<camState<double>>*>& truth_cams = {}) {
    const size_t n = size();
    if (truth.size() != n || (!truth_cams.empty() && truth_cams.size() != n))
      throw std::invalid_argument("MSCKFBatch::nees: one truth (and none or one truth window) per filter");
    flushImu();
    std::vector<std::vector<double>> im(n), poses(n);
    std::vector<const double*> pi(n), pp(n, nullptr);
    for (size_t i = 0; i < n; ++i) {
      const std::vector<camState<double>>* tc = truth_cams.empty() ? nullptr : truth_cams[i];
      filters_[i]->neesPack(truth[i], tc, im[i], poses[i]);
      pi[i] = im[i].data();
      if (tc) pp[i] = poses[i].data();
    }
    std::vector<msckf_b200_nees_result> r(n);
    MSCKF<_S>::check(msckf_b200_batch_nees(batch_, pi.data(), pp.data(), r.data()), "msckf_b200_batch_nees");
    return r;
  }
  // MSCKF::aidedUpdate of every filter (aid[i].model < 0: filter i is left alone) as one msckf_b200_batch_aid_update: one
  // launch per 32 updated filters and one synchronisation.  result[i] of a filter left alone is value-initialised.
  std::vector<msckf_b200_aid_result> aidedUpdate(const std::vector<msckf_b200_aid>& aid) {
    if (aid.size() != size()) throw std::invalid_argument("MSCKFBatch::aidedUpdate: one aided measurement per filter");
    flushImu();
    std::vector<msckf_b200_aid_result> r(size(), msckf_b200_aid_result());
    const int rc = msckf_b200_batch_aid_update(batch_, aid.data(), r.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch aided update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_aid_update");
    for (size_t i = 0; i < size(); ++i)
      if (aid[i].model >= 0) filters_[i]->aidAbsorb(r[i]);
    return r;
  }
  // MSCKF::aidedUpdate(items) of every filter (items[i] empty: filter i is left alone) as one msckf_b200_batch_aid_stack_update:
  // one launch per 32 updated filters and one synchronisation.  result[i] of a filter left alone is value-initialised.
  std::vector<msckf_b200_aid_result> aidedUpdate(const std::vector<std::vector<msckf_b200_aid_item>>& items, double chi2_max = 0) {
    const size_t n = size();
    if (items.size() != n) throw std::invalid_argument("MSCKFBatch::aidedUpdate: one item list per filter");
    std::vector<const msckf_b200_aid_item*> p(n, nullptr);
    std::vector<int> k(n, 0);
    for (size_t i = 0; i < n; ++i) {
      p[i] = items[i].empty() ? nullptr : items[i].data();
      k[i] = (int)items[i].size();
    }
    flushImu();
    std::vector<msckf_b200_aid_result> r(n, msckf_b200_aid_result());
    const int rc = msckf_b200_batch_aid_stack_update(batch_, p.data(), k.data(), chi2_max, r.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch stacked aided update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_aid_stack_update");
    for (size_t i = 0; i < n; ++i)
      if (!items[i].empty()) filters_[i]->aidAbsorb(r[i]);
    return r;
  }
  // MSCKF::aidedUpdate(items, fde) of every filter (items[i] empty: filter i is left alone) as one
  // msckf_b200_batch_aid_stack_update_fde with one fde: one launch per 32 updated filters and one synchronisation.
  std::vector<msckf_b200_aid_fde_result> aidedUpdate(const std::vector<std::vector<msckf_b200_aid_item>>& items, const msckf_b200_aid_fde& fde) {
    const size_t n = size();
    if (items.size() != n) throw std::invalid_argument("MSCKFBatch::aidedUpdate: one item list per filter");
    MSCKF<_S>::checkFde(fde);
    std::vector<const msckf_b200_aid_item*> p(n, nullptr);
    std::vector<int> k(n, 0);
    for (size_t i = 0; i < n; ++i) {
      p[i] = items[i].empty() ? nullptr : items[i].data();
      k[i] = (int)items[i].size();
    }
    flushImu();
    std::vector<msckf_b200_aid_fde_result> r(n, msckf_b200_aid_fde_result());
    const int rc = msckf_b200_batch_aid_stack_update_fde(batch_, p.data(), k.data(), &fde, r.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch stacked aided update (FDE): " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_aid_stack_update_fde");
    for (size_t i = 0; i < n; ++i)
      if (!items[i].empty()) filters_[i]->aidAbsorb(r[i].stack);
    return r;
  }
  // MSCKF::aidedUpdate(items, chi2_max, iter[i], iter_out[i]) of every filter (items[i] empty: filter i is left alone, iter[i]
  // not read) as one msckf_b200_batch_aid_stack_update_iter: one launch per 32 updated filters and one synchronisation.
  std::vector<msckf_b200_aid_result> aidedUpdate(const std::vector<std::vector<msckf_b200_aid_item>>& items, double chi2_max,
                                                 const std::vector<msckf_b200_aid_iter>& iter,
                                                 std::vector<msckf_b200_aid_iter_result>& iter_out) {
    std::vector<const msckf_b200_aid_item*> p;
    std::vector<int> k;
    iterArgs(items, iter, p, k, iter_out);
    std::vector<msckf_b200_aid_result> r(size(), msckf_b200_aid_result());
    const int rc = msckf_b200_batch_aid_stack_update_iter(batch_, p.data(), k.data(), chi2_max, iter.data(), r.data(), iter_out.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch stacked aided update (iterated): " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_aid_stack_update_iter");
    for (size_t i = 0; i < size(); ++i)
      if (!items[i].empty()) filters_[i]->aidAbsorb(r[i]);
    return r;
  }
  // the same with fault detection and exclusion, one fde for the batch (msckf_b200_batch_aid_stack_update_fde_iter)
  std::vector<msckf_b200_aid_fde_result> aidedUpdate(const std::vector<std::vector<msckf_b200_aid_item>>& items, const msckf_b200_aid_fde& fde,
                                                     const std::vector<msckf_b200_aid_iter>& iter,
                                                     std::vector<msckf_b200_aid_iter_result>& iter_out) {
    MSCKF<_S>::checkFde(fde);
    std::vector<const msckf_b200_aid_item*> p;
    std::vector<int> k;
    iterArgs(items, iter, p, k, iter_out);
    std::vector<msckf_b200_aid_fde_result> r(size(), msckf_b200_aid_fde_result());
    const int rc = msckf_b200_batch_aid_stack_update_fde_iter(batch_, p.data(), k.data(), &fde, iter.data(), r.data(), iter_out.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch stacked aided update (FDE, iterated): " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_aid_stack_update_fde_iter");
    for (size_t i = 0; i < size(); ++i)
      if (!items[i].empty()) filters_[i]->aidAbsorb(r[i].stack);
    return r;
  }
  // MSCKF::standstillUpdate of every filter (readings[i] empty: filter i is left alone and result[i] value-initialised) as one
  // msckf_b200_batch_standstill_update: one launch per 32 filters at rest by their scatter, none when no filter is, one
  // synchronisation.  Bad readings or a bad cfg throw before any device call.
  std::vector<msckf_b200_standstill_result> standstillUpdate(const std::vector<std::vector<imuReading<_S>>>& readings,
                                                             const msckf_b200_standstill& cfg) {
    const size_t n = size();
    if (readings.size() != n) throw std::invalid_argument("MSCKFBatch::standstillUpdate: one reading list per filter");
    std::vector<std::vector<_S>> r(n);
    std::vector<const void*> p(n, nullptr);
    std::vector<int> k(n, 0);
    for (size_t i = 0; i < n; ++i) {
      if (readings[i].empty()) continue;
      MSCKF<_S>::packStandstill(readings[i], cfg, r[i], "MSCKFBatch::standstillUpdate");
      p[i] = r[i].data();
      k[i] = (int)readings[i].size();
    }
    flushImu();
    std::vector<msckf_b200_standstill_result> o(n, msckf_b200_standstill_result());
    const int rc = msckf_b200_batch_standstill_update(batch_, p.data(), k.data(), &cfg, o.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch standstill update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_standstill_update");
    for (size_t i = 0; i < n; ++i)
      if (k[i]) filters_[i]->aidAbsorb(o[i].stack);
    return o;
  }
  // MSCKF::landmarkUpdate of every filter (obs[i] empty: filter i is left alone) as one msckf_b200_batch_landmark_update: three
  // launches per 32 updated filters and one synchronisation.  gamma / flag (optional) receive one list per filter.  An unknown
  // state_id throws before any device call.  result[i] of a filter left alone is value-initialised.  max_iter / tol: the
  // iterated update of MSCKF::landmarkUpdate for every updated filter (still one synchronisation).
  std::vector<msckf_b200_landmark_result> landmarkUpdate(const std::vector<std::vector<landmarkObservation>>& obs,
                                                         const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                                         std::vector<std::vector<double>>* gamma = nullptr,
                                                         std::vector<std::vector<int>>* flag = nullptr, int max_iter = 1,
                                                         double tol = 1e-10) {
    const size_t n = size();
    if (obs.size() != n) throw std::invalid_argument("MSCKFBatch::landmarkUpdate: one observation list per filter");
    if (gamma) gamma->assign(n, std::vector<double>());
    if (flag) flag->assign(n, std::vector<int>());
    std::vector<msckf_b200_landmarks> lm(n, msckf_b200_landmarks());
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty())
        filters_[i]->landmarkPack(obs[i], R, chi2_obs, gamma ? &(*gamma)[i] : nullptr, flag ? &(*flag)[i] : nullptr, lm[i]);
    for (size_t i = 0; i < n; ++i) { lm[i].max_iter = max_iter; lm[i].tol = tol; }
    flushImu();
    std::vector<msckf_b200_landmark_result> r(n, msckf_b200_landmark_result());
    const int rc = msckf_b200_batch_landmark_update(batch_, lm.data(), r.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch landmark update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_landmark_update");
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty()) filters_[i]->landmarkAbsorb(r[i]);
    return r;
  }
  // MSCKF::landmarkUpdate with map uncertainty for every filter (obs[i] empty: filter i is left alone; landmarks[i] is filter
  // i's landmark list) as one msckf_b200_batch_map_landmark_update.  Bad ids throw before any device call.
  std::vector<msckf_b200_landmark_result> landmarkUpdate(const std::vector<std::vector<mapObservation>>& obs,
                                                         const std::vector<std::vector<mapLandmark>>& landmarks,
                                                         const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                                         std::vector<std::vector<double>>* gamma = nullptr,
                                                         std::vector<std::vector<int>>* flag = nullptr, int max_iter = 1,
                                                         double tol = 1e-10) {
    const size_t n = size();
    if (obs.size() != n || landmarks.size() != n)
      throw std::invalid_argument("MSCKFBatch::landmarkUpdate: one observation list and one landmark list per filter");
    if (gamma) gamma->assign(n, std::vector<double>());
    if (flag) flag->assign(n, std::vector<int>());
    std::vector<msckf_b200_landmarks> lm(n, msckf_b200_landmarks());
    std::vector<msckf_b200_landmark_map> map(n, msckf_b200_landmark_map());
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty())
        filters_[i]->mapPack(obs[i], landmarks[i], R, chi2_obs, gamma ? &(*gamma)[i] : nullptr, flag ? &(*flag)[i] : nullptr, lm[i],
                             map[i]);
    for (size_t i = 0; i < n; ++i) { lm[i].max_iter = max_iter; lm[i].tol = tol; }
    flushImu();
    std::vector<msckf_b200_landmark_result> r(n, msckf_b200_landmark_result());
    const int rc = msckf_b200_batch_map_landmark_update(batch_, lm.data(), map.data(), r.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch map landmark update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_map_landmark_update");
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty()) filters_[i]->landmarkAbsorb(r[i]);
    return r;
  }
  // the two MSCKFBatch::landmarkUpdate forms above with a consensus per filter (cons[i], cons_out[i]) as one
  // msckf_b200_batch_landmark_update_consensus; an invalid consensus or id throws before any device call.  landmarks empty:
  // the exact map (landmarkObservation), else filter i's landmark list (mapObservation through obs_map).
  std::vector<msckf_b200_landmark_result> landmarkUpdate(const std::vector<std::vector<landmarkObservation>>& obs,
                                                         const std::vector<msckf_b200_landmark_consensus>& cons,
                                                         std::vector<msckf_b200_landmark_consensus_result>& cons_out,
                                                         const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                                         std::vector<std::vector<double>>* gamma = nullptr,
                                                         std::vector<std::vector<int>>* flag = nullptr, int max_iter = 1,
                                                         double tol = 1e-10) {
    const size_t n = size();
    if (obs.size() != n || cons.size() != n)
      throw std::invalid_argument("MSCKFBatch::landmarkUpdate: one observation list and one consensus per filter");
    for (const auto& c : cons) MSCKF<_S>::checkConsensus(c);
    if (gamma) gamma->assign(n, std::vector<double>());
    if (flag) flag->assign(n, std::vector<int>());
    std::vector<msckf_b200_landmarks> lm(n, msckf_b200_landmarks());
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty())
        filters_[i]->landmarkPack(obs[i], R, chi2_obs, gamma ? &(*gamma)[i] : nullptr, flag ? &(*flag)[i] : nullptr, lm[i]);
    for (size_t i = 0; i < n; ++i) { lm[i].max_iter = max_iter; lm[i].tol = tol; }
    return consensusCall(obs, lm, nullptr, cons, cons_out);
  }
  std::vector<msckf_b200_landmark_result> landmarkUpdate(const std::vector<std::vector<mapObservation>>& obs,
                                                         const std::vector<std::vector<mapLandmark>>& landmarks,
                                                         const std::vector<msckf_b200_landmark_consensus>& cons,
                                                         std::vector<msckf_b200_landmark_consensus_result>& cons_out,
                                                         const FixedMatrix<double, 2, 2>* R = nullptr, double chi2_obs = 0,
                                                         std::vector<std::vector<double>>* gamma = nullptr,
                                                         std::vector<std::vector<int>>* flag = nullptr, int max_iter = 1,
                                                         double tol = 1e-10) {
    const size_t n = size();
    if (obs.size() != n || landmarks.size() != n || cons.size() != n)
      throw std::invalid_argument("MSCKFBatch::landmarkUpdate: one observation list, one landmark list and one consensus per filter");
    for (const auto& c : cons) MSCKF<_S>::checkConsensus(c);
    if (gamma) gamma->assign(n, std::vector<double>());
    if (flag) flag->assign(n, std::vector<int>());
    std::vector<msckf_b200_landmarks> lm(n, msckf_b200_landmarks());
    std::vector<msckf_b200_landmark_map> map(n, msckf_b200_landmark_map());
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty())
        filters_[i]->mapPack(obs[i], landmarks[i], R, chi2_obs, gamma ? &(*gamma)[i] : nullptr, flag ? &(*flag)[i] : nullptr, lm[i],
                             map[i]);
    for (size_t i = 0; i < n; ++i) { lm[i].max_iter = max_iter; lm[i].tol = tol; }
    return consensusCall(obs, lm, map.data(), cons, cons_out);
  }
  template <class Obs>
  std::vector<msckf_b200_landmark_result> consensusCall(const std::vector<std::vector<Obs>>& obs, std::vector<msckf_b200_landmarks>& lm,
                                                        const msckf_b200_landmark_map* map,
                                                        const std::vector<msckf_b200_landmark_consensus>& cons,
                                                        std::vector<msckf_b200_landmark_consensus_result>& cons_out) {
    const size_t n = size();
    flushImu();
    std::vector<msckf_b200_landmark_result> r(n, msckf_b200_landmark_result());
    cons_out.assign(n, msckf_b200_landmark_consensus_result());
    const int rc = msckf_b200_batch_landmark_update_consensus(batch_, lm.data(), map, cons.data(), r.data(), cons_out.data());
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch landmark update: " << msckf_b200_last_error() << std::endl;
    else MSCKF<_S>::check(rc, "msckf_b200_batch_landmark_update_consensus");
    for (size_t i = 0; i < n; ++i)
      if (!obs[i].empty()) filters_[i]->landmarkAbsorb(r[i]);
    return r;
  }
  msckf_b200_batch* handle() { return batch_; }

 private:
  std::vector<MSCKF<_S>*> filters_;
  std::vector<msckf_b200_tracks> tracks_;
  std::vector<msckf_b200_report> reports_;
  std::vector<char> active_;
  std::vector<std::vector<int>> keep_;
  msckf_b200_batch* batch_ = nullptr;
  int threads_ = 1;

  // the iterated batch forms' arguments: one item list and one iter per filter (each updated filter's iter checked as
  // MSCKF::aidedUpdate does), the item pointers and counts, iter_out sized; then the IMU queues are handed over
  void iterArgs(const std::vector<std::vector<msckf_b200_aid_item>>& items, const std::vector<msckf_b200_aid_iter>& iter,
                std::vector<const msckf_b200_aid_item*>& p, std::vector<int>& k, std::vector<msckf_b200_aid_iter_result>& iter_out) {
    const size_t n = size();
    if (items.size() != n || iter.size() != n) throw std::invalid_argument("MSCKFBatch::aidedUpdate: one item list and one iter per filter");
    p.assign(n, nullptr);
    k.assign(n, 0);
    for (size_t i = 0; i < n; ++i) {
      if (!items[i].empty()) MSCKF<_S>::checkIter(iter[i]);
      p[i] = items[i].empty() ? nullptr : items[i].data();
      k[i] = (int)items[i].size();
    }
    iter_out.assign(n, msckf_b200_aid_iter_result());
    flushImu();
  }

  // the IMU readings queued on every filter, as one msckf_b200_batch_propagate_n
  void flushImu() {
    const size_t n = size();
    std::vector<const void*> r(n, nullptr);
    std::vector<int> k(n, 0);
    bool any = false;
    for (size_t i = 0; i < n; ++i) {
      k[i] = (int)(filters_[i]->imu_queue_.size() / 7);
      r[i] = filters_[i]->imu_queue_.data();
      any |= k[i] > 0;
    }
    if (!any) return;
    const int rc = msckf_b200_batch_propagate_n(batch_, r.data(), k.data());
    for (auto* f : filters_) f->imu_queue_.clear();
    MSCKF<_S>::check(rc, "msckf_b200_batch_propagate_n");
  }
  // MSCKF::refreshState of the filters with which[i] whose mirror is stale, as one msckf_b200_batch_get_state
  void refresh(const std::vector<char>& which) {
    const size_t n = size();
    std::vector<std::vector<_S>> im(n), poses(n);
    std::vector<void*> pi(n, nullptr), pp(n, nullptr);
    bool any = false;
    for (size_t i = 0; i < n; ++i) {
      if (!which[i] || !filters_[i]->state_dirty_) continue;
      im[i].resize(29);
      poses[i].resize(7 * std::max<size_t>(filters_[i]->cam_states_.size(), 1));
      pi[i] = im[i].data(); pp[i] = poses[i].data();
      any = true;
    }
    if (!any) return;
    MSCKF<_S>::check(msckf_b200_batch_get_state(batch_, pi.data(), pp.data()), "msckf_b200_batch_get_state");
    for (size_t i = 0; i < n; ++i)
      if (pi[i]) filters_[i]->refreshAbsorb(im[i].data(), poses[i].data());
  }
  void resetUpdate() {
    tracks_.assign(size(), msckf_b200_tracks());  // (n_tracks = 0: a member with nothing to do)
    reports_.assign(size(), msckf_b200_report());
    active_.assign(size(), 0);
  }
  void runUpdate(int mode) {
    const int rc = msckf_b200_batch_update(batch_, mode, tracks_.data(), reports_.data(), threads_);
    if (rc == MSCKF_B200_ERR_NUMERIC) std::cout << "[msckf_b200] batch update: " << msckf_b200_last_error() << std::endl;
    else if (rc != 0) throw std::runtime_error(std::string("msckf_b200_batch_update failed: ") + msckf_b200_last_error());
  }
  void prune(const std::vector<int>& n_keep) {
    std::vector<const int*> kp(size());
    for (size_t i = 0; i < size(); ++i) kp[i] = keep_[i].data();
    MSCKF<_S>::check(msckf_b200_batch_prune(batch_, kp.data(), n_keep.data()), "msckf_b200_batch_prune");
  }
};

}  // namespace msckf_mono
#endif /* MSCKF_HPP_ */
