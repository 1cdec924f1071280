// msckf_mono_b200/csrc/filter_capi.cpp -- C view (include/msckf_mono_c.h) of the drop-in class
// msckf_mono::MSCKF<float|double> (include/msckf_mono/msckf.h).  Host code only; links against the engine C-ABI.
#include <cstring>
#include <algorithm>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
namespace msckf_view {
thread_local std::string g_err;
}  // namespace msckf_view
using namespace msckf_view;

namespace {
template <class S>
struct Impl : Base {
  MSCKF<S> f;
  void set_engine_options(int dev, int mc, int mt, int mo) override { f.setEngineOptions(dev, mc, mt, mo); }
  void initialize(const double* c, const double* nz, const double* pr, const double* im) override {
    Camera<S> cam;
    cam.c_u = (S)c[0]; cam.c_v = (S)c[1]; cam.f_u = (S)c[2]; cam.f_v = (S)c[3]; cam.b = (S)c[4];
    cam.q_CI = Quaternion<S>((S)c[8], (S)c[5], (S)c[6], (S)c[7]);
    for (int i = 0; i < 3; ++i) cam.p_C_I(i) = (S)c[9 + i];
    noiseParams<S> noise;
    noise.u_var_prime = (S)nz[0]; noise.v_var_prime = (S)nz[1];
    for (int i = 0; i < 12; ++i) for (int j = 0; j < 12; ++j) noise.Q_imu(i, j) = (S)nz[2 + 12 * i + j];
    for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) noise.initial_imu_covar(i, j) = (S)nz[146 + 15 * i + j];
    MSCKFParams<S> p;
    p.max_gn_cost_norm = (S)pr[0]; p.min_rcond = (S)pr[1]; p.translation_threshold = (S)pr[2];
    p.redundancy_angle_thresh = (S)pr[3]; p.redundancy_distance_thresh = (S)pr[4];
    p.min_track_length = (int)pr[5]; p.max_track_length = (int)pr[6]; p.max_cam_states = (int)pr[7];
    imuState<S> s;
    for (int i = 0; i < 3; ++i) {
      s.p_I_G(i) = (S)im[i]; s.v_I_G(i) = (S)im[3 + i]; s.b_g(i) = (S)im[6 + i]; s.b_a(i) = (S)im[9 + i]; s.g(i) = (S)im[12 + i];
    }
    s.q_IG = Quaternion<S>((S)im[18], (S)im[15], (S)im[16], (S)im[17]);
    f.initialize(cam, noise, p, s);
  }
  void propagate(const double* m) override {
    imuReading<S> r;
    for (int i = 0; i < 3; ++i) { r.omega(i) = (S)m[i]; r.a(i) = (S)m[3 + i]; }
    r.dT = (S)m[6];
    f.propagate(r);
  }
  void augment(int id, double t) override { f.augmentState(id, (S)t); }
  static void conv(const double* z, const uint64_t* ids, int n, aligned_vector<Vector2<S>>& o, std::vector<size_t>& i) {
    o.resize(n); i.resize(n);
    for (int k = 0; k < n; ++k) { o[k](0) = (S)z[2 * k]; o[k](1) = (S)z[2 * k + 1]; i[k] = (size_t)ids[k]; }
  }
  void update(const double* z, const uint64_t* ids, int n) override {
    aligned_vector<Vector2<S>> o; std::vector<size_t> i; conv(z, ids, n, o, i); f.update(o, i);
  }
  void add(const double* z, const uint64_t* ids, int n) override {
    aligned_vector<Vector2<S>> o; std::vector<size_t> i; conv(z, ids, n, o, i); f.addFeatures(o, i);
  }
  void marginalize() override { f.marginalize(); }
  void marginalize_launch() override { f.marginalizeLaunch(); }
  void marginalize_collect() override { f.marginalizeCollect(); }
  void prune_redundant() override { f.pruneRedundantStates(); }
  void prune_empty() override { f.pruneEmptyStates(); }
  void finish() override { f.finish(); }
  int num_cam() override { return (int)f.getNumCamStates(); }
  void imu_state(double* o) override {
    const imuState<S> s = f.getImuState();
    for (int i = 0; i < 3; ++i) {
      o[i] = s.p_I_G(i); o[3 + i] = s.v_I_G(i); o[6 + i] = s.b_g(i); o[9 + i] = s.b_a(i); o[12 + i] = s.g(i);
      o[19 + i] = s.p_I_G_null(i); o[22 + i] = s.v_I_G_null(i);
    }
    o[15] = s.q_IG.x(); o[16] = s.q_IG.y(); o[17] = s.q_IG.z(); o[18] = s.q_IG.w();
    o[25] = s.q_IG_null.x(); o[26] = s.q_IG_null.y(); o[27] = s.q_IG_null.z(); o[28] = s.q_IG_null.w();
  }
  static void put_pose(double* p, const camState<S>& c) {
    for (int i = 0; i < 3; ++i) p[i] = c.p_C_G(i);
    p[3] = c.q_CG.x(); p[4] = c.q_CG.y(); p[5] = c.q_CG.z(); p[6] = c.q_CG.w();
  }
  void cam_states(double* poses, int* ids, double* times) override {
    const auto cs = f.getCamStates();
    for (size_t k = 0; k < cs.size(); ++k) {
      put_pose(poses + 7 * k, cs[k]);
      ids[2 * k] = cs[k].state_id; ids[2 * k + 1] = cs[k].last_correlated_id;
      times[k] = cs[k].time;
    }
  }
  int cam_tracked(int cam, uint64_t* out, int cap) override {
    const auto c = f.getCamState(cam);
    const int n = (int)c.tracked_feature_ids.size();
    for (int i = 0; i < std::min(n, cap); ++i) out[i] = c.tracked_feature_ids[i];
    return n;
  }
  int covariance(double* out) override {
    const std::vector<S> P = f.getCovariance();
    for (size_t i = 0; i < P.size(); ++i) out[i] = P[i];
    return 15 + 6 * (int)f.getNumCamStates();
  }
  int map(double* out, int cap) override {
    const auto m = f.getMap();
    for (int i = 0; i < std::min((int)m.size(), cap); ++i) for (int k = 0; k < 3; ++k) out[3 * i + k] = m[i](k);
    return (int)m.size();
  }
  int pruned(double* poses, int* ids, int cap) override {
    const auto ps = f.getPrunedStates();
    for (int k = 0; k < std::min((int)ps.size(), cap); ++k) {
      put_pose(poses + 7 * k, ps[k]); ids[2 * k] = ps[k].state_id; ids[2 * k + 1] = ps[k].last_correlated_id;
    }
    return (int)ps.size();
  }
  int tracked_ids(uint64_t* out, int cap) override {
    const auto& t = f.trackedFeatureIds();
    for (int i = 0; i < std::min((int)t.size(), cap); ++i) out[i] = t[i];
    return (int)t.size();
  }
  int report(int* flags, double* gamma, double* pfg, int cap) override {
    const auto& r = f.lastReport();
    for (int i = 0; i < std::min((int)r.size(), cap); ++i) {
      flags[4 * i] = r[i].cm_ok; flags[4 * i + 1] = r[i].valid; flags[4 * i + 2] = r[i].accepted; flags[4 * i + 3] = r[i].rows;
      gamma[i] = r[i].gamma;
      for (int k = 0; k < 3; ++k) pfg[3 * i + k] = r[i].p_f_G(k);
    }
    return (int)r.size();
  }
  int queued(uint64_t* ids, int* nobs, int cap) override {
    const auto& q = f.tracksToResidualize();
    for (int i = 0; i < std::min((int)q.size(), cap); ++i) { ids[i] = q[i].feature_id; nobs[i] = (int)q[i].observations.size(); }
    return (int)q.size();
  }
  int pack_queued(int* off, double* obs, int* idx, int cap_tracks, int cap_obs) override {
    const auto& q = f.tracksToResidualize();
    int tot = 0;
    if ((int)q.size() > cap_tracks) return -2;
    for (size_t t = 0; t < q.size(); ++t) {
      off[t] = tot;
      for (size_t i = 0; i < q[t].observations.size(); ++i) {
        if (tot >= cap_obs) return -2;
        obs[2 * tot] = q[t].observations[i](0); obs[2 * tot + 1] = q[t].observations[i](1);
        idx[tot] = (int)q[t].cam_state_indices[i];
        ++tot;
      }
    }
    off[q.size()] = tot;
    return (int)q.size();
  }
  msckf_b200_engine* engine() override { return f.engine(); }
  void* filter_ptr() override { return &f; }
  int last_m() override { return f.lastStackedRows(); }
  int last_rank() override { return f.lastRank(); }
};
}  // namespace

#define H ((Base*)h)
extern "C" {
const char* msckf_mono_last_error(void) { return g_err.c_str(); }
int msckf_mono_create(int dtype, void** out) {
  return guard([&] {
    Base* b = (dtype == 0) ? (Base*)new Impl<float>() : (Base*)new Impl<double>();
    b->dtype = dtype;
    *out = b;
    return 0;
  });
}
void msckf_mono_destroy(void* h) { delete H; }
int msckf_mono_set_engine_options(void* h, int device, int mc, int mt, int mo) { return guard([&] { H->set_engine_options(device, mc, mt, mo); return 0; }); }
int msckf_mono_initialize(void* h, const double* c, const double* n, const double* p, const double* i) { return guard([&] { H->initialize(c, n, p, i); return 0; }); }
int msckf_mono_propagate(void* h, const double* m) { return guard([&] { H->propagate(m); return 0; }); }
int msckf_mono_augment_state(void* h, int id, double t) { return guard([&] { H->augment(id, t); return 0; }); }
int msckf_mono_update(void* h, const double* z, const uint64_t* ids, int n) { return guard([&] { H->update(z, ids, n); return 0; }); }
int msckf_mono_add_features(void* h, const double* z, const uint64_t* ids, int n) { return guard([&] { H->add(z, ids, n); return 0; }); }
int msckf_mono_marginalize(void* h) { return guard([&] { H->marginalize(); return 0; }); }
int msckf_mono_marginalize_launch(void* h) { return guard([&] { H->marginalize_launch(); return 0; }); }
int msckf_mono_marginalize_collect(void* h) { return guard([&] { H->marginalize_collect(); return 0; }); }
int msckf_mono_prune_redundant_states(void* h) { return guard([&] { H->prune_redundant(); return 0; }); }
int msckf_mono_prune_empty_states(void* h) { return guard([&] { H->prune_empty(); return 0; }); }
int msckf_mono_finish(void* h) { return guard([&] { H->finish(); return 0; }); }
int msckf_mono_get_num_cam_states(void* h) { return guard([&] { return H->num_cam(); }); }
int msckf_mono_get_imu_state(void* h, double* o) { return guard([&] { H->imu_state(o); return 0; }); }
int msckf_mono_get_cam_states(void* h, double* p, int* ids, double* t) { return guard([&] { H->cam_states(p, ids, t); return 0; }); }
int msckf_mono_get_cam_tracked_ids(void* h, int cam, uint64_t* out, int cap) { return guard([&] { return H->cam_tracked(cam, out, cap); }); }
int msckf_mono_get_covariance(void* h, double* out) { return guard([&] { return H->covariance(out); }); }
int msckf_mono_get_map(void* h, double* out, int cap) { return guard([&] { return H->map(out, cap); }); }
int msckf_mono_get_pruned_states(void* h, double* p, int* ids, int cap) { return guard([&] { return H->pruned(p, ids, cap); }); }
int msckf_mono_get_tracked_feature_ids(void* h, uint64_t* out, int cap) { return guard([&] { return H->tracked_ids(out, cap); }); }
int msckf_mono_last_report(void* h, int* flags, double* gamma, double* pfg, int cap) { return guard([&] { return H->report(flags, gamma, pfg, cap); }); }
int msckf_mono_get_counters(void* h, long* out) {
  return guard([&] {
    long long c[8];
    int rc = msckf_b200_get_counters(H->engine(), c);
    if (rc != 0) throw std::runtime_error(msckf_b200_last_error());
    out[0] = (long)c[0]; out[1] = (long)c[1]; out[2] = (long)c[2]; out[3] = (long)c[3];
    out[4] = H->last_rank(); out[5] = H->last_m(); out[6] = 0; out[7] = 0;
    return 0;
  });
}
int msckf_mono_set_option(void* h, int key, double v) {
  return guard([&] {
    if (key >= 100) {  // engine options: 100 + key of msckf_b200_set_option
      int rc = msckf_b200_set_option(H->engine(), key - 100, v);
      if (rc) throw std::runtime_error(msckf_b200_last_error());
    }
    return 0;  // oracle-only keys (0..2) are accepted and ignored
  });
}
int msckf_mono_last_delta_x(void* h, double* out, int cap) { return guard([&] { return msckf_b200_last_delta_x(H->engine(), out, cap); }); }
int msckf_mono_queued_tracks(void* h, uint64_t* ids, int* nobs, int cap) { return guard([&] { return H->queued(ids, nobs, cap); }); }
int msckf_mono_pack_queued(void* h, int* off, double* obs, int* idx, int cap_tracks, int cap_obs) { return guard([&] { return H->pack_queued(off, obs, idx, cap_tracks, cap_obs); }); }
void* msckf_mono_engine(void* h) { return H->engine(); }
int msckf_mono_clone_from(void* dst, void* src) {
  (void)dst; (void)src;
  g_err = "clone_from: not implemented (use msckf_b200_copy_state on the engines of identically driven filters)";
  return -1;
}
}
