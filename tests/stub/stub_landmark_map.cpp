// tests/stub/stub_landmark_map.cpp -- TEST INFRASTRUCTURE ONLY.
// The mapped-landmark calls with map uncertainty of include/msckf_b200.h (msckf_b200_map_landmark_update /
// _batch_map_landmark_update) for the recording fake tests/stub/stub_engine.cpp, with NO numerics: every observation is used
// and reported as applied, nothing changes.  Each call records the window positions, landmark ids and Sigma it was given and
// the number of IMU readings the engine had been handed by then.  Linked with stub_engine.cpp, stub_batch_state.cpp,
// stub_landmark_iter.cpp and the C view (filter_capi.cpp, batch_capi.cpp, landmark_capi.cpp, map_capi.cpp) into
// tests/stub/libmsckf_landmark_map_view_stub.so by tests/test_landmark_map_cpu.py.  Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>

#include <map>
#include <vector>

// the fake's handles: the same definitions as in stub_engine.cpp (one type across the translation units)
struct msckf_b200_engine {
  int dtype = 0, M = 0, max_clones = 0;
  double imu[19] = {0};
  std::vector<int> last_len;
  std::vector<int> buf_off, buf_idx;
  std::vector<double> buf_obs, buf_pfg;
  long long imu_readings = 0;
  int pending = 0, mode = 0;
  long long updates = 0, launches = 0;
};
struct msckf_b200_batch { std::vector<msckf_b200_engine*> es; long long launches = 0; };

namespace {
struct Calls {
  long long single = 0, batch = 0, readings_at_last = -1;
  std::vector<int> clones, landmark;
  std::vector<double> p, sigma;
};
std::map<const msckf_b200_engine*, Calls> g_calls;
bool valid(const msckf_b200_engine* e, const msckf_b200_landmarks& l, const msckf_b200_landmark_map* m) {
  if (l.n_obs < 0 || (l.n_obs > 0 && (!l.clone || !l.z || !l.p_L_G))) return false;
  for (int i = 0; i < l.n_obs; ++i)
    if (l.clone[i] < 0 || l.clone[i] >= e->M) return false;
  if (m && m->Sigma_L)
    for (int i = 0; i < l.n_obs; ++i)
      if (!m->landmark || m->landmark[i] < 0 || m->landmark[i] >= m->n_landmarks) return false;
  return true;
}
void apply(msckf_b200_engine* e, const msckf_b200_landmarks& l, const msckf_b200_landmark_map* m, msckf_b200_landmark_result* r) {
  r->nis = 0.0; r->dx_norm = 0.0; r->dof = 2 * l.n_obs; r->rows = 0; r->used = l.n_obs; r->applied = 1; r->status = 0;
  r->iterations = 1; r->converged = 0; r->step = 0.0;
  for (int i = 0; i < l.n_obs; ++i) {
    if (l.gamma) l.gamma[i] = 0.0;
    if (l.flag) l.flag[i] = 0;
  }
  Calls& c = g_calls[e];
  c.readings_at_last = e->imu_readings;
  c.clones.assign(l.clone, l.clone + l.n_obs);
  c.p.assign(l.p_L_G, l.p_L_G + 3 * l.n_obs);
  c.landmark.clear(); c.sigma.clear();
  if (m && m->Sigma_L) {
    c.landmark.assign(m->landmark, m->landmark + l.n_obs);
    c.sigma.assign(m->Sigma_L, m->Sigma_L + 6 * m->n_landmarks);
  }
}
}  // namespace

extern "C" {
int msckf_b200_map_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                   msckf_b200_landmark_result* out) {
  if (!e || !lm || !out || !valid(e, *lm, map)) return MSCKF_B200_ERR_ARG;
  apply(e, *lm, map, out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_map_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         msckf_b200_landmark_result* out) {
  if (!b || !lm || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (!valid(b->es[i], lm[i], map ? map + i : nullptr)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (lm[i].n_obs > 0) { apply(b->es[i], lm[i], map ? map + i : nullptr, out + i); g_calls[b->es[i]].batch++; }
  return 0;
}
// test hooks: out3 = single map calls, batched map calls naming this engine, IMU readings handed over before its last call
void msckf_b200_stub_map_calls(const msckf_b200_engine* e, long long* out3) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
}
// the last call's window positions, landmark ids, p_L_G [n][3] (cap observations) and Sigma (cap6 doubles); returns n_obs and
// writes the number of Sigma doubles to n6
int msckf_b200_stub_map_last(const msckf_b200_engine* e, int* clones, int* landmark, double* p, int cap, double* sigma, int cap6,
                             int* n6) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  for (int i = 0; i < (int)c.clones.size() && i < cap; ++i) {
    clones[i] = c.clones[i];
    landmark[i] = i < (int)c.landmark.size() ? c.landmark[i] : -1;
    for (int k = 0; k < 3; ++k) p[3 * i + k] = c.p[3 * i + k];
  }
  for (int i = 0; i < (int)c.sigma.size() && i < cap6; ++i) sigma[i] = c.sigma[i];
  *n6 = (int)c.sigma.size();
  return (int)c.clones.size();
}
}
