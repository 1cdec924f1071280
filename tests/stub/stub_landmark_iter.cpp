// tests/stub/stub_landmark_iter.cpp -- TEST INFRASTRUCTURE ONLY.
// The mapped-landmark calls of include/msckf_b200.h (msckf_b200_landmark_update / _batch_landmark_update) for the recording
// fake tests/stub/stub_engine.cpp, with NO numerics: an "update" uses every observation, reports it as applied and changes
// nothing.  Each call records the window positions it was given and the number of IMU readings the engine had been handed by
// then, and the max_iter / tol it was given; it reports max(max_iter, 1) linearisations, converged when max_iter >= 2.  Linked
// with stub_engine.cpp, stub_batch_state.cpp and the C view (filter_capi.cpp, batch_capi.cpp, landmark_capi.cpp) into
// tests/stub/libmsckf_landmark_iter_view_stub.so by tests/test_landmark_iter_cpu.py.  Nothing outside tests/ builds or loads it.
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
struct Calls { long long single = 0, batch = 0, readings_at_last = -1; std::vector<int> clones; int max_iter = -1; double tol = -1.0; };
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;
bool valid(const msckf_b200_engine* e, const msckf_b200_landmarks& l) {
  if (l.max_iter < 0 || l.max_iter > 16 || !(l.tol >= 0.0)) return false;
  if (l.n_obs < 0 || (l.n_obs > 0 && (!l.clone || !l.z || !l.p_L_G))) return false;
  for (int i = 0; i < l.n_obs; ++i)
    if (l.clone[i] < 0 || l.clone[i] >= e->M) return false;
  return true;
}
void apply(msckf_b200_engine* e, const msckf_b200_landmarks& l, msckf_b200_landmark_result* r) {
  r->nis = 0.0; r->dx_norm = 0.0; r->dof = 2 * l.n_obs; r->rows = 0; r->used = l.n_obs; r->applied = 1; r->status = 0;
  r->iterations = l.max_iter > 1 ? l.max_iter : 1; r->converged = l.max_iter > 1; r->step = 0.0;
  for (int i = 0; i < l.n_obs; ++i) {
    if (l.gamma) l.gamma[i] = 0.0;
    if (l.flag) l.flag[i] = 0;
  }
  Calls& c = g_calls[e];
  c.readings_at_last = e->imu_readings;
  c.clones.assign(l.clone, l.clone + l.n_obs);
  c.max_iter = l.max_iter; c.tol = l.tol;
}
}  // namespace

extern "C" {
int msckf_b200_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  if (!e || !lm || !out || !valid(e, *lm)) return MSCKF_B200_ERR_ARG;
  apply(e, *lm, out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  if (!b || !lm || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (!valid(b->es[i], lm[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (lm[i].n_obs > 0) { apply(b->es[i], lm[i], out + i); g_calls[b->es[i]].batch++; }
  g_batch_calls[b]++;
  return 0;
}
// test hooks: out3 = single calls, batched calls naming this engine, IMU readings handed over before its last call; the
// window positions of its last call (returns their number); the batched calls made on b
void msckf_b200_stub_landmark_calls(const msckf_b200_engine* e, long long* out3) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
}
int msckf_b200_stub_landmark_clones(const msckf_b200_engine* e, int* out, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  for (int i = 0; i < (int)c.clones.size() && i < cap; ++i) out[i] = c.clones[i];
  return (int)c.clones.size();
}
// max_iter and tol of this engine's last call
void msckf_b200_stub_landmark_iter(const msckf_b200_engine* e, int* max_iter, double* tol) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  *max_iter = c.max_iter; *tol = c.tol;
}
long long msckf_b200_stub_batch_landmark_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
}
