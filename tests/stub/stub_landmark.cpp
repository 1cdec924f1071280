// tests/stub/stub_landmark.cpp -- TEST INFRASTRUCTURE ONLY.
// The mapped-landmark calls of include/msckf_b200.h (msckf_b200_landmark_update / _batch_landmark_update) for the recording
// fake of the C-ABI (tests/stub/stub.hpp), with NO numerics: an "update" uses every observation, reports it as applied and
// changes nothing.  Each call records the window positions it was given, the number of IMU readings the engine had been handed
// by then, and the max_iter / tol it was given; it reports max(max_iter, 1) linearisations, converged when max_iter >= 2.
// Nothing outside tests/ builds or loads it.
#include "stub.hpp"

namespace {
struct Calls : stub::Calls { std::vector<int> clones; int max_iter = -1; double tol = -1.0; };
stub::Records<Calls> g_calls;
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
  Calls& c = g_calls.last(e);
  c.clones.assign(l.clone, l.clone + l.n_obs);
  c.max_iter = l.max_iter; c.tol = l.tol;
}
}  // namespace

extern "C" {
int msckf_b200_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  if (!e || !lm || !out || !valid(e, *lm)) return MSCKF_B200_ERR_ARG;
  apply(e, *lm, out);
  g_calls.engine[e].single++;
  return 0;
}
int msckf_b200_batch_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  if (!b || !lm || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (!valid(b->es[i], lm[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (lm[i].n_obs > 0) { apply(b->es[i], lm[i], out + i); g_calls.engine[b->es[i]].batch++; }
  g_calls.batch[b]++;
  return 0;
}
// test hooks: out3 = single calls, batched calls naming this engine, IMU readings handed over before its last call; the
// window positions of its last call (returns their number); max_iter and tol of its last call; the batched calls made on b
void msckf_b200_stub_landmark_calls(const msckf_b200_engine* e, long long* out3) { g_calls.counts(e, out3); }
int msckf_b200_stub_landmark_clones(const msckf_b200_engine* e, int* out, int cap) {
  const Calls c = g_calls.of(e);
  for (int i = 0; i < (int)c.clones.size() && i < cap; ++i) out[i] = c.clones[i];
  return (int)c.clones.size();
}
void msckf_b200_stub_landmark_iter(const msckf_b200_engine* e, int* max_iter, double* tol) {
  const Calls c = g_calls.of(e);
  *max_iter = c.max_iter; *tol = c.tol;
}
long long msckf_b200_stub_batch_landmark_calls(const msckf_b200_batch* b) { return g_calls.of(b); }
}
