// tests/stub/stub_landmark_consensus.cpp -- TEST INFRASTRUCTURE ONLY.
// The consensus forms of the mapped-landmark calls of include/msckf_b200.h (msckf_b200_landmark_update_consensus /
// _batch_landmark_update_consensus) for the recording fake tests/stub/stub_engine.cpp, with NO numerics: the consensus keeps
// every even observation and excludes (flag 3) every odd one, and nothing changes.  Each call records the window positions and
// consensus settings it was given and the number of IMU readings the engine had been handed by then.  Linked with
// stub_engine.cpp, stub_batch_state.cpp, stub_landmark_iter.cpp and the C view (filter_capi.cpp, batch_capi.cpp,
// landmark_capi.cpp, consensus_capi.cpp) into tests/stub/libmsckf_consensus_view_stub.so by
// tests/test_landmark_consensus_cpu.py.  Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>

#include <cmath>
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
  std::vector<int> clones;
  msckf_b200_landmark_consensus cons{};
};
std::map<const msckf_b200_engine*, Calls> g_calls;
bool valid(const msckf_b200_engine* e, const msckf_b200_landmarks& l, const msckf_b200_landmark_consensus* c) {
  if (l.n_obs < 0 || (l.n_obs > 0 && (!l.clone || !l.z || !l.p_L_G))) return false;
  for (int i = 0; i < l.n_obs; ++i)
    if (l.clone[i] < 0 || l.clone[i] >= e->M) return false;
  if (c && (c->hypotheses < 0 || c->hypotheses > 1024)) return false;
  if (c && c->hypotheses > 0 && (!std::isfinite(c->thresh) || !(c->thresh > 0.0) || c->min_inliers < 2)) return false;
  return true;
}
void apply(msckf_b200_engine* e, const msckf_b200_landmarks& l, const msckf_b200_landmark_consensus* c, msckf_b200_landmark_result* r,
           msckf_b200_landmark_consensus_result* co) {
  const bool on = c && c->hypotheses > 0;
  int used = 0;
  for (int i = 0; i < l.n_obs; ++i) {
    const int f = on && (i & 1) ? 3 : 0;
    used += f == 0;
    if (l.gamma) l.gamma[i] = 0.0;
    if (l.flag) l.flag[i] = f;
  }
  r->nis = 0.0; r->dx_norm = 0.0; r->dof = 2 * used; r->rows = 0; r->used = used; r->applied = used > 0; r->status = 0;
  r->iterations = used > 0; r->converged = 0; r->step = 0.0;
  if (co) {
    *co = msckf_b200_landmark_consensus_result{};
    co->best = on ? 0 : -1; co->valid = on ? c->hypotheses : 0; co->inliers = on ? used : 0;
  }
  if (on && c->scores)
    for (int k = 0; k < c->hypotheses; ++k) c->scores[k] = used;
  Calls& k = g_calls[e];
  k.readings_at_last = e->imu_readings;
  k.clones.assign(l.clone, l.clone + l.n_obs);
  k.cons = c ? *c : msckf_b200_landmark_consensus{};
}
}  // namespace

extern "C" {
int msckf_b200_landmark_update_consensus(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                         msckf_b200_landmark_consensus_result* cons_out) {
  (void)map;
  if (!e || !lm || !out || !valid(e, *lm, cons)) return MSCKF_B200_ERR_ARG;
  apply(e, *lm, cons, out, cons_out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_landmark_update_consensus(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                               const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                               msckf_b200_landmark_consensus_result* cons_out) {
  (void)map;
  if (!b || !lm || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (!valid(b->es[i], lm[i], cons ? cons + i : nullptr)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (lm[i].n_obs > 0) {
      apply(b->es[i], lm[i], cons ? cons + i : nullptr, out + i, cons_out ? cons_out + i : nullptr);
      g_calls[b->es[i]].batch++;
    }
  return 0;
}
// test hooks: out3 = single consensus calls, batched consensus calls naming this engine, IMU readings handed over before its
// last call; the last call's window positions (cap) and hypotheses / min_inliers / seed (c3); returns n_obs
void msckf_b200_stub_consensus_calls(const msckf_b200_engine* e, long long* out3) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
}
int msckf_b200_stub_consensus_last(const msckf_b200_engine* e, int* clones, int cap, unsigned long long* c3) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  for (int i = 0; i < (int)c.clones.size() && i < cap; ++i) clones[i] = c.clones[i];
  c3[0] = (unsigned long long)c.cons.hypotheses; c3[1] = (unsigned long long)c.cons.min_inliers; c3[2] = c.cons.seed;
  return (int)c.clones.size();
}
}
