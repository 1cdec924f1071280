// tests/stub/stub_aid.cpp -- TEST INFRASTRUCTURE ONLY.
// The aided-update calls of include/msckf_b200.h (msckf_b200_aid_update / _batch_aid_update) for the recording fake
// tests/stub/stub_engine.cpp, with NO numerics: a VELOCITY or POSITION "update" copies z into the fake's IMU state (so that a
// caller can see whether its host mirror was refreshed), every other model changes nothing.  Each call is recorded with
// the number of IMU readings the engine had been handed by then.  Linked with stub_engine.cpp, stub_batch_state.cpp and the
// C view (filter_capi.cpp, batch_capi.cpp, aid_capi.cpp) into tests/stub/libmsckf_aid_view_stub.so by tests/test_aid_cpu.py.
// Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>

#include <map>
#include <string>
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
struct Calls { long long single = 0, batch = 0, readings_at_last = -1; };
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;
bool valid(const msckf_b200_engine* e, const msckf_b200_aid& a) {
  if (a.model > MSCKF_B200_AID_LINEAR || !a.z || !a.R) return false;
  if (a.model == MSCKF_B200_AID_CLONE_POSE && (a.clone < 0 || a.clone >= e->M)) return false;
  if (a.model == MSCKF_B200_AID_LINEAR && (a.m < 1 || a.m > 32 || a.n != 15 + 6 * e->M || !a.H)) return false;
  return true;
}
void apply(msckf_b200_engine* e, const msckf_b200_aid& a, msckf_b200_aid_result* r) {
  const int off = a.model == MSCKF_B200_AID_VELOCITY ? 3 : a.model == MSCKF_B200_AID_POSITION ? 0 : -1;
  if (off >= 0)
    for (int i = 0; i < 3; ++i) e->imu[off + i] = a.z[i];
  r->nis = 0.0; r->dx_norm = 0.0; r->applied = 1; r->status = 0;
  r->dof = a.model == MSCKF_B200_AID_LINEAR ? a.m : a.model <= MSCKF_B200_AID_POSITION ? 3 : 6;
  g_calls[e].readings_at_last = e->imu_readings;
}
}  // namespace

extern "C" {
int msckf_b200_aid_update(msckf_b200_engine* e, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  if (!e || !aid || !out || aid->model < 0 || !valid(e, *aid)) return MSCKF_B200_ERR_ARG;
  apply(e, *aid, out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_aid_update(msckf_b200_batch* b, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  if (!b || !aid || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (aid[i].model >= 0 && !valid(b->es[i], aid[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (aid[i].model >= 0) { apply(b->es[i], aid[i], out + i); g_calls[b->es[i]].batch++; }
  g_batch_calls[b]++;
  return 0;
}
// test hooks: out3 = single calls, batched calls naming this engine, IMU readings handed over before its last aided call;
// the batched calls made on b
void msckf_b200_stub_aid_calls(const msckf_b200_engine* e, long long* out3) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
}
long long msckf_b200_stub_batch_aid_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
}
