// tests/stub/stub_aid_stack.cpp -- TEST INFRASTRUCTURE ONLY.
// The stacked aided-update calls of include/msckf_b200.h (msckf_b200_aid_stack_update / _batch_aid_stack_update) for the
// recording fake tests/stub/stub_engine.cpp, with NO numerics: a VELOCITY or POSITION item copies z into the fake's IMU state
// (so that a caller can see whether its host mirror was refreshed), every other item changes nothing.  Each call is recorded
// with its items and the number of IMU readings the engine had been handed by then.  Linked with stub_engine.cpp,
// stub_batch_state.cpp, stub_aid.cpp and the C view (filter_capi.cpp, batch_capi.cpp, aid_capi.cpp, aid_stack_capi.cpp) into
// tests/stub/libmsckf_odometry_view_stub.so by tests/test_odometry_cpu.py.  Nothing outside tests/ builds or loads it.
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
struct Calls {
  long long single = 0, batch = 0, readings_at_last = -1;
  std::vector<int> last;  // (model, a, b) of the items of the last call
};
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;
int rows(const msckf_b200_aid_item& it) {
  if (it.model == MSCKF_B200_AID_BODY_VELOCITY) return (it.a & 1) + ((it.a >> 1) & 1) + ((it.a >> 2) & 1);
  return it.model <= MSCKF_B200_AID_POSITION ? 3 : 6;
}
bool valid(const msckf_b200_engine* e, const msckf_b200_aid_item* items, int n) {
  if (n < 1 || n > 8 || !items) return false;
  int m = 0;
  for (int k = 0; k < n; ++k) {
    const msckf_b200_aid_item& it = items[k];
    if (it.model < 0 || it.model > MSCKF_B200_AID_RELATIVE_POSE || it.model == MSCKF_B200_AID_LINEAR || !it.z || !it.R) return false;
    if (it.model == MSCKF_B200_AID_CLONE_POSE && (it.a < 0 || it.a >= e->M)) return false;
    if (it.model == MSCKF_B200_AID_RELATIVE_POSE && (it.a < 0 || it.a >= e->M || it.b < 0 || it.b >= e->M || it.a == it.b)) return false;
    if (it.model == MSCKF_B200_AID_BODY_VELOCITY && (it.a < 1 || it.a > 7)) return false;
    m += rows(it);
  }
  return m <= 32;
}
void apply(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, msckf_b200_aid_result* r) {
  Calls& c = g_calls[e];
  c.last.clear();
  r->nis = 0.0; r->dx_norm = 0.0; r->applied = 1; r->status = 0; r->dof = 0;
  for (int k = 0; k < n; ++k) {
    const msckf_b200_aid_item& it = items[k];
    const int off = it.model == MSCKF_B200_AID_VELOCITY ? 3 : it.model == MSCKF_B200_AID_POSITION ? 0 : -1;
    if (off >= 0)
      for (int i = 0; i < 3; ++i) e->imu[off + i] = it.z[i];
    r->dof += rows(it);
    c.last.insert(c.last.end(), {it.model, it.a, it.b});
  }
  c.readings_at_last = e->imu_readings;
}
}  // namespace

extern "C" {
int msckf_b200_aid_stack_update(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                msckf_b200_aid_result* out) {
  (void)chi2_max;
  if (!e || !out || !valid(e, items, n_items)) return MSCKF_B200_ERR_ARG;
  apply(e, items, n_items, out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_aid_stack_update(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                      double chi2_max, msckf_b200_aid_result* out) {
  (void)chi2_max;
  if (!b || !items || !n_items || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0 && !valid(b->es[i], items[i], n_items[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0) { apply(b->es[i], items[i], n_items[i], out + i); g_calls[b->es[i]].batch++; }
  g_batch_calls[b]++;
  return 0;
}
// test hooks: out3 = single calls, batched calls naming this engine, IMU readings handed over before its last stacked call;
// items3 (cap triples) = (model, a, b) of that call's items, returns their count; the batched calls made on b
int msckf_b200_stub_aid_stack_calls(const msckf_b200_engine* e, long long* out3, int* items3, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
  const int n = (int)c.last.size() / 3;
  for (int k = 0; k < n && k < cap; ++k)
    for (int j = 0; j < 3; ++j) items3[3 * k + j] = c.last[3 * k + j];
  return n;
}
long long msckf_b200_stub_batch_aid_stack_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
}
