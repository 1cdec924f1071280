// tests/stub/stub_standstill.cpp -- TEST INFRASTRUCTURE ONLY.
// The standstill calls of include/msckf_b200.h (msckf_b200_standstill_update / _batch_standstill_update) for the recording
// fake of the C-ABI (tests/stub/stub.hpp), with NO numerics.  Each call is checked as the engine checks it and recorded per
// engine: the single and batched calls, the IMU readings the engine had been handed by the last call, that call's readings (as
// doubles) and its cfg.  The answer is fixed so that a test can see every field travel back: stack = {nis k, dx_norm 0.5, dof 9,
// applied 1, status 0}, scatter = k + 0.25, outcome 0.  The at-rest class forms reach the engine as stacked calls: their hooks
// here read what tests/stub/stub_aid_stack.cpp recorded.  Nothing outside tests/ builds or loads it.
#include "stub.hpp"

#include <cmath>

namespace {
struct Calls : stub::Calls {
  std::vector<double> readings;          // of the last standstill call, [k][7]
  double cfg[4] = {NAN, NAN, NAN, NAN};  // noise_scale, sigma_v, scatter_max, chi2_max
};
stub::Records<Calls> g_calls;

bool finite_pos(double x) { return std::isfinite(x) && x > 0.0; }
bool valid_cfg(const msckf_b200_standstill* c) {
  return c && std::isfinite(c->noise_scale) && c->noise_scale >= 1.0 && finite_pos(c->sigma_v) && finite_pos(c->scatter_max) &&
         finite_pos(c->chi2_max);
}
template <class S>
bool valid_readings(const S* r, int k) {
  if (!r || k < 2 || k > 4096) return false;
  for (int j = 0; j < k; ++j) {
    for (int i = 0; i < 7; ++i)
      if (!std::isfinite((double)r[7 * j + i])) return false;
    if (!((double)r[7 * j + 6] > 0.0)) return false;
  }
  return true;
}
bool valid(const msckf_b200_engine* e, const void* r, int k) {
  return e->dtype == MSCKF_B200_F32 ? valid_readings((const float*)r, k) : valid_readings((const double*)r, k);
}
void record(msckf_b200_engine* e, const void* r, int k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out) {
  Calls& c = g_calls.last(e);
  c.readings.assign(7 * (size_t)k, 0.0);
  for (int i = 0; i < 7 * k; ++i) c.readings[i] = e->dtype == MSCKF_B200_F32 ? (double)((const float*)r)[i] : ((const double*)r)[i];
  c.cfg[0] = cfg->noise_scale; c.cfg[1] = cfg->sigma_v; c.cfg[2] = cfg->scatter_max; c.cfg[3] = cfg->chi2_max;
  out->stack = msckf_b200_aid_result{(double)k, 0.5, 9, 1, 0};
  out->scatter = k + 0.25;
  out->outcome = 0;
}
}  // namespace

extern "C" {
int msckf_b200_standstill_update(msckf_b200_engine* e, const void* readings, int k, const msckf_b200_standstill* cfg,
                                 msckf_b200_standstill_result* out) {
  if (!e || !out || !valid_cfg(cfg) || !valid(e, readings, k)) return MSCKF_B200_ERR_ARG;
  record(e, readings, k, cfg, out);
  g_calls.engine[e].single++;
  return 0;
}
int msckf_b200_batch_standstill_update(msckf_b200_batch* b, const void* const* readings, const int* k, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out) {
  if (!b || !readings || !k || !out || !valid_cfg(cfg)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k[i] != 0 && !valid(b->es[i], readings[i], k[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k[i] != 0) { record(b->es[i], readings[i], k[i], cfg, out + i); g_calls.engine[b->es[i]].batch++; }
  g_calls.batch[b]++;
  return 0;
}
// test hooks: out4 = single standstill calls, batched calls naming e, IMU readings handed over before its last standstill call,
// single stacked calls; cfg4 = that call's cfg; readings (cap x 7 doubles) = its readings, returns their count
int msckf_b200_stub_standstill_calls(const msckf_b200_engine* e, long long* out4, double* cfg4, double* readings, int cap) {
  const Calls c = g_calls.of(e);
  g_calls.counts(e, out4);
  long long stack[3];
  double fde[33];
  msckf_b200_stub_aid_stack_calls(e, stack, fde, nullptr, 0);
  out4[3] = stack[0];
  for (int i = 0; i < 4; ++i) cfg4[i] = c.cfg[i];
  const int k = (int)c.readings.size() / 7;
  for (int i = 0; i < 7 * k && i < 7 * cap; ++i) readings[i] = c.readings[i];
  return k;
}
// the items of e's last stacked call (cap x 15 doubles: model, a, b, z[3], R[9]); returns their count
int msckf_b200_stub_standstill_items(const msckf_b200_engine* e, double* rec, int cap) {
  long long calls[3];
  double fde[33], items[20 * 8];  // (model, a, b, z[8], R[9] per item)
  const int n = msckf_b200_stub_aid_stack_calls(e, calls, fde, items, 8);
  for (int k = 0; k < n && k < cap; ++k) {
    const double* it = items + 20 * k;
    for (int i = 0; i < 6; ++i) rec[15 * k + i] = it[i];
    for (int i = 0; i < 9; ++i) rec[15 * k + 6 + i] = it[11 + i];
  }
  return n;
}
long long msckf_b200_stub_batch_standstill_calls(const msckf_b200_batch* b) { return g_calls.of(b); }
}
