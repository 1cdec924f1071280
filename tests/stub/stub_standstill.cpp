// tests/stub/stub_standstill.cpp -- TEST INFRASTRUCTURE ONLY.
// The standstill calls of include/msckf_b200.h (msckf_b200_standstill_update / _batch_standstill_update) and the stacked
// aided update (msckf_b200_aid_stack_update, for the at-rest class forms) for the recording fake tests/stub/stub_engine.cpp,
// with NO numerics.  Each call is checked as the engine checks it and recorded per engine: the single and batched calls, the
// IMU readings the engine had been handed by the last call, that call's readings (as doubles), its cfg, and the at-rest items
// of the last stacked call.  The answer is fixed so that a test can see every field travel back: stack = {nis k, dx_norm 0.5,
// dof 9, applied 1, status 0}, scatter = k + 0.25, outcome 0.  Linked with stub_engine.cpp, stub_batch_state.cpp and the C
// view (filter_capi.cpp, batch_capi.cpp, standstill_capi.cpp) into tests/stub/libmsckf_standstill_view_stub.so by
// tests/test_standstill_views_cpu.py.  Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>
#include <msckf_mono/msckf.h>

#include <cmath>
#include <map>
#include <vector>

#include "filter_view.hpp"

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
  long long single = 0, batch = 0, readings_at_last = -1, stack = 0;
  std::vector<double> readings;          // of the last standstill call, [k][7]
  double cfg[4] = {NAN, NAN, NAN, NAN};  // noise_scale, sigma_v, scatter_max, chi2_max
  std::vector<double> items;             // of the last stacked call: per item model, a, b, z[3], R[9]
};
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;

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
  Calls& c = g_calls[e];
  c.readings.assign(7 * (size_t)k, 0.0);
  for (int i = 0; i < 7 * k; ++i) c.readings[i] = e->dtype == MSCKF_B200_F32 ? (double)((const float*)r)[i] : ((const double*)r)[i];
  c.cfg[0] = cfg->noise_scale; c.cfg[1] = cfg->sigma_v; c.cfg[2] = cfg->scatter_max; c.cfg[3] = cfg->chi2_max;
  c.readings_at_last = e->imu_readings;
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
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_standstill_update(msckf_b200_batch* b, const void* const* readings, const int* k, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out) {
  if (!b || !readings || !k || !out || !valid_cfg(cfg)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k[i] != 0 && !valid(b->es[i], readings[i], k[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k[i] != 0) { record(b->es[i], readings[i], k[i], cfg, out + i); g_calls[b->es[i]].batch++; }
  g_batch_calls[b]++;
  return 0;
}
// the at-rest class forms reach the engine as a stack of one item: recorded, nothing applied
int msckf_b200_aid_stack_update(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double,
                                msckf_b200_aid_result* out) {
  if (!e || !out || !items || n_items < 1 || n_items > 8) return MSCKF_B200_ERR_ARG;
  Calls& c = g_calls[e];
  c.items.clear();
  for (int k = 0; k < n_items; ++k) {
    const msckf_b200_aid_item& it = items[k];
    if ((it.model != MSCKF_B200_AID_GYRO_AT_REST && it.model != MSCKF_B200_AID_ACCEL_AT_REST) || it.a || it.b || !it.z || !it.R)
      return MSCKF_B200_ERR_ARG;
    c.items.push_back(it.model); c.items.push_back(it.a); c.items.push_back(it.b);
    for (int i = 0; i < 3; ++i) c.items.push_back(it.z[i]);
    for (int i = 0; i < 9; ++i) c.items.push_back(it.R[i]);
  }
  c.stack++;
  *out = msckf_b200_aid_result{0.0, 0.0, 3 * n_items, 1, 0};
  return 0;
}
// test hooks: out4 = single standstill calls, batched calls naming e, IMU readings handed over before its last standstill call,
// stacked calls; cfg4 = that call's cfg; readings (cap x 7 doubles) = its readings, returns their count
int msckf_b200_stub_standstill_calls(const msckf_b200_engine* e, long long* out4, double* cfg4, double* readings, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out4[0] = c.single; out4[1] = c.batch; out4[2] = c.readings_at_last; out4[3] = c.stack;
  for (int i = 0; i < 4; ++i) cfg4[i] = c.cfg[i];
  const int k = (int)c.readings.size() / 7;
  for (int i = 0; i < 7 * k && i < 7 * cap; ++i) readings[i] = c.readings[i];
  return k;
}
// the items of e's last stacked call (cap x 15 doubles: model, a, b, z[3], R[9]); returns their count
int msckf_b200_stub_standstill_items(const msckf_b200_engine* e, double* rec, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  const int n = (int)c.items.size() / 15;
  for (int i = 0; i < 15 * n && i < 15 * cap; ++i) rec[i] = c.items[i];
  return n;
}
long long msckf_b200_stub_batch_standstill_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
// the at-rest class forms on a C view filter handle: which = 0 gyroAtRestUpdate(v3, R), 1 accelAtRestUpdate(v3, R); R is
// R_rows x R_rows row-major.  -1 with msckf_mono_last_error() for an exception.
int msckf_b200_stub_at_rest_class_call(void* h, int which, const double* v3, const double* R, int R_rows, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> v;
    for (int i = 0; i < 3; ++i) v(i) = v3[i];
    msckf_mono::MatrixX<double> Rm(R_rows, R_rows);
    for (int i = 0; i < R_rows; ++i)
      for (int j = 0; j < R_rows; ++j) Rm(i, j) = R[i * R_rows + j];
    msckf_view::Base* b = static_cast<msckf_view::Base*>(h);
    auto call = [&](auto& f) { *out = which == 0 ? f.gyroAtRestUpdate(v, Rm) : f.accelAtRestUpdate(v, Rm); return 0; };
    if (b->dtype == 0) return call(*static_cast<msckf_mono::MSCKF<float>*>(b->filter_ptr()));
    return call(*static_cast<msckf_mono::MSCKF<double>*>(b->filter_ptr()));
  });
}
}
