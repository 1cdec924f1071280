// tests/stub/stub_range_stack.cpp -- TEST INFRASTRUCTURE ONLY.
// The stacked aided-update calls of include/msckf_b200.h (msckf_b200_aid_stack_update / _batch_aid_stack_update) for the
// recording fake tests/stub/stub_engine.cpp, with NO numerics, like stub_gnss_stack.cpp but accepting every stack model up to
// CLONE_PLANE_RANGE: every item is recorded in full -- model, a, b, its z and its R -- so that a test can see exactly what the
// class's range forms and the C view send.  A VELOCITY or POSITION item copies z into the fake's IMU state.  Also the class forms
// themselves for a C view handle (MSCKF<_S>::rangeUpdate, cloneRangeUpdate, planeRangeUpdate, clonePlaneRangeUpdate), which have
// no C view entry points.  Linked with stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp and the C view (filter_capi.cpp,
// batch_capi.cpp, aid_capi.cpp, aid_stack_capi.cpp) into tests/stub/libmsckf_range_view_stub.so by tests/test_range_cpu.py.
// Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>
#include <msckf_mono/msckf.h>

#include <cmath>
#include <map>
#include <string>
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
constexpr int kRec = 20;  // per recorded item: model, a, b, z[8] (NaN past the model's length), R[9] (rows x rows, then NaN)
struct Calls {
  long long single = 0, batch = 0;
  std::vector<double> last;  // the items of the last call
};
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;
int popc(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1); }
int rows(const msckf_b200_aid_item& it) {
  switch (it.model) {
    case MSCKF_B200_AID_VELOCITY: case MSCKF_B200_AID_POSITION: return 3;
    case MSCKF_B200_AID_BODY_VELOCITY: case MSCKF_B200_AID_ANTENNA_POSITION: return popc(it.a);
    case MSCKF_B200_AID_CLONE_ANTENNA_POSITION: return popc(it.b);
    case MSCKF_B200_AID_HEADING: case MSCKF_B200_AID_CLONE_HEADING:
    case MSCKF_B200_AID_RANGE: case MSCKF_B200_AID_CLONE_RANGE:
    case MSCKF_B200_AID_PLANE_RANGE: case MSCKF_B200_AID_CLONE_PLANE_RANGE: return 1;
    default: return 6;
  }
}
int zlen(int model) {
  switch (model) {
    case MSCKF_B200_AID_VELOCITY: case MSCKF_B200_AID_POSITION: case MSCKF_B200_AID_BODY_VELOCITY: return 3;
    case MSCKF_B200_AID_ANTENNA_POSITION: case MSCKF_B200_AID_CLONE_ANTENNA_POSITION: return 6;
    case MSCKF_B200_AID_HEADING: case MSCKF_B200_AID_CLONE_HEADING: return 4;
    case MSCKF_B200_AID_PLANE_RANGE: case MSCKF_B200_AID_CLONE_PLANE_RANGE: return 8;
    default: return 7;
  }
}
bool valid(const msckf_b200_engine* e, const msckf_b200_aid_item* items, int n) {
  if (n < 1 || n > 8 || !items) return false;
  int m = 0;
  for (int k = 0; k < n; ++k) {
    const msckf_b200_aid_item& it = items[k];
    if (it.model < 0 || it.model > MSCKF_B200_AID_CLONE_PLANE_RANGE || it.model == MSCKF_B200_AID_LINEAR || !it.z || !it.R) return false;
    const bool clone = it.model == MSCKF_B200_AID_CLONE_POSE || it.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION ||
                       it.model == MSCKF_B200_AID_CLONE_HEADING || it.model == MSCKF_B200_AID_RELATIVE_POSE ||
                       it.model == MSCKF_B200_AID_CLONE_RANGE || it.model == MSCKF_B200_AID_CLONE_PLANE_RANGE;
    if (clone && (it.a < 0 || it.a >= e->M)) return false;
    if (it.model == MSCKF_B200_AID_RELATIVE_POSE && (it.b < 0 || it.b >= e->M || it.a == it.b)) return false;
    if ((it.model == MSCKF_B200_AID_BODY_VELOCITY || it.model == MSCKF_B200_AID_ANTENNA_POSITION) && (it.a < 1 || it.a > 7)) return false;
    if (it.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION && (it.b < 1 || it.b > 7)) return false;
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
    const int m = rows(it), nz = zlen(it.model);
    r->dof += m;
    std::vector<double> rec(kRec, NAN);
    rec[0] = it.model; rec[1] = it.a; rec[2] = it.b;
    for (int i = 0; i < nz; ++i) rec[3 + i] = it.z[i];
    for (int i = 0; i < m * m && i < 9; ++i) rec[11 + i] = it.R[i];
    c.last.insert(c.last.end(), rec.begin(), rec.end());
  }
}
template <class F>
int on_filter(void* h, F&& f) {
  msckf_view::Base* b = static_cast<msckf_view::Base*>(h);
  if (b->dtype == 0) return f(*static_cast<msckf_mono::MSCKF<float>*>(b->filter_ptr()));
  return f(*static_cast<msckf_mono::MSCKF<double>*>(b->filter_ptr()));
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
// test hooks: out2 = single calls, batched calls naming this engine; rec (cap x 20 doubles) = the items of its last stacked call
// (model, a, b, z[8], R[9], NaN-padded), returns their count; the batched calls made on b
int msckf_b200_stub_range_calls(const msckf_b200_engine* e, long long* out2, double* rec, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out2[0] = c.single; out2[1] = c.batch;
  const int n = (int)c.last.size() / kRec;
  for (int k = 0; k < n && k < cap; ++k)
    for (int j = 0; j < kRec; ++j) rec[kRec * k + j] = c.last[kRec * k + j];
  return n;
}
long long msckf_b200_stub_range_batch_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
// the class forms on a C view filter handle: which = 0 rangeUpdate(rho, a3, l3, var), 1 cloneRangeUpdate(state_id, rho, a3, l3,
// var), 2 planeRangeUpdate(rho, h, l3, f3, var), 3 clonePlaneRangeUpdate(state_id, rho, h, l3, f3, var).  -1 with
// msckf_mono_last_error() for an exception.
int msckf_b200_stub_range_class_call(void* h, int which, int state_id, double rho, double height, const double* a3, const double* l3,
                                     const double* f3, double var, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> a, l, f;
    for (int i = 0; i < 3; ++i) { a(i) = a3[i]; l(i) = l3[i]; f(i) = f3[i]; }
    return on_filter(h, [&](auto& flt) {
      if (which == 0) *out = flt.rangeUpdate(rho, a, l, var);
      else if (which == 1) *out = flt.cloneRangeUpdate(state_id, rho, a, l, var);
      else if (which == 2) *out = flt.planeRangeUpdate(rho, height, l, f, var);
      else *out = flt.clonePlaneRangeUpdate(state_id, rho, height, l, f, var);
      return 0;
    });
  });
}
}
