// tests/stub/stub_aid_stack.cpp -- TEST INFRASTRUCTURE ONLY.
// The stacked aided-update calls of include/msckf_b200.h (msckf_b200_aid_stack_update / _batch_aid_stack_update and their
// fault detection and exclusion forms, _fde) for the recording fake tests/stub/stub_engine.cpp, with NO numerics.  Each call's
// items are checked as the engine checks them (every stack model; for _fde also the thresholds and max_exclude) and recorded
// per engine: the single and batched calls, the IMU readings the engine had been handed by the last call, that call's fde
// (chi2[32], max_exclude) and its items in full -- model, a, b, z (8 doubles, NaN past the model's length) and R (rows x
// rows, then NaN) -- so that a test can see exactly what the class forms and the C view send.  A VELOCITY or POSITION item
// copies z into the fake's IMU state (so that a caller can see whether its host mirror was refreshed); every other item
// changes nothing, and the _fde forms answer outcome 0 with every item used.  Also the GNSS and range class forms themselves
// for a C view handle, which have no C view entry points.  Linked with stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp
// and the C view (filter_capi.cpp, batch_capi.cpp, aid_capi.cpp, aid_stack_capi.cpp, fde_capi.cpp) into
// tests/stub/libmsckf_aid_stack_view_stub.so by tests/aid_stack_stub.py.  Nothing outside tests/ builds or loads it.
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
constexpr int kRec = 20;  // per recorded item: model, a, b, z[8], R[9]
constexpr int kFde = 33;  // chi2[32], max_exclude
struct Calls {
  long long single = 0, batch = 0, readings_at_last = -1;
  std::vector<double> fde;   // of the last call (NaN: a call without FDE)
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
bool valid_fde(const msckf_b200_aid_fde* fde) {
  if (!fde || fde->max_exclude < 0 || fde->max_exclude > 7) return false;
  for (int d = 0; d < 32; ++d)
    if (!(std::isfinite(fde->chi2[d]) && fde->chi2[d] > 0.0)) return false;
  return true;
}
// records the call and returns its rows
int record(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, const msckf_b200_aid_fde* fde) {
  Calls& c = g_calls[e];
  c.fde.assign(kFde, NAN);
  if (fde) {
    for (int d = 0; d < 32; ++d) c.fde[d] = fde->chi2[d];
    c.fde[32] = fde->max_exclude;
  }
  c.last.clear();
  int dof = 0;
  for (int k = 0; k < n; ++k) {
    const msckf_b200_aid_item& it = items[k];
    const int off = it.model == MSCKF_B200_AID_VELOCITY ? 3 : it.model == MSCKF_B200_AID_POSITION ? 0 : -1;
    if (off >= 0)
      for (int i = 0; i < 3; ++i) e->imu[off + i] = it.z[i];
    const int m = rows(it), nz = zlen(it.model);
    dof += m;
    std::vector<double> rec(kRec, NAN);
    rec[0] = it.model; rec[1] = it.a; rec[2] = it.b;
    for (int i = 0; i < nz; ++i) rec[3 + i] = it.z[i];
    for (int i = 0; i < m * m && i < 9; ++i) rec[11 + i] = it.R[i];
    c.last.insert(c.last.end(), rec.begin(), rec.end());
  }
  c.readings_at_last = e->imu_readings;
  return dof;
}
void answer(int dof, int, msckf_b200_aid_result* r) { r->nis = 0.0; r->dx_norm = 0.0; r->dof = dof; r->applied = 1; r->status = 0; }
void answer(int dof, int n, msckf_b200_aid_fde_result* r) {
  *r = msckf_b200_aid_fde_result();
  answer(dof, n, &r->stack);
  for (int k = 0; k < 8; ++k) r->item[k] = {NAN, NAN, k < n ? 0 : -1, -1};
}
template <class Out>
int single(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, const msckf_b200_aid_fde* fde, Out* out) {
  if (!e || !out || !valid(e, items, n)) return MSCKF_B200_ERR_ARG;
  answer(record(e, items, n, fde), n, out);
  g_calls[e].single++;
  return 0;
}
template <class Out>
int batch(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items, const msckf_b200_aid_fde* fde, Out* out) {
  if (!b || !items || !n_items || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0 && !valid(b->es[i], items[i], n_items[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0) { answer(record(b->es[i], items[i], n_items[i], fde), n_items[i], out + i); g_calls[b->es[i]].batch++; }
  g_batch_calls[b]++;
  return 0;
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
  return single(e, items, n_items, nullptr, out);
}
int msckf_b200_batch_aid_stack_update(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                      double chi2_max, msckf_b200_aid_result* out) {
  (void)chi2_max;
  return batch(b, items, n_items, nullptr, out);
}
int msckf_b200_aid_stack_update_fde(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                    const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out) {
  return valid_fde(fde) ? single(e, items, n_items, fde, out) : MSCKF_B200_ERR_ARG;
}
int msckf_b200_batch_aid_stack_update_fde(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                          const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out) {
  return valid_fde(fde) ? batch(b, items, n_items, fde, out) : MSCKF_B200_ERR_ARG;
}
// test hooks: out3 = single calls, batched calls naming e, IMU readings handed over before its last stacked call; fde33 = that
// call's chi2[32], max_exclude (NaN: a call without FDE); rec (cap x 20 doubles) = its items, returns their count; the
// batched calls made on b
int msckf_b200_stub_aid_stack_calls(const msckf_b200_engine* e, long long* out3, double* fde33, double* rec, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out3[0] = c.single; out3[1] = c.batch; out3[2] = c.readings_at_last;
  for (int j = 0; j < kFde; ++j) fde33[j] = j < (int)c.fde.size() ? c.fde[j] : NAN;
  const int n = (int)c.last.size() / kRec;
  for (int k = 0; k < n && k < cap; ++k)
    for (int j = 0; j < kRec; ++j) rec[kRec * k + j] = c.last[kRec * k + j];
  return n;
}
long long msckf_b200_stub_batch_aid_stack_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls[b] : 0; }
// the GNSS class forms on a C view filter handle: which = 0 antennaPositionUpdate(p, v, R, mask), 1 cloneAntennaPositionUpdate
// (state_id, p, v, R, mask), 2 headingUpdate(psi, v, var), 3 cloneHeadingUpdate(state_id, psi, v, var); R is rows x rows
// row-major with rows = R_rows.  -1 with msckf_mono_last_error() for an exception.
int msckf_b200_stub_gnss_class_call(void* h, int which, int state_id, const double* p3, const double* v3, const double* R, int R_rows,
                                    int mask, double psi, double var, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> p, v;
    for (int i = 0; i < 3; ++i) { p(i) = p3[i]; v(i) = v3[i]; }
    msckf_mono::MatrixX<double> Rm(R_rows, R_rows);
    for (int i = 0; i < R_rows; ++i)
      for (int j = 0; j < R_rows; ++j) Rm(i, j) = R[i * R_rows + j];
    return on_filter(h, [&](auto& f) {
      if (which == 0) *out = f.antennaPositionUpdate(p, v, Rm, mask);
      else if (which == 1) *out = f.cloneAntennaPositionUpdate(state_id, p, v, Rm, mask);
      else if (which == 2) *out = f.headingUpdate(psi, v, var);
      else *out = f.cloneHeadingUpdate(state_id, psi, v, var);
      return 0;
    });
  });
}
// the range class forms: which = 0 rangeUpdate(rho, a3, l3, var), 1 cloneRangeUpdate(state_id, rho, a3, l3, var),
// 2 planeRangeUpdate(rho, h, l3, f3, var), 3 clonePlaneRangeUpdate(state_id, rho, h, l3, f3, var).  -1 with
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
