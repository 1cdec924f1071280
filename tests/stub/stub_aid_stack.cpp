// tests/stub/stub_aid_stack.cpp -- TEST INFRASTRUCTURE ONLY.
// The stacked aided-update calls of include/msckf_b200.h (msckf_b200_aid_stack_update / _batch_aid_stack_update and their
// fault detection and exclusion forms, _fde) for the recording fake of the C-ABI (tests/stub/stub.hpp), with NO numerics.  Each
// call's items are checked as the engine checks them (every stack model, the at-rest ones included; for _fde also the
// thresholds and max_exclude) and recorded per engine: the single and batched calls, the IMU readings the engine had been
// handed by the last call, that call's fde (chi2[32], max_exclude) and its items in full -- model, a, b, z (8 doubles, NaN past
// the model's length) and R (rows x rows, then NaN) -- so that a test can see exactly what the class forms and the C view send.
// A VELOCITY or POSITION item copies z into the fake's IMU state (so that a caller can see whether its host mirror was
// refreshed); every other item changes nothing, and the _fde forms answer outcome 0 with every item used.  Nothing outside
// tests/ builds or loads it.
#include "stub.hpp"

#include <cmath>

namespace {
constexpr int kRec = 20;  // per recorded item: model, a, b, z[8], R[9]
constexpr int kFde = 33;  // chi2[32], max_exclude
struct Calls : stub::Calls {
  std::vector<double> fde;   // of the last call (NaN: a call without FDE)
  std::vector<double> last;  // the items of the last call
};
stub::Records<Calls> g_calls;
int popc(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1); }
int rows(const msckf_b200_aid_item& it) {
  switch (it.model) {
    case MSCKF_B200_AID_VELOCITY: case MSCKF_B200_AID_POSITION: return 3;
    case MSCKF_B200_AID_BODY_VELOCITY: case MSCKF_B200_AID_ANTENNA_POSITION: return popc(it.a);
    case MSCKF_B200_AID_CLONE_ANTENNA_POSITION: return popc(it.b);
    case MSCKF_B200_AID_HEADING: case MSCKF_B200_AID_CLONE_HEADING:
    case MSCKF_B200_AID_RANGE: case MSCKF_B200_AID_CLONE_RANGE:
    case MSCKF_B200_AID_PLANE_RANGE: case MSCKF_B200_AID_CLONE_PLANE_RANGE: return 1;
    case MSCKF_B200_AID_GYRO_AT_REST: case MSCKF_B200_AID_ACCEL_AT_REST: return 3;
    default: return 6;
  }
}
int zlen(int model) {
  switch (model) {
    case MSCKF_B200_AID_VELOCITY: case MSCKF_B200_AID_POSITION: case MSCKF_B200_AID_BODY_VELOCITY:
    case MSCKF_B200_AID_GYRO_AT_REST: case MSCKF_B200_AID_ACCEL_AT_REST: return 3;
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
    if (it.model < 0 || it.model > MSCKF_B200_AID_ACCEL_AT_REST || it.model == MSCKF_B200_AID_LINEAR || !it.z || !it.R) return false;
    const bool clone = it.model == MSCKF_B200_AID_CLONE_POSE || it.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION ||
                       it.model == MSCKF_B200_AID_CLONE_HEADING || it.model == MSCKF_B200_AID_RELATIVE_POSE ||
                       it.model == MSCKF_B200_AID_CLONE_RANGE || it.model == MSCKF_B200_AID_CLONE_PLANE_RANGE;
    if (clone && (it.a < 0 || it.a >= e->M)) return false;
    if (it.model == MSCKF_B200_AID_RELATIVE_POSE && (it.b < 0 || it.b >= e->M || it.a == it.b)) return false;
    if ((it.model == MSCKF_B200_AID_BODY_VELOCITY || it.model == MSCKF_B200_AID_ANTENNA_POSITION) && (it.a < 1 || it.a > 7)) return false;
    if (it.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION && (it.b < 1 || it.b > 7)) return false;
    const bool at_rest = it.model == MSCKF_B200_AID_GYRO_AT_REST || it.model == MSCKF_B200_AID_ACCEL_AT_REST;
    if (at_rest && (it.a != 0 || it.b != 0)) return false;
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
  Calls& c = g_calls.last(e);
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
  g_calls.engine[e].single++;
  return 0;
}
template <class Out>
int batch(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items, const msckf_b200_aid_fde* fde, Out* out) {
  if (!b || !items || !n_items || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0 && !valid(b->es[i], items[i], n_items[i])) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0) { answer(record(b->es[i], items[i], n_items[i], fde), n_items[i], out + i); g_calls.engine[b->es[i]].batch++; }
  g_calls.batch[b]++;
  return 0;
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
  const Calls c = g_calls.of(e);
  g_calls.counts(e, out3);
  for (int j = 0; j < kFde; ++j) fde33[j] = j < (int)c.fde.size() ? c.fde[j] : NAN;
  const int n = (int)c.last.size() / kRec;
  for (int k = 0; k < n && k < cap; ++k)
    for (int j = 0; j < kRec; ++j) rec[kRec * k + j] = c.last[kRec * k + j];
  return n;
}
long long msckf_b200_stub_batch_aid_stack_calls(const msckf_b200_batch* b) { return g_calls.of(b); }
}
