// tests/stub/stub_aid_fde.cpp -- TEST INFRASTRUCTURE ONLY.
// The stacked aided update with fault detection and exclusion of include/msckf_b200.h (msckf_b200_aid_stack_update_fde /
// _batch_aid_stack_update_fde) for the recording fake tests/stub/stub_engine.cpp, with NO numerics: each call records, per
// engine, its fde (chi2[32], max_exclude) and every item in full -- model, a, b, z (8 doubles, NaN past the model's length) and R
// (rows x rows, then NaN) -- and answers outcome 0 with every item used, so that a test can see exactly what the class forms
// (MSCKF::aidedUpdate(items, fde), MSCKFBatch::aidedUpdate(items, fde)) and the C view (fde_capi.cpp) send.  Linked with
// stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp, stub_range_stack.cpp and the C view into
// tests/stub/libmsckf_fde_view_stub.so by tests/test_aid_fde_cpu.py.  Nothing outside tests/ builds or loads it.
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
constexpr int kRec = 20;  // per recorded item: model, a, b, z[8], R[9]
struct Calls {
  long long single = 0, batch = 0;
  std::vector<double> fde;   // chi2[32], max_exclude of the last call
  std::vector<double> last;  // the items of the last call
};
std::map<const msckf_b200_engine*, Calls> g_calls;
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
bool valid(const msckf_b200_aid_item* items, int n, const msckf_b200_aid_fde* fde) {
  if (n < 1 || n > 8 || !items || !fde || fde->max_exclude < 0 || fde->max_exclude > 7) return false;
  for (int d = 0; d < 32; ++d)
    if (!(std::isfinite(fde->chi2[d]) && fde->chi2[d] > 0.0)) return false;
  for (int k = 0; k < n; ++k)
    if (items[k].model < 0 || items[k].model > MSCKF_B200_AID_CLONE_PLANE_RANGE || items[k].model == MSCKF_B200_AID_LINEAR ||
        !items[k].z || !items[k].R)
      return false;
  return true;
}
void apply(const msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* r) {
  Calls& c = g_calls[e];
  c.last.clear();
  c.fde.assign(fde->chi2, fde->chi2 + 32);
  c.fde.push_back(fde->max_exclude);
  *r = msckf_b200_aid_fde_result();
  r->stack.applied = 1;
  for (int k = 0; k < 8; ++k) r->item[k] = {NAN, NAN, k < n ? 0 : -1, -1};
  for (int k = 0; k < n; ++k) {
    const msckf_b200_aid_item& it = items[k];
    const int m = rows(it), nz = zlen(it.model);
    r->stack.dof += m;
    std::vector<double> rec(kRec, NAN);
    rec[0] = it.model; rec[1] = it.a; rec[2] = it.b;
    for (int i = 0; i < nz; ++i) rec[3 + i] = it.z[i];
    for (int i = 0; i < m * m && i < 9; ++i) rec[11 + i] = it.R[i];
    c.last.insert(c.last.end(), rec.begin(), rec.end());
  }
}
}  // namespace

extern "C" {
int msckf_b200_aid_stack_update_fde(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                    const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out) {
  if (!e || !out || !valid(items, n_items, fde)) return MSCKF_B200_ERR_ARG;
  apply(e, items, n_items, fde, out);
  g_calls[e].single++;
  return 0;
}
int msckf_b200_batch_aid_stack_update_fde(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                          const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out) {
  if (!b || !items || !n_items || !out) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0 && !valid(items[i], n_items[i], fde)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0) { apply(b->es[i], items[i], n_items[i], fde, out + i); g_calls[b->es[i]].batch++; }
  return 0;
}
// test hook: out2 = single calls, batched calls naming e; fde33 = the last call's chi2[32], max_exclude; rec (cap x 20 doubles)
// = its items; returns their count
int msckf_b200_stub_fde_calls(const msckf_b200_engine* e, long long* out2, double* fde33, double* rec, int cap) {
  const Calls c = g_calls.count(e) ? g_calls[e] : Calls();
  out2[0] = c.single; out2[1] = c.batch;
  for (size_t j = 0; j < c.fde.size(); ++j) fde33[j] = c.fde[j];
  const int n = (int)c.last.size() / kRec;
  for (int k = 0; k < n && k < cap; ++k)
    for (int j = 0; j < kRec; ++j) rec[kRec * k + j] = c.last[kRec * k + j];
  return n;
}
}
