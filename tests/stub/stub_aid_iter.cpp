// tests/stub/stub_aid_iter.cpp -- TEST INFRASTRUCTURE ONLY.
// The iterated stacked aided-update calls of include/msckf_b200.h (msckf_b200_aid_stack_update_iter / _fde_iter and their batch
// forms) for the recording fake tests/stub/stub_engine.cpp, with NO numerics.  Each call checks what the engine checks of its
// arguments besides the items (a NULL iter or iter_out, max_iter outside 0..16, a tol that is not finite and >= 0, 1 to 8 items)
// and records per engine: the single and batched calls, the IMU readings the engine had been handed by the last call, that
// call's max_iter, tol, chi2_max (NaN with FDE), max_exclude (-1 without) and item models.  It answers applied with
// iterations = max(max_iter, 1), converged 1 and step tol / 2.  Linked with stub_engine.cpp, stub_batch_state.cpp, stub_aid.cpp,
// stub_aid_stack.cpp and the C view (filter_capi.cpp, batch_capi.cpp, aid_capi.cpp, aid_stack_capi.cpp, fde_capi.cpp,
// aid_iter_capi.cpp) into tests/stub/libmsckf_aid_iter_view_stub.so by tests/test_aid_iter_cpu.py.  Nothing outside tests/ builds
// or loads it.
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
constexpr int kRec = 13;  // single, batch, readings at the last call, max_iter, tol, chi2_max, max_exclude, n_items, models[5]
struct Calls {
  long long single = 0, batch = 0, readings_at_last = -1;
  double max_iter = NAN, tol = NAN, chi2_max = NAN, max_exclude = NAN;
  std::vector<int> models;
};
std::map<const msckf_b200_engine*, Calls> g_calls;
std::map<const msckf_b200_batch*, long long> g_batch_calls;

bool valid(const msckf_b200_aid_item* items, int n, const msckf_b200_aid_iter* iter) {
  return items && n >= 1 && n <= 8 && iter && iter->max_iter >= 0 && iter->max_iter <= 16 && std::isfinite(iter->tol) && iter->tol >= 0.0;
}
void record(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, double chi2_max, const msckf_b200_aid_fde* fde,
            const msckf_b200_aid_iter* iter) {
  Calls& c = g_calls[e];
  c.readings_at_last = e->imu_readings;
  c.max_iter = iter->max_iter; c.tol = iter->tol;
  c.chi2_max = fde ? NAN : chi2_max;
  c.max_exclude = fde ? fde->max_exclude : -1;
  c.models.assign(n, 0);
  for (int k = 0; k < n; ++k) c.models[k] = items[k].model;
}
void answer(int n, msckf_b200_aid_result* r) { r->nis = 1.0; r->dx_norm = 0.5; r->dof = n; r->applied = 1; r->status = 0; }
void answer(int n, msckf_b200_aid_fde_result* r) {
  *r = msckf_b200_aid_fde_result();
  answer(n, &r->stack);
  for (int k = 0; k < 8; ++k) r->item[k] = {NAN, NAN, k < n ? 0 : -1, -1};
}
void answer(const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* r) {
  r->iterations = iter->max_iter > 1 ? iter->max_iter : 1; r->converged = 1; r->step = iter->tol / 2;
}
template <class Out>
int single(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n, double chi2_max, const msckf_b200_aid_fde* fde,
           const msckf_b200_aid_iter* iter, Out* out, msckf_b200_aid_iter_result* iout) {
  if (!e || !out || !iout || !valid(items, n, iter)) return MSCKF_B200_ERR_ARG;
  record(e, items, n, chi2_max, fde, iter);
  answer(n, out);
  answer(iter, iout);
  g_calls[e].single++;
  return 0;
}
template <class Out>
int batch(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items, double chi2_max, const msckf_b200_aid_fde* fde,
          const msckf_b200_aid_iter* iter, Out* out, msckf_b200_aid_iter_result* iout) {
  if (!b || !items || !n_items || !iter || !out || !iout) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0 && !valid(items[i], n_items[i], iter + i)) return MSCKF_B200_ERR_ARG;
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_items[i] != 0) {
      record(b->es[i], items[i], n_items[i], chi2_max, fde, iter + i);
      answer(n_items[i], out + i);
      answer(iter + i, iout + i);
      g_calls[b->es[i]].batch++;
    }
  g_batch_calls[b]++;
  return 0;
}
}  // namespace

extern "C" {
int msckf_b200_aid_stack_update_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                     const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out, msckf_b200_aid_iter_result* iter_out) {
  return single(e, items, n_items, chi2_max, nullptr, iter, out, iter_out);
}
int msckf_b200_aid_stack_update_fde_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                         const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                         msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out) {
  return fde ? single(e, items, n_items, 0.0, fde, iter, out, iter_out) : MSCKF_B200_ERR_ARG;
}
int msckf_b200_batch_aid_stack_update_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                           double chi2_max, const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out,
                                           msckf_b200_aid_iter_result* iter_out) {
  return batch(b, items, n_items, chi2_max, nullptr, iter, out, iter_out);
}
int msckf_b200_batch_aid_stack_update_fde_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                               const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                               msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out) {
  return fde ? batch(b, items, n_items, 0.0, fde, iter, out, iter_out) : MSCKF_B200_ERR_ARG;
}
// test hooks: rec (kRec doubles) = single and batched calls naming e, the IMU readings handed over before its last iterated
// call, that call's max_iter, tol, chi2_max (NaN: FDE), max_exclude (-1: no FDE), item count and first 5 item models; the
// batched iterated calls made on b
void msckf_b200_stub_aid_iter_calls(const msckf_b200_engine* e, double* rec) {
  const Calls c = g_calls.count(e) ? g_calls.at(e) : Calls();
  const double v[8] = {(double)c.single, (double)c.batch, (double)c.readings_at_last, c.max_iter, c.tol, c.chi2_max, c.max_exclude,
                       (double)c.models.size()};
  for (int j = 0; j < kRec; ++j) rec[j] = j < 8 ? v[j] : (j - 8 < (int)c.models.size() ? c.models[j - 8] : NAN);
}
long long msckf_b200_stub_batch_aid_iter_calls(const msckf_b200_batch* b) { return g_batch_calls.count(b) ? g_batch_calls.at(b) : 0; }
}
