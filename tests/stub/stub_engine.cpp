// tests/stub/stub_engine.cpp -- TEST INFRASTRUCTURE ONLY.
// The single-engine calls of the recording fake of the C-ABI of include/msckf_b200.h, with NO numerics: it counts clones,
// remembers the last batch and fabricates a report in which every track is valid and accepted.  With the other
// tests/stub/stub_*.cpp it lets the CPU tests (-m "not gpu") drive the drop-in class shim (include/msckf_mono/msckf.h) and
// compare its INTEGER bookkeeping -- track lists, clone ids, last_correlated_id, queued tracks, pruneEmptyStates -- with the
// oracle on a box without a GPU.  It is not a CPU fallback: it never computes a state, a covariance or a residual, and nothing
// outside tests/ builds or loads it (tests/fake_engine.py does).
#include "stub.hpp"

#include <cstring>
#include <string>

static thread_local std::string g_err;
int stub::fail(int code, const char* msg) { g_err = msg; return code; }
using stub::fail;
static stub::Records<> g_jac;  // msckf_b200_jac_group per engine, msckf_b200_batch_jac_occupancy per batch
template <class T> static void put(void* p, size_t i, double v, int dtype) {
  (void)sizeof(T);
  if (dtype == MSCKF_B200_F32) ((float*)p)[i] = (float)v; else ((double*)p)[i] = v;
}

extern "C" {
int msckf_b200_create(const msckf_b200_config* cfg, msckf_b200_engine** out) {
  if (!cfg || !out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  auto* e = new msckf_b200_engine();
  e->dtype = cfg->dtype; e->max_clones = cfg->max_clones;
  *out = e;
  return 0;
}
int msckf_b200_destroy(msckf_b200_engine* e) { delete e; return 0; }
int msckf_b200_initialize(msckf_b200_engine* e, const void*, const void*, const void*, const void* imu) {
  for (int i = 0; i < 19; ++i) e->imu[i] = e->dtype == MSCKF_B200_F32 ? (double)((const float*)imu)[i] : ((const double*)imu)[i];
  e->M = 0;
  return 0;
}
int msckf_b200_propagate(msckf_b200_engine* e, const void*) { e->imu_readings++; return 0; }
int msckf_b200_propagate_n(msckf_b200_engine* e, const void*, int k) { e->imu_readings += k; return 0; }
int msckf_b200_input_buffer(msckf_b200_engine* e, int n_tracks, int n_obs, msckf_b200_tracks* out) {
  e->buf_off.assign(n_tracks + 1, 0); e->buf_idx.assign(n_obs + 1, 0); e->buf_obs.assign(2 * n_obs + 2, 0.0); e->buf_pfg.assign(3 * n_tracks + 3, 0.0);
  out->n_tracks = n_tracks; out->obs_offset = e->buf_off.data(); out->clone_index = e->buf_idx.data();
  out->obs = e->buf_obs.data(); out->p_f_G = e->buf_pfg.data();
  return 0;
}
int msckf_b200_augment(msckf_b200_engine* e) {
  if (e->M >= 192) return fail(MSCKF_B200_ERR_CAPACITY, "stub: window above the engine's hard limit");  // (capacities grow on demand)
  e->M++;
  return 0;
}
int msckf_b200_stage(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tr) {
  if (e->pending) return fail(MSCKF_B200_ERR_STATE, "stub: previous update not fetched");
  e->last_len.clear();
  if (tr->n_tracks > 0 && tr->obs_offset[0] != 0) return fail(MSCKF_B200_ERR_ARG, "stub: obs_offset[0] must be 0");
  for (int t = 0; t < tr->n_tracks; ++t) {
    const int L = tr->obs_offset[t + 1] - tr->obs_offset[t];
    if (L < 1 || L > 98) return fail(MSCKF_B200_ERR_ARG, "stub: bad track length");
    for (int o = tr->obs_offset[t]; o < tr->obs_offset[t + 1]; ++o) {
      if (tr->clone_index[o] < 0 || tr->clone_index[o] >= e->M) return fail(MSCKF_B200_ERR_ARG, "stub: clone_index out of range");
      for (int q = tr->obs_offset[t]; q < o; ++q)
        if (tr->clone_index[q] == tr->clone_index[o]) return fail(MSCKF_B200_ERR_ARG, "stub: a track names one clone twice");
    }
    e->last_len.push_back(L);
  }
  e->mode = mode;
  return 0;
}
int msckf_b200_launch(msckf_b200_engine* e) { e->pending = 1; e->launches++; return 0; }
int msckf_b200_launch_timed(msckf_b200_engine* e, float* ms) { if (ms) *ms = 0; return msckf_b200_launch(e); }
int msckf_b200_update_async(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tr) {
  int rc = msckf_b200_stage(e, mode, tr);
  return rc ? rc : msckf_b200_launch(e);
}
int msckf_b200_fetch(msckf_b200_engine* e, msckf_b200_report* rep) {
  if (!e->pending) return fail(MSCKF_B200_ERR_STATE, "stub: fetch without a pending update");
  e->pending = 0;
  if (!rep) return 0;
  int m = 0;
  for (size_t t = 0; t < e->last_len.size(); ++t) {
    if (rep->cm_ok) rep->cm_ok[t] = 1;
    if (rep->tri_ok) rep->tri_ok[t] = 1;
    if (rep->valid) rep->valid[t] = 1;
    if (rep->accepted) rep->accepted[t] = 1;
    if (rep->gamma) put<double>(rep->gamma, t, 0.0, e->dtype);
    if (rep->p_f_G) for (int k = 0; k < 3; ++k) put<double>(rep->p_f_G, 3 * t + k, k == 2 ? 5.0 : (double)t, e->dtype);
    m += 2 * e->last_len[t] - 3;
  }
  rep->m = m;
  rep->rank = m;
  if (m > 0) e->updates++;
  return 0;
}
int msckf_b200_update(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tr, msckf_b200_report* rep) {
  int rc = msckf_b200_update_async(e, mode, tr);
  return rc ? rc : msckf_b200_fetch(e, rep);
}
int msckf_b200_update_batch(msckf_b200_engine** es, int n, int mode, const msckf_b200_tracks* tr, msckf_b200_report* reps, int) {
  for (int i = 0; i < n; ++i) { int rc = msckf_b200_update(es[i], mode, &tr[i], reps ? &reps[i] : nullptr); if (rc) return rc; }
  return 0;
}
int msckf_b200_batch_create(msckf_b200_engine** es, int n, msckf_b200_batch** out) { auto* b = new msckf_b200_batch(); b->es.assign(es, es + n); *out = b; return 0; }
int msckf_b200_batch_destroy(msckf_b200_batch* b) { delete b; return 0; }
int msckf_b200_batch_stage(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tr, int) {
  for (size_t i = 0; i < b->es.size(); ++i) { int rc = msckf_b200_stage(b->es[i], mode, &tr[i]); if (rc) return rc; }
  return 0;
}
int msckf_b200_batch_launch(msckf_b200_batch* b) { for (auto* e : b->es) msckf_b200_launch(e); b->launches++; return 0; }
int msckf_b200_batch_launch_timed(msckf_b200_batch* b, float* ms) { if (ms) *ms = 0; return msckf_b200_batch_launch(b); }
int msckf_b200_batch_update_async(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tr, int t) {
  int rc = msckf_b200_batch_stage(b, mode, tr, t);
  return rc ? rc : msckf_b200_batch_launch(b);
}
int msckf_b200_batch_fetch(msckf_b200_batch* b, msckf_b200_report* reps) {
  for (size_t i = 0; i < b->es.size(); ++i) { int rc = msckf_b200_fetch(b->es[i], reps ? &reps[i] : nullptr); if (rc) return rc; }
  return 0;
}
int msckf_b200_batch_update(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tr, msckf_b200_report* reps, int t) {
  int rc = msckf_b200_batch_update_async(b, mode, tr, t);
  return rc ? rc : msckf_b200_batch_fetch(b, reps);
}
int msckf_b200_batch_kernel_times(msckf_b200_batch*, float*, const char**, int) { return 0; }
long long msckf_b200_batch_launch_count(const msckf_b200_batch* b) { return b->launches; }
void* msckf_b200_batch_stream(msckf_b200_batch*) { return nullptr; }
// no kernel ever runs: both answer "before the first launch"
int msckf_b200_batch_jac_occupancy(const msckf_b200_batch* b) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "stub: null batch");
  g_jac.batch[b]++;
  return 0;
}
int msckf_b200_jac_group(msckf_b200_engine* e) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "stub: null engine");
  g_jac.last(e).single++;
  return 0;
}
int msckf_b200_kernel_times(msckf_b200_engine*, float*, const char**, int) { return 0; }
int msckf_b200_tail_profile(msckf_b200_engine*, unsigned long long*, int) { return 0; }
int msckf_b200_prune(msckf_b200_engine* e, const int* keep, int n_keep) {
  for (int i = 0; i < n_keep; ++i)
    if (keep[i] < 0 || keep[i] >= e->M || (i && keep[i] <= keep[i - 1])) return fail(MSCKF_B200_ERR_ARG, "stub: keep[] must be ascending positions");
  e->M = n_keep;
  return 0;
}
int msckf_b200_num_clones(msckf_b200_engine* e) { return e->M; }
int msckf_b200_get_state(msckf_b200_engine* e, void* imu, void* poses) {
  if (imu) {
    for (int i = 0; i < 19; ++i) put<double>(imu, i, e->imu[i], e->dtype);
    for (int i = 0; i < 3; ++i) { put<double>(imu, 19 + i, e->imu[i], e->dtype); put<double>(imu, 22 + i, e->imu[3 + i], e->dtype); }
    for (int i = 0; i < 4; ++i) put<double>(imu, 25 + i, e->imu[15 + i], e->dtype);
  }
  if (poses)
    for (int k = 0; k < e->M; ++k)
      for (int i = 0; i < 7; ++i) put<double>(poses, 7 * k + i, i == 6 ? 1.0 : 0.0, e->dtype);  // p = 0, q = (0,0,0,1)
  return 0;
}
int msckf_b200_get_covariance(msckf_b200_engine* e, void* out) {
  const int n = 15 + 6 * e->M;
  std::memset(out, 0, (size_t)n * n * (e->dtype == MSCKF_B200_F32 ? 4 : 8));
  return n;
}
int msckf_b200_set_covariance(msckf_b200_engine*, const void*) { return 0; }
int msckf_b200_get_counters(msckf_b200_engine* e, long long* c) { for (int i = 0; i < 8; ++i) c[i] = 0; c[3] = e->updates; return 0; }
int msckf_b200_last_delta_x(msckf_b200_engine* e, double* out, int cap) {
  const int n = 15 + 6 * e->M;
  for (int i = 0; i < n && i < cap; ++i) out[i] = 0.0;
  return n;
}
int msckf_b200_rank_pivots(msckf_b200_engine* e, double* out, int cap) {
  const int n = 15 + 6 * e->M;
  for (int i = 0; i < n && i < cap; ++i) out[i] = 1.0;
  return n;
}
int msckf_b200_set_option(msckf_b200_engine*, int, double) { return 0; }
int msckf_b200_stage_buffer(msckf_b200_engine*, int, void*, int) { return 0; }  // (no update buffers: none recorded)
int msckf_b200_copy_state(msckf_b200_engine* dst, const msckf_b200_engine* src) { *dst = *src; return 0; }
long long msckf_b200_launch_count(const msckf_b200_engine* e) { return e->launches; }
void* msckf_b200_stream(msckf_b200_engine*) { return nullptr; }
int msckf_b200_synchronize(msckf_b200_engine*) { return 0; }
const char* msckf_b200_last_error(void) { return g_err.c_str(); }
// test hook: out2 = msckf_b200_jac_group calls on e, msckf_b200_batch_jac_occupancy calls on b
void msckf_b200_stub_jac_calls(const msckf_b200_engine* e, const msckf_b200_batch* b, long long* out2) {
  out2[0] = g_jac.of(e).single; out2[1] = g_jac.of(b);
}
}
