// tests/stub/stub_batch_state.cpp -- TEST INFRASTRUCTURE ONLY.
// The batched state calls of include/msckf_b200.h (msckf_b200_batch_propagate_n / _augment / _prune / _get_state) for the
// recording fake of the C-ABI (tests/stub/stub.hpp), with NO numerics: each validates every member first, then forwards to
// the fake's single-engine calls, and records one call per batched operation.  Nothing outside tests/ builds or loads it.
#include "stub.hpp"

using stub::fail;

namespace {
std::map<const msckf_b200_batch*, std::vector<long long>> g_calls;  // per batch: propagate_n, augment, prune, get_state
void record(const msckf_b200_batch* b, int op) {
  auto& c = g_calls[b];
  c.resize(4, 0);
  c[op]++;
}
}  // namespace

extern "C" {
int msckf_b200_batch_propagate_n(msckf_b200_batch* b, const void* const* readings, const int* k) {
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k && (k[i] < 0 || (k[i] > 0 && (!readings || !readings[i])))) return fail(MSCKF_B200_ERR_ARG, "stub: bad readings");
  for (size_t i = 0; i < b->es.size(); ++i)
    if (k && k[i] > 0) msckf_b200_propagate_n(b->es[i], readings[i], k[i]);
  record(b, 0);
  return 0;
}
int msckf_b200_batch_augment(msckf_b200_batch* b, const int* which) {
  for (size_t i = 0; i < b->es.size(); ++i)
    if ((!which || which[i]) && msckf_b200_num_clones(b->es[i]) >= 192) return fail(MSCKF_B200_ERR_CAPACITY, "stub: window above the engine's hard limit");
  for (size_t i = 0; i < b->es.size(); ++i)
    if (!which || which[i]) msckf_b200_augment(b->es[i]);
  record(b, 1);
  return 0;
}
int msckf_b200_batch_prune(msckf_b200_batch* b, const int* const* keep, const int* n_keep) {
  if (!n_keep) return fail(MSCKF_B200_ERR_ARG, "stub: null n_keep");
  for (size_t i = 0; i < b->es.size(); ++i) {
    const int M = msckf_b200_num_clones(b->es[i]), n = n_keep[i];
    if (n < 0 || n == M) continue;
    if (n > M || (n > 0 && (!keep || !keep[i]))) return fail(MSCKF_B200_ERR_ARG, "stub: bad keep list");
    for (int j = 0; j < n; ++j)
      if (keep[i][j] < 0 || keep[i][j] >= M || (j && keep[i][j] <= keep[i][j - 1])) return fail(MSCKF_B200_ERR_ARG, "stub: keep[] must be ascending positions");
  }
  for (size_t i = 0; i < b->es.size(); ++i)
    if (n_keep[i] >= 0 && n_keep[i] != msckf_b200_num_clones(b->es[i])) msckf_b200_prune(b->es[i], n_keep[i] ? keep[i] : nullptr, n_keep[i]);
  record(b, 2);
  return 0;
}
int msckf_b200_batch_get_state(msckf_b200_batch* b, void* const* imu, void* const* poses) {
  for (size_t i = 0; i < b->es.size(); ++i) msckf_b200_get_state(b->es[i], imu ? imu[i] : nullptr, poses ? poses[i] : nullptr);
  record(b, 3);
  return 0;
}
// test hook: the batched calls recorded for b so far (propagate_n, augment, prune, get_state)
void msckf_b200_stub_batch_calls(const msckf_b200_batch* b, long long* out) {
  auto it = g_calls.find(b);
  for (int i = 0; i < 4; ++i) out[i] = it == g_calls.end() || it->second.empty() ? 0 : it->second[i];
}
}
