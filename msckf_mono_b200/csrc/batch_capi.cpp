// msckf_mono_b200/csrc/batch_capi.cpp -- device batches in the C view (include/msckf_mono_c.h, msckf_mono_batch_*):
// msckf_mono::MSCKFBatch<float|double> over filters created by filter_capi.cpp.  Host code only; links against the engine
// C-ABI, batched entry points (msckf_b200_batch_*) included.
#include <stdexcept>
#include <string>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
template <class S>
void batch_propagate(MSCKFBatch<S>& b, int member, const double* m) {
  imuReading<S> r;
  for (int i = 0; i < 3; ++i) { r.omega(i) = (S)m[i]; r.a(i) = (S)m[3 + i]; }
  r.dT = (S)m[6];
  b.propagate((size_t)member, r);
}
template <class S>
void batch_augment(MSCKFBatch<S>& b, const int* state_ids, const double* times) {
  std::vector<S> t(b.size());
  for (size_t i = 0; i < t.size(); ++i) t[i] = (S)times[i];
  b.augmentState(std::vector<int>(state_ids, state_ids + b.size()), t);
}
// fn(batch) on the batch of the view's scalar type
template <class F>
int on_batch(void* b, F&& fn) {
  return guard([&] {
    auto* vb = static_cast<ViewBatch*>(b);
    if (vb->bf) fn(*vb->bf); else fn(*vb->bd);
    return 0;
  });
}
}  // namespace

extern "C" {
int msckf_mono_batch_create(void** handles, int n, int threads, void** out) {
  return guard([&] {
    if (n <= 0 || !handles || !out) throw std::runtime_error("batch_create: bad arguments");
    const int dtype = static_cast<Base*>(handles[0])->dtype;
    auto* vb = new ViewBatch();
    vb->dtype = dtype;
    try {
      if (dtype == 0) {
        std::vector<MSCKF<float>*> fs;
        for (int i = 0; i < n; ++i) { Base* b = static_cast<Base*>(handles[i]); if (b->dtype != dtype) throw std::runtime_error("batch_create: mixed scalar types"); fs.push_back(static_cast<MSCKF<float>*>(b->filter_ptr())); }
        vb->bf = new MSCKFBatch<float>(fs, threads);
      } else {
        std::vector<MSCKF<double>*> fs;
        for (int i = 0; i < n; ++i) { Base* b = static_cast<Base*>(handles[i]); if (b->dtype != dtype) throw std::runtime_error("batch_create: mixed scalar types"); fs.push_back(static_cast<MSCKF<double>*>(b->filter_ptr())); }
        vb->bd = new MSCKFBatch<double>(fs, threads);
      }
    } catch (...) { delete vb; throw; }
    *out = vb;
    return 0;
  });
}
void msckf_mono_batch_destroy(void* b) { delete static_cast<ViewBatch*>(b); }
int msckf_mono_batch_propagate(void* b, int member, const double* m) {
  return on_batch(b, [&](auto& bb) {
    if (member < 0 || member >= (int)bb.size()) throw std::out_of_range("batch_propagate: member index");
    batch_propagate(bb, member, m);
  });
}
int msckf_mono_batch_augment_state(void* b, const int* state_ids, const double* times) {
  return on_batch(b, [&](auto& bb) { batch_augment(bb, state_ids, times); });
}
int msckf_mono_batch_marginalize(void* b) { return on_batch(b, [](auto& bb) { bb.marginalize(); }); }
int msckf_mono_batch_prune_empty_states(void* b) { return on_batch(b, [](auto& bb) { bb.pruneEmptyStates(); }); }
int msckf_mono_batch_prune_redundant_states(void* b) { return on_batch(b, [](auto& bb) { bb.pruneRedundantStates(); }); }
int msckf_mono_batch_finish(void* b) { return on_batch(b, [](auto& bb) { bb.finish(); }); }
int msckf_mono_batch_refresh_state(void* b) { return on_batch(b, [](auto& bb) { bb.refreshState(); }); }
void* msckf_mono_batch_handle(void* b) {
  auto* vb = static_cast<ViewBatch*>(b);
  return vb->bf ? (void*)vb->bf->handle() : (void*)vb->bd->handle();
}
// one-shot form: a temporary batch around one marginalize() of every filter
int msckf_mono_marginalize_batch(void** handles, int n, int threads) {
  if (n <= 0) return 0;
  void* b = nullptr;
  int rc = msckf_mono_batch_create(handles, n, threads, &b);
  if (rc != 0) return rc;
  rc = msckf_mono_batch_marginalize(b);
  const std::string keep = g_err;
  msckf_mono_batch_destroy(b);
  g_err = keep;
  return rc;
}
}
