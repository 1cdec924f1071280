// msckf_mono_b200/csrc/filter_view.hpp -- what the two translation units of the C view (include/msckf_mono_c.h) share:
// filter_capi.cpp (one filter, msckf_mono::MSCKF<_S>), batch_capi.cpp (device batches, msckf_mono::MSCKFBatch<_S>),
// nees_capi.cpp (consistency against ground truth, msckf_mono_nees / _batch_nees), aid_capi.cpp (aided measurement
// updates, msckf_mono_aid_update / _batch_aid_update) and landmark_capi.cpp (mapped landmarks, msckf_mono_landmark_update /
// _batch_landmark_update).
#pragma once
#include <cstdint>
#include <exception>
#include <string>
#include <msckf_b200.h>
#include <msckf_mono/msckf.h>

namespace msckf_view {
extern thread_local std::string g_err;  // msckf_mono_last_error()

// a C view handle: MSCKF<float> or MSCKF<double> behind one interface
struct Base {
  virtual ~Base() {}
  virtual void set_engine_options(int, int, int, int) = 0;
  virtual void initialize(const double*, const double*, const double*, const double*) = 0;
  virtual void propagate(const double*) = 0;
  virtual void augment(int, double) = 0;
  virtual void update(const double*, const uint64_t*, int) = 0;
  virtual void add(const double*, const uint64_t*, int) = 0;
  virtual void marginalize() = 0;
  virtual void marginalize_launch() = 0;
  virtual void marginalize_collect() = 0;
  virtual void prune_redundant() = 0;
  virtual void prune_empty() = 0;
  virtual void finish() = 0;
  virtual int num_cam() = 0;
  virtual void imu_state(double*) = 0;
  virtual void cam_states(double*, int*, double*) = 0;
  virtual int cam_tracked(int, uint64_t*, int) = 0;
  virtual int covariance(double*) = 0;
  virtual int map(double*, int) = 0;
  virtual int pruned(double*, int*, int) = 0;
  virtual int tracked_ids(uint64_t*, int) = 0;
  virtual int report(int*, double*, double*, int) = 0;
  virtual int queued(uint64_t*, int*, int) = 0;
  virtual int pack_queued(int*, double*, int*, int, int) = 0;
  virtual msckf_b200_engine* engine() = 0;
  virtual void* filter_ptr() = 0;
  virtual int last_m() = 0;
  virtual int last_rank() = 0;
  int dtype = 0;
};

// a persistent device batch over n filters of one scalar type (msckf_mono::MSCKFBatch<_S>): a msckf_mono_batch_* handle
struct ViewBatch {
  int dtype = 0;
  msckf_mono::MSCKFBatch<float>* bf = nullptr;
  msckf_mono::MSCKFBatch<double>* bd = nullptr;
  ~ViewBatch() { delete bf; delete bd; }
};

// runs fn(), turning an exception into -1 and its message into msckf_mono_last_error()
template <class F>
int guard(F&& fn) {
  try {
    return fn();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}
}  // namespace msckf_view
