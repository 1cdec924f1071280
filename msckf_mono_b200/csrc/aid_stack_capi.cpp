// msckf_mono_b200/csrc/aid_stack_capi.cpp -- stacked aided updates (odometry) in the C view (include/msckf_mono_c.h,
// msckf_mono_aid_stack_update / _batch_aid_stack_update / _body_velocity_update / _relative_pose_update): MSCKF<_S>::aidedUpdate
// (items), bodyVelocityUpdate, relativePoseUpdate and MSCKFBatch<_S>::aidedUpdate(items) over handles created by filter_capi.cpp
// and batch_capi.cpp.  Host code only; its own translation unit, so that the other view files link against a C-ABI without
// msckf_b200_aid_stack_update / msckf_b200_batch_aid_stack_update.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
template <class S>
void batch_stack(MSCKFBatch<S>& b, const int* n_items, const msckf_b200_aid_item* items, double chi2_max, msckf_b200_aid_result* out) {
  std::vector<std::vector<msckf_b200_aid_item>> it(b.size());
  for (size_t i = 0, o = 0; i < b.size(); o += n_items[i], ++i) {
    if (n_items[i] < 0) throw std::invalid_argument("batch_aid_stack_update: negative item count");
    it[i].assign(items + o, items + o + n_items[i]);
  }
  const std::vector<msckf_b200_aid_result> r = b.aidedUpdate(it, chi2_max);
  for (size_t i = 0; i < r.size(); ++i)
    if (n_items[i] > 0) out[i] = r[i];
}
template <class F>
int on_filter(void* h, F&& f) {
  Base* b = static_cast<Base*>(h);
  if (b->dtype == 0) return f(*static_cast<MSCKF<float>*>(b->filter_ptr()));
  return f(*static_cast<MSCKF<double>*>(b->filter_ptr()));
}
}  // namespace

extern "C" {
int msckf_mono_aid_stack_update(void* h, const msckf_b200_aid_item* items, int n_items, double chi2_max, msckf_b200_aid_result* out) {
  return guard([&] {
    if (!h || !out || n_items < 0 || (n_items > 0 && !items)) throw std::invalid_argument("aid_stack_update: null argument");
    const std::vector<msckf_b200_aid_item> it(items, items + n_items);
    return on_filter(h, [&](auto& f) { *out = f.aidedUpdate(it, chi2_max); return 0; });
  });
}
int msckf_mono_batch_aid_stack_update(void* batch, const int* n_items, const msckf_b200_aid_item* items, double chi2_max,
                                      msckf_b200_aid_result* out) {
  return guard([&] {
    if (!batch || !n_items || !out) throw std::invalid_argument("batch_aid_stack_update: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_stack(*vb->bf, n_items, items, chi2_max, out);
    else batch_stack(*vb->bd, n_items, items, chi2_max, out);
    return 0;
  });
}
int msckf_mono_body_velocity_update(void* h, const double* v3, int mask, const double* R, double chi2_max, msckf_b200_aid_result* out) {
  return guard([&] {
    if (!h || !v3 || !R || !out) throw std::invalid_argument("body_velocity_update: null argument");
    const int m = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);
    MatrixX<double> Rm(m, m);
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < m; ++j) Rm(i, j) = R[i * m + j];
    Vector3<double> v;
    for (int i = 0; i < 3; ++i) v(i) = v3[i];
    return on_filter(h, [&](auto& f) { *out = f.bodyVelocityUpdate(v, Rm, mask, chi2_max); return 0; });
  });
}
int msckf_mono_relative_pose_update(void* h, int state_id_a, int state_id_b, const double* p3, const double* q4, const double* R36,
                                    double chi2_max, msckf_b200_aid_result* out) {
  return guard([&] {
    if (!h || !p3 || !q4 || !R36 || !out) throw std::invalid_argument("relative_pose_update: null argument");
    FixedMatrix<double, 6, 6> R;
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) R(i, j) = R36[i * 6 + j];
    Vector3<double> p;
    for (int i = 0; i < 3; ++i) p(i) = p3[i];
    const Quaternion<double> q(q4[3], q4[0], q4[1], q4[2]);
    return on_filter(h, [&](auto& f) { *out = f.relativePoseUpdate(state_id_a, state_id_b, p, q, R, chi2_max); return 0; });
  });
}
}
