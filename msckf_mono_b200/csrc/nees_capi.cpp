// msckf_mono_b200/csrc/nees_capi.cpp -- consistency against ground truth in the C view (include/msckf_mono_c.h,
// msckf_mono_nees / msckf_mono_batch_nees): MSCKF<_S>::nees and MSCKFBatch<_S>::nees over handles created by filter_capi.cpp
// and batch_capi.cpp.  Host code only; its own translation unit, so that the other two link against a C-ABI without
// msckf_b200_nees / msckf_b200_batch_nees.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
imuState<double> truth_imu_of(const double* im) {
  if (!im) throw std::invalid_argument("nees: null truth_imu");
  imuState<double> s;
  for (int i = 0; i < 3; ++i) {
    s.p_I_G(i) = im[i]; s.v_I_G(i) = im[3 + i]; s.b_g(i) = im[6 + i]; s.b_a(i) = im[9 + i]; s.g(i) = im[12 + i];
  }
  s.q_IG = Quaternion<double>(im[18], im[15], im[16], im[17]);
  return s;
}
std::vector<camState<double>> truth_cams_of(const double* poses, size_t M) {
  std::vector<camState<double>> cs(M);
  for (size_t k = 0; k < M; ++k) {
    const double* p = poses + 7 * k;
    for (int i = 0; i < 3; ++i) cs[k].p_C_G(i) = p[i];
    cs[k].q_CG = Quaternion<double>(p[6], p[3], p[4], p[5]);
  }
  return cs;
}
void put(const msckf_b200_nees_result& r, double* o) {
  o[0] = r.orientation; o[1] = r.position; o[2] = r.pose; o[3] = r.imu; o[4] = r.full; o[5] = r.dim_full; o[6] = r.first_bad_pivot;
}
template <class S>
void filter_nees(MSCKF<S>& f, const double* im, const double* poses, double* out7) {
  const imuState<double> truth = truth_imu_of(im);
  std::vector<camState<double>> cams;
  if (poses) cams = truth_cams_of(poses, f.getNumCamStates());
  put(f.nees(truth, poses ? &cams : nullptr), out7);
}
template <class S>
void batch_nees(MSCKFBatch<S>& b, const std::vector<MSCKF<S>*>& fs, const double* const* im, const double* const* poses, double* out7) {
  if (!im) throw std::invalid_argument("batch_nees: null truth_imu");
  const size_t n = b.size();
  std::vector<imuState<double>> truth(n);
  std::vector<std::vector<camState<double>>> cams(n);
  std::vector<const std::vector<camState<double>>*> tc(n, nullptr);
  for (size_t i = 0; i < n; ++i) {
    truth[i] = truth_imu_of(im[i]);
    if (poses && poses[i]) { cams[i] = truth_cams_of(poses[i], fs[i]->getNumCamStates()); tc[i] = &cams[i]; }
  }
  const std::vector<msckf_b200_nees_result> r = b.nees(truth, tc);
  for (size_t i = 0; i < n; ++i) put(r[i], out7 + 7 * i);
}
}  // namespace

extern "C" {
int msckf_mono_nees(void* h, const double* truth_imu, const double* truth_poses, double* out7) {
  return guard([&] {
    if (!h || !out7) throw std::invalid_argument("nees: null argument");
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) filter_nees(*static_cast<MSCKF<float>*>(b->filter_ptr()), truth_imu, truth_poses, out7);
    else filter_nees(*static_cast<MSCKF<double>*>(b->filter_ptr()), truth_imu, truth_poses, out7);
    return 0;
  });
}
int msckf_mono_batch_nees(void* batch, const double* const* truth_imu, const double* const* truth_poses, double* out7) {
  return guard([&] {
    if (!batch || !out7) throw std::invalid_argument("batch_nees: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_nees(*vb->bf, vb->bf->filters(), truth_imu, truth_poses, out7);
    else batch_nees(*vb->bd, vb->bd->filters(), truth_imu, truth_poses, out7);
    return 0;
  });
}
}
