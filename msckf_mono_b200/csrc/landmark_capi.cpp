// msckf_mono_b200/csrc/landmark_capi.cpp -- mapped-landmark updates in the C view (include/msckf_mono_c.h,
// msckf_mono_landmark_update / msckf_mono_batch_landmark_update and their _iter forms): MSCKF<_S>::landmarkUpdate and MSCKFBatch<_S>::landmarkUpdate
// over handles created by filter_capi.cpp and batch_capi.cpp.  Host code only; its own translation unit, so that the other view
// files link against a C-ABI without msckf_b200_landmark_update / msckf_b200_batch_landmark_update.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
std::vector<landmarkObservation> observations(int n, const int* state_ids, const double* z, const double* p_L_G) {
  if (n < 0 || (n > 0 && (!state_ids || !z || !p_L_G))) throw std::invalid_argument("landmark_update: bad observation arrays");
  std::vector<landmarkObservation> o(n);
  for (int i = 0; i < n; ++i) {
    o[i].state_id = state_ids[i];
    o[i].z[0] = z[2 * i]; o[i].z[1] = z[2 * i + 1];
    for (int c = 0; c < 3; ++c) o[i].p_L_G[c] = p_L_G[3 * i + c];
  }
  return o;
}
FixedMatrix<double, 2, 2> noise(const double* R3) {
  FixedMatrix<double, 2, 2> R;
  R(0, 0) = R3[0]; R(1, 0) = R3[1]; R(0, 1) = R3[1]; R(1, 1) = R3[2];
  return R;
}
template <class S>
void batch_landmarks(MSCKFBatch<S>& b, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G,
                     const double* R3, double chi2_obs, int max_iter, double tol, double* gamma, int* flag,
                     msckf_b200_landmark_result* out) {
  const size_t nf = b.size();
  std::vector<std::vector<landmarkObservation>> obs(nf);
  size_t o = 0;
  for (size_t i = 0; i < nf; ++i) {
    obs[i] = observations(n_obs[i], state_ids + o, z + 2 * o, p_L_G + 3 * o);
    o += n_obs[i];
  }
  const FixedMatrix<double, 2, 2> R = R3 ? noise(R3) : FixedMatrix<double, 2, 2>();
  std::vector<std::vector<double>> g;
  std::vector<std::vector<int>> fl;
  const std::vector<msckf_b200_landmark_result> r = b.landmarkUpdate(obs, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
  o = 0;
  for (size_t i = 0; i < nf; ++i) {
    if (n_obs[i] > 0) {
      out[i] = r[i];
      for (int j = 0; j < n_obs[i]; ++j) {
        if (gamma) gamma[o + j] = g[i][j];
        if (flag) flag[o + j] = fl[i][j];
      }
    }
    o += n_obs[i];
  }
}
int single_landmarks(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                     double chi2_obs, int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return guard([&] {
    if (!h || !out) throw std::invalid_argument("landmark_update: null argument");
    const std::vector<landmarkObservation> obs = observations(n_obs, state_ids, z, p_L_G);
    const FixedMatrix<double, 2, 2> R = R3 ? noise(R3) : FixedMatrix<double, 2, 2>();
    std::vector<double> g;
    std::vector<int> fl;
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0)
      *out = static_cast<MSCKF<float>*>(b->filter_ptr())->landmarkUpdate(obs, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
    else
      *out = static_cast<MSCKF<double>*>(b->filter_ptr())->landmarkUpdate(obs, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
    for (int i = 0; i < n_obs; ++i) {
      if (gamma) gamma[i] = g[i];
      if (flag) flag[i] = fl[i];
    }
    return 0;
  });
}
int many_landmarks(void* batch, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                   double chi2_obs, int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return guard([&] {
    if (!batch || !n_obs || !out) throw std::invalid_argument("batch_landmark_update: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_landmarks(*vb->bf, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, gamma, flag, out);
    else batch_landmarks(*vb->bd, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, gamma, flag, out);
    return 0;
  });
}
}  // namespace

extern "C" {
int msckf_mono_landmark_update(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                               double chi2_obs, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return single_landmarks(h, n_obs, state_ids, z, p_L_G, R3, chi2_obs, 1, 1e-10, gamma, flag, out);
}
int msckf_mono_batch_landmark_update(void* batch, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                     const double* R3, double chi2_obs, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return many_landmarks(batch, n_obs, state_ids, z, p_L_G, R3, chi2_obs, 1, 1e-10, gamma, flag, out);
}
int msckf_mono_landmark_update_iter(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                                    double chi2_obs, int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return single_landmarks(h, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, gamma, flag, out);
}
int msckf_mono_batch_landmark_update_iter(void* batch, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                          const double* R3, double chi2_obs, int max_iter, double tol, double* gamma, int* flag,
                                          msckf_b200_landmark_result* out) {
  return many_landmarks(batch, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, gamma, flag, out);
}
}
