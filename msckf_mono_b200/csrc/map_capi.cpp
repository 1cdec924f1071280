// msckf_mono_b200/csrc/map_capi.cpp -- mapped-landmark updates with map uncertainty in the C view (include/msckf_mono_c.h,
// msckf_mono_map_update / msckf_mono_batch_map_update): MSCKF<_S>::landmarkUpdate and MSCKFBatch<_S>::landmarkUpdate over
// mapObservation / mapLandmark, on handles created by filter_capi.cpp and batch_capi.cpp.  Host code only; its own translation
// unit, so that the other view files link against a C-ABI without msckf_b200_map_landmark_update.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
std::vector<mapObservation> observations(int n, const int* state_ids, const int* landmark, const double* z) {
  if (n < 0 || (n > 0 && (!state_ids || !landmark || !z))) throw std::invalid_argument("map_update: bad observation arrays");
  std::vector<mapObservation> o(n);
  for (int i = 0; i < n; ++i) {
    o[i].state_id = state_ids[i];
    o[i].landmark = landmark[i];
    o[i].z[0] = z[2 * i]; o[i].z[1] = z[2 * i + 1];
  }
  return o;
}
std::vector<mapLandmark> landmarks(int n, const double* p_L_G, const double* Sigma) {
  if (n < 0 || (n > 0 && (!p_L_G || !Sigma))) throw std::invalid_argument("map_update: bad landmark arrays");
  std::vector<mapLandmark> l(n);
  for (int i = 0; i < n; ++i) {
    for (int c = 0; c < 3; ++c) l[i].p_L_G[c] = p_L_G[3 * i + c];
    for (int c = 0; c < 6; ++c) l[i].Sigma[c] = Sigma[6 * i + c];
  }
  return l;
}
FixedMatrix<double, 2, 2> noise(const double* R3) {
  FixedMatrix<double, 2, 2> R;
  R(0, 0) = R3[0]; R(1, 0) = R3[1]; R(0, 1) = R3[1]; R(1, 1) = R3[2];
  return R;
}
template <class S>
void batch_map(MSCKFBatch<S>& b, const int* n_obs, const int* state_ids, const int* landmark, const double* z, const int* n_landmarks,
               const double* p_L_G, const double* Sigma, const double* R3, double chi2_obs, int max_iter, double tol, double* gamma,
               int* flag, msckf_b200_landmark_result* out) {
  const size_t nf = b.size();
  std::vector<std::vector<mapObservation>> obs(nf);
  std::vector<std::vector<mapLandmark>> lms(nf);
  size_t o = 0, l = 0;
  for (size_t i = 0; i < nf; ++i) {
    obs[i] = observations(n_obs[i], state_ids + o, landmark + o, z + 2 * o);
    lms[i] = landmarks(n_landmarks[i], p_L_G + 3 * l, Sigma + 6 * l);
    o += n_obs[i];
    l += n_landmarks[i];
  }
  const FixedMatrix<double, 2, 2> R = R3 ? noise(R3) : FixedMatrix<double, 2, 2>();
  std::vector<std::vector<double>> g;
  std::vector<std::vector<int>> fl;
  const std::vector<msckf_b200_landmark_result> r = b.landmarkUpdate(obs, lms, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
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
}  // namespace

extern "C" {
int msckf_mono_map_update(void* h, int n_obs, const int* state_ids, const int* landmark, const double* z, int n_landmarks,
                          const double* p_L_G, const double* Sigma, const double* R3, double chi2_obs, int max_iter, double tol,
                          double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return guard([&] {
    if (!h || !out) throw std::invalid_argument("map_update: null argument");
    const std::vector<mapObservation> obs = observations(n_obs, state_ids, landmark, z);
    const std::vector<mapLandmark> lms = landmarks(n_landmarks, p_L_G, Sigma);
    const FixedMatrix<double, 2, 2> R = R3 ? noise(R3) : FixedMatrix<double, 2, 2>();
    std::vector<double> g;
    std::vector<int> fl;
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0)
      *out = static_cast<MSCKF<float>*>(b->filter_ptr())->landmarkUpdate(obs, lms, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
    else
      *out = static_cast<MSCKF<double>*>(b->filter_ptr())->landmarkUpdate(obs, lms, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
    for (int i = 0; i < n_obs; ++i) {
      if (gamma) gamma[i] = g[i];
      if (flag) flag[i] = fl[i];
    }
    return 0;
  });
}
int msckf_mono_batch_map_update(void* batch, const int* n_obs, const int* state_ids, const int* landmark, const double* z,
                                const int* n_landmarks, const double* p_L_G, const double* Sigma, const double* R3, double chi2_obs,
                                int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out) {
  return guard([&] {
    if (!batch || !n_obs || !n_landmarks || !out) throw std::invalid_argument("batch_map_update: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_map(*vb->bf, n_obs, state_ids, landmark, z, n_landmarks, p_L_G, Sigma, R3, chi2_obs, max_iter, tol, gamma, flag, out);
    else batch_map(*vb->bd, n_obs, state_ids, landmark, z, n_landmarks, p_L_G, Sigma, R3, chi2_obs, max_iter, tol, gamma, flag, out);
    return 0;
  });
}
}
