// msckf_mono_b200/csrc/consensus_capi.cpp -- mapped-landmark updates with a consensus on the matches in the C view
// (include/msckf_mono_c.h, msckf_mono_landmark_update_consensus / msckf_mono_batch_landmark_update_consensus):
// MSCKF<_S>::landmarkUpdate and MSCKFBatch<_S>::landmarkUpdate with a msckf_b200_landmark_consensus, exact map, on handles
// created by filter_capi.cpp and batch_capi.cpp.  Host code only; calls the engine C-ABI's
// msckf_b200_landmark_update_consensus / _batch_landmark_update_consensus.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
std::vector<landmarkObservation> observations(int n, const int* state_ids, const double* z, const double* p_L_G) {
  if (n < 0 || (n > 0 && (!state_ids || !z || !p_L_G))) throw std::invalid_argument("landmark_update_consensus: bad observation arrays");
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
void batch_consensus(MSCKFBatch<S>& b, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                     double chi2_obs, int max_iter, double tol, const msckf_b200_landmark_consensus* cons, double* gamma, int* flag,
                     msckf_b200_landmark_result* out, msckf_b200_landmark_consensus_result* cons_out) {
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
  std::vector<msckf_b200_landmark_consensus_result> co;
  const std::vector<msckf_b200_landmark_consensus> cs(cons, cons + nf);
  const std::vector<msckf_b200_landmark_result> r = b.landmarkUpdate(obs, cs, co, R3 ? &R : nullptr, chi2_obs, &g, &fl, max_iter, tol);
  o = 0;
  for (size_t i = 0; i < nf; ++i) {
    if (cons_out) cons_out[i] = co[i];
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
int msckf_mono_landmark_update_consensus(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                         const double* R3, double chi2_obs, int max_iter, double tol,
                                         const msckf_b200_landmark_consensus* cons, double* gamma, int* flag,
                                         msckf_b200_landmark_result* out, msckf_b200_landmark_consensus_result* cons_out) {
  return guard([&] {
    if (!h || !out || !cons || !cons_out) throw std::invalid_argument("landmark_update_consensus: null argument");
    const std::vector<landmarkObservation> obs = observations(n_obs, state_ids, z, p_L_G);
    const FixedMatrix<double, 2, 2> R = R3 ? noise(R3) : FixedMatrix<double, 2, 2>();
    std::vector<double> g;
    std::vector<int> fl;
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0)
      *out = static_cast<MSCKF<float>*>(b->filter_ptr())->landmarkUpdate(obs, *cons, *cons_out, R3 ? &R : nullptr, chi2_obs, &g, &fl,
                                                                         max_iter, tol);
    else
      *out = static_cast<MSCKF<double>*>(b->filter_ptr())->landmarkUpdate(obs, *cons, *cons_out, R3 ? &R : nullptr, chi2_obs, &g, &fl,
                                                                          max_iter, tol);
    for (int i = 0; i < n_obs; ++i) {
      if (gamma) gamma[i] = g[i];
      if (flag) flag[i] = fl[i];
    }
    return 0;
  });
}
int msckf_mono_batch_landmark_update_consensus(void* batch, const int* n_obs, const int* state_ids, const double* z,
                                               const double* p_L_G, const double* R3, double chi2_obs, int max_iter, double tol,
                                               const msckf_b200_landmark_consensus* cons, double* gamma, int* flag,
                                               msckf_b200_landmark_result* out, msckf_b200_landmark_consensus_result* cons_out) {
  return guard([&] {
    if (!batch || !n_obs || !out || !cons) throw std::invalid_argument("batch_landmark_update_consensus: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_consensus(*vb->bf, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, cons, gamma, flag, out, cons_out);
    else batch_consensus(*vb->bd, n_obs, state_ids, z, p_L_G, R3, chi2_obs, max_iter, tol, cons, gamma, flag, out, cons_out);
    return 0;
  });
}
}
