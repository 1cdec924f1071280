// msckf_mono_b200/csrc/standstill_capi.cpp -- standstill detection and the zero-motion update in the C view
// (include/msckf_mono_c.h, msckf_mono_standstill_update / _batch_standstill_update): MSCKF<_S>::standstillUpdate and
// MSCKFBatch<_S>::standstillUpdate over handles created by filter_capi.cpp and batch_capi.cpp.  Host code only; calls the
// engine C-ABI's msckf_b200_standstill_update /
// msckf_b200_batch_standstill_update.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
// k readings [k][7] (omega, a, dT) as the filter's imuReading<S>
template <class S>
std::vector<imuReading<S>> readings_of(const double* r, int k) {
  std::vector<imuReading<S>> out(k);
  for (int j = 0; j < k; ++j) {
    for (int i = 0; i < 3; ++i) { out[j].omega(i) = (S)r[7 * j + i]; out[j].a(i) = (S)r[7 * j + 3 + i]; }
    out[j].dT = (S)r[7 * j + 6];
  }
  return out;
}
template <class S>
void batch_standstill(MSCKFBatch<S>& b, const int* k, const double* readings, const msckf_b200_standstill& cfg,
                      msckf_b200_standstill_result* out) {
  std::vector<std::vector<imuReading<S>>> rs(b.size());
  for (size_t i = 0, o = 0; i < b.size(); o += 7 * (size_t)k[i], ++i) {
    if (k[i] < 0) throw std::invalid_argument("batch_standstill_update: negative reading count");
    if (k[i] > 0 && !readings) throw std::invalid_argument("batch_standstill_update: null readings");
    if (k[i] > 0) rs[i] = readings_of<S>(readings + o, k[i]);
  }
  const std::vector<msckf_b200_standstill_result> r = b.standstillUpdate(rs, cfg);
  for (size_t i = 0; i < r.size(); ++i)
    if (k[i] > 0) out[i] = r[i];
}
}  // namespace

extern "C" {
int msckf_mono_standstill_update(void* h, const double* readings, int k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out) {
  return guard([&] {
    if (!h || !readings || !cfg || !out || k < 0) throw std::invalid_argument("standstill_update: null argument");
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) *out = static_cast<MSCKF<float>*>(b->filter_ptr())->standstillUpdate(readings_of<float>(readings, k), *cfg);
    else *out = static_cast<MSCKF<double>*>(b->filter_ptr())->standstillUpdate(readings_of<double>(readings, k), *cfg);
    return 0;
  });
}
int msckf_mono_batch_standstill_update(void* batch, const int* k, const double* readings, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out) {
  return guard([&] {
    if (!batch || !k || !cfg || !out) throw std::invalid_argument("batch_standstill_update: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_standstill(*vb->bf, k, readings, *cfg, out);
    else batch_standstill(*vb->bd, k, readings, *cfg, out);
    return 0;
  });
}
}
