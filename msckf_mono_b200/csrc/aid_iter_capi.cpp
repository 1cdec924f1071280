// msckf_mono_b200/csrc/aid_iter_capi.cpp -- iterated stacked aided updates in the C view (include/msckf_mono_c.h,
// msckf_mono_aid_stack_update_iter / _fde_iter and their batch forms): MSCKF<_S>::aidedUpdate(items, chi2_max | fde, iter,
// iter_out) and the MSCKFBatch<_S> forms over handles created by filter_capi.cpp and batch_capi.cpp.  Host code only; calls
// the engine C-ABI's _iter entry points.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
// the concatenated items of a batch call, one list per filter
std::vector<std::vector<msckf_b200_aid_item>> split(size_t n, const int* n_items, const msckf_b200_aid_item* items, const char* what) {
  std::vector<std::vector<msckf_b200_aid_item>> it(n);
  for (size_t i = 0, o = 0; i < n; o += n_items[i], ++i) {
    if (n_items[i] < 0) throw std::invalid_argument(std::string(what) + ": negative item count");
    if (n_items[i] > 0 && !items) throw std::invalid_argument(std::string(what) + ": null items");
    it[i].assign(items + o, items + o + n_items[i]);
  }
  return it;
}

// fde NULL: the plain form (out is msckf_b200_aid_result [n]); else the FDE form (msckf_b200_aid_fde_result [n])
template <class S>
void batch_iter(MSCKFBatch<S>& b, const int* n_items, const msckf_b200_aid_item* items, double chi2_max, const msckf_b200_aid_fde* fde,
                const msckf_b200_aid_iter* iter, void* out, msckf_b200_aid_iter_result* iter_out) {
  const auto it = split(b.size(), n_items, items, fde ? "batch_aid_stack_update_fde_iter" : "batch_aid_stack_update_iter");
  const std::vector<msckf_b200_aid_iter> opt(iter, iter + b.size());
  std::vector<msckf_b200_aid_iter_result> io;
  if (fde) {
    const std::vector<msckf_b200_aid_fde_result> r = b.aidedUpdate(it, *fde, opt, io);
    for (size_t i = 0; i < r.size(); ++i)
      if (n_items[i] > 0) static_cast<msckf_b200_aid_fde_result*>(out)[i] = r[i];
  } else {
    const std::vector<msckf_b200_aid_result> r = b.aidedUpdate(it, chi2_max, opt, io);
    for (size_t i = 0; i < r.size(); ++i)
      if (n_items[i] > 0) static_cast<msckf_b200_aid_result*>(out)[i] = r[i];
  }
  for (size_t i = 0; i < io.size(); ++i)
    if (n_items[i] > 0) iter_out[i] = io[i];
}
}  // namespace

extern "C" {
int msckf_mono_aid_stack_update_iter(void* h, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                     const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out, msckf_b200_aid_iter_result* iter_out) {
  return guard([&] {
    if (!h || !iter || !out || !iter_out || n_items < 0 || (n_items > 0 && !items))
      throw std::invalid_argument("aid_stack_update_iter: null argument");
    const std::vector<msckf_b200_aid_item> it(items, items + n_items);
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) *out = static_cast<MSCKF<float>*>(b->filter_ptr())->aidedUpdate(it, chi2_max, *iter, *iter_out);
    else *out = static_cast<MSCKF<double>*>(b->filter_ptr())->aidedUpdate(it, chi2_max, *iter, *iter_out);
    return 0;
  });
}
int msckf_mono_aid_stack_update_fde_iter(void* h, const msckf_b200_aid_item* items, int n_items, const msckf_b200_aid_fde* fde,
                                         const msckf_b200_aid_iter* iter, msckf_b200_aid_fde_result* out,
                                         msckf_b200_aid_iter_result* iter_out) {
  return guard([&] {
    if (!h || !fde || !iter || !out || !iter_out || n_items < 0 || (n_items > 0 && !items))
      throw std::invalid_argument("aid_stack_update_fde_iter: null argument");
    const std::vector<msckf_b200_aid_item> it(items, items + n_items);
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) *out = static_cast<MSCKF<float>*>(b->filter_ptr())->aidedUpdate(it, *fde, *iter, *iter_out);
    else *out = static_cast<MSCKF<double>*>(b->filter_ptr())->aidedUpdate(it, *fde, *iter, *iter_out);
    return 0;
  });
}
int msckf_mono_batch_aid_stack_update_iter(void* batch, const int* n_items, const msckf_b200_aid_item* items, double chi2_max,
                                           const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out,
                                           msckf_b200_aid_iter_result* iter_out) {
  return guard([&] {
    if (!batch || !n_items || !iter || !out || !iter_out) throw std::invalid_argument("batch_aid_stack_update_iter: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_iter(*vb->bf, n_items, items, chi2_max, nullptr, iter, out, iter_out);
    else batch_iter(*vb->bd, n_items, items, chi2_max, nullptr, iter, out, iter_out);
    return 0;
  });
}
int msckf_mono_batch_aid_stack_update_fde_iter(void* batch, const int* n_items, const msckf_b200_aid_item* items,
                                               const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                               msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out) {
  return guard([&] {
    if (!batch || !n_items || !fde || !iter || !out || !iter_out)
      throw std::invalid_argument("batch_aid_stack_update_fde_iter: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_iter(*vb->bf, n_items, items, 0.0, fde, iter, out, iter_out);
    else batch_iter(*vb->bd, n_items, items, 0.0, fde, iter, out, iter_out);
    return 0;
  });
}
}
