// msckf_mono_b200/csrc/fde_capi.cpp -- stacked aided updates with fault detection and exclusion in the C view
// (include/msckf_mono_c.h, msckf_mono_aid_stack_update_fde / msckf_mono_batch_aid_stack_update_fde): MSCKF<_S>::aidedUpdate(items,
// fde) and MSCKFBatch<_S>::aidedUpdate(items, fde) over handles created by filter_capi.cpp and batch_capi.cpp.  Host code only;
// its own translation unit, so that the other view files link against a C-ABI without msckf_b200_aid_stack_update_fde.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
template <class S>
void batch_fde(MSCKFBatch<S>& b, const int* n_items, const msckf_b200_aid_item* items, const msckf_b200_aid_fde& fde,
               msckf_b200_aid_fde_result* out) {
  std::vector<std::vector<msckf_b200_aid_item>> it(b.size());
  for (size_t i = 0, o = 0; i < b.size(); o += n_items[i], ++i) {
    if (n_items[i] < 0) throw std::invalid_argument("batch_aid_stack_update_fde: negative item count");
    if (n_items[i] > 0 && !items) throw std::invalid_argument("batch_aid_stack_update_fde: null items");
    it[i].assign(items + o, items + o + n_items[i]);
  }
  const std::vector<msckf_b200_aid_fde_result> r = b.aidedUpdate(it, fde);
  for (size_t i = 0; i < r.size(); ++i)
    if (n_items[i] > 0) out[i] = r[i];
}
}  // namespace

extern "C" {
int msckf_mono_aid_stack_update_fde(void* h, const msckf_b200_aid_item* items, int n_items, const msckf_b200_aid_fde* fde,
                                    msckf_b200_aid_fde_result* out) {
  return guard([&] {
    if (!h || !fde || !out || n_items < 0 || (n_items > 0 && !items)) throw std::invalid_argument("aid_stack_update_fde: null argument");
    const std::vector<msckf_b200_aid_item> it(items, items + n_items);
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) *out = static_cast<MSCKF<float>*>(b->filter_ptr())->aidedUpdate(it, *fde);
    else *out = static_cast<MSCKF<double>*>(b->filter_ptr())->aidedUpdate(it, *fde);
    return 0;
  });
}
int msckf_mono_batch_aid_stack_update_fde(void* batch, const int* n_items, const msckf_b200_aid_item* items, const msckf_b200_aid_fde* fde,
                                          msckf_b200_aid_fde_result* out) {
  return guard([&] {
    if (!batch || !n_items || !fde || !out) throw std::invalid_argument("batch_aid_stack_update_fde: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_fde(*vb->bf, n_items, items, *fde, out);
    else batch_fde(*vb->bd, n_items, items, *fde, out);
    return 0;
  });
}
}
