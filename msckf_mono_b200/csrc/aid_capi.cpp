// msckf_mono_b200/csrc/aid_capi.cpp -- aided measurement updates in the C view (include/msckf_mono_c.h,
// msckf_mono_aid_update / msckf_mono_batch_aid_update): MSCKF<_S>::aidedUpdate and MSCKFBatch<_S>::aidedUpdate over handles
// created by filter_capi.cpp and batch_capi.cpp.  Host code only; calls the engine C-ABI's
// msckf_b200_aid_update / msckf_b200_batch_aid_update.
#include <stdexcept>
#include <vector>
#include <msckf_mono/msckf.h>
#include <msckf_mono_c.h>
#include "filter_view.hpp"

using namespace msckf_mono;
using namespace msckf_view;

namespace {
template <class S>
void batch_aid(MSCKFBatch<S>& b, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  const std::vector<msckf_b200_aid_result> r = b.aidedUpdate(std::vector<msckf_b200_aid>(aid, aid + b.size()));
  for (size_t i = 0; i < r.size(); ++i)
    if (aid[i].model >= 0) out[i] = r[i];
}
}  // namespace

extern "C" {
int msckf_mono_aid_update(void* h, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  return guard([&] {
    if (!h || !aid || !out) throw std::invalid_argument("aid_update: null argument");
    Base* b = static_cast<Base*>(h);
    if (b->dtype == 0) *out = static_cast<MSCKF<float>*>(b->filter_ptr())->aidedUpdate(*aid);
    else *out = static_cast<MSCKF<double>*>(b->filter_ptr())->aidedUpdate(*aid);
    return 0;
  });
}
int msckf_mono_batch_aid_update(void* batch, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  return guard([&] {
    if (!batch || !aid || !out) throw std::invalid_argument("batch_aid_update: null argument");
    auto* vb = static_cast<ViewBatch*>(batch);
    if (vb->bf) batch_aid(*vb->bf, aid, out);
    else batch_aid(*vb->bd, aid, out);
    return 0;
  });
}
}
