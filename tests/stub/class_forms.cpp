// tests/stub/class_forms.cpp -- TEST INFRASTRUCTURE ONLY.
// Test hooks that call class forms of msckf_mono::MSCKF<_S> (include/msckf_mono/msckf.h) which have no C view entry point
// -- the GNSS, range and at-rest updates -- on a C view filter handle, so that a CPU test can see what they send to the
// recording fake of the C-ABI (tests/stub/stub_aid_stack.cpp).  Built into the fake's library with the C view, whose handles
// (msckf_mono_b200/csrc/filter_view.hpp) they take.  Nothing outside tests/ builds or loads it.
#include <msckf_b200.h>
#include <msckf_mono/msckf.h>

#include "filter_view.hpp"

namespace {
template <class F>
int on_filter(void* h, F&& f) {
  msckf_view::Base* b = static_cast<msckf_view::Base*>(h);
  if (b->dtype == 0) return f(*static_cast<msckf_mono::MSCKF<float>*>(b->filter_ptr()));
  return f(*static_cast<msckf_mono::MSCKF<double>*>(b->filter_ptr()));
}
msckf_mono::MatrixX<double> matrix(const double* R, int rows) {  // rows x rows, row-major
  msckf_mono::MatrixX<double> Rm(rows, rows);
  for (int i = 0; i < rows; ++i)
    for (int j = 0; j < rows; ++j) Rm(i, j) = R[i * rows + j];
  return Rm;
}
}  // namespace

extern "C" {
// the GNSS class forms on a C view filter handle: which = 0 antennaPositionUpdate(p, v, R, mask), 1 cloneAntennaPositionUpdate
// (state_id, p, v, R, mask), 2 headingUpdate(psi, v, var), 3 cloneHeadingUpdate(state_id, psi, v, var); R is rows x rows
// row-major with rows = R_rows.  -1 with msckf_mono_last_error() for an exception.
int msckf_b200_stub_gnss_class_call(void* h, int which, int state_id, const double* p3, const double* v3, const double* R, int R_rows,
                                    int mask, double psi, double var, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> p, v;
    for (int i = 0; i < 3; ++i) { p(i) = p3[i]; v(i) = v3[i]; }
    const msckf_mono::MatrixX<double> Rm = matrix(R, R_rows);
    return on_filter(h, [&](auto& f) {
      if (which == 0) *out = f.antennaPositionUpdate(p, v, Rm, mask);
      else if (which == 1) *out = f.cloneAntennaPositionUpdate(state_id, p, v, Rm, mask);
      else if (which == 2) *out = f.headingUpdate(psi, v, var);
      else *out = f.cloneHeadingUpdate(state_id, psi, v, var);
      return 0;
    });
  });
}
// the range class forms: which = 0 rangeUpdate(rho, a3, l3, var), 1 cloneRangeUpdate(state_id, rho, a3, l3, var),
// 2 planeRangeUpdate(rho, h, l3, f3, var), 3 clonePlaneRangeUpdate(state_id, rho, h, l3, f3, var).  -1 with
// msckf_mono_last_error() for an exception.
int msckf_b200_stub_range_class_call(void* h, int which, int state_id, double rho, double height, const double* a3, const double* l3,
                                     const double* f3, double var, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> a, l, f;
    for (int i = 0; i < 3; ++i) { a(i) = a3[i]; l(i) = l3[i]; f(i) = f3[i]; }
    return on_filter(h, [&](auto& flt) {
      if (which == 0) *out = flt.rangeUpdate(rho, a, l, var);
      else if (which == 1) *out = flt.cloneRangeUpdate(state_id, rho, a, l, var);
      else if (which == 2) *out = flt.planeRangeUpdate(rho, height, l, f, var);
      else *out = flt.clonePlaneRangeUpdate(state_id, rho, height, l, f, var);
      return 0;
    });
  });
}
// the at-rest class forms: which = 0 gyroAtRestUpdate(v3, R), 1 accelAtRestUpdate(v3, R); R is R_rows x R_rows row-major.  -1
// with msckf_mono_last_error() for an exception.
int msckf_b200_stub_at_rest_class_call(void* h, int which, const double* v3, const double* R, int R_rows, msckf_b200_aid_result* out) {
  return msckf_view::guard([&] {
    msckf_mono::Vector3<double> v;
    for (int i = 0; i < 3; ++i) v(i) = v3[i];
    const msckf_mono::MatrixX<double> Rm = matrix(R, R_rows);
    return on_filter(h, [&](auto& f) {
      *out = which == 0 ? f.gyroAtRestUpdate(v, Rm) : f.accelAtRestUpdate(v, Rm);
      return 0;
    });
  });
}
}
