// tests/stub/stub_nees.cpp -- TEST INFRASTRUCTURE ONLY.
// The consistency calls of include/msckf_b200.h (msckf_b200_nees / _batch_nees) for the recording fake of the C-ABI
// (tests/stub/stub.hpp), with NO numerics: each call checks its arguments as the engine does (truth and out not NULL, a finite
// truth, non-zero quaternions, no un-fetched update) and is recorded per engine with the IMU readings the engine had been
// handed by then.  The answer is every NEES 0 (full NaN and dim_full 0 without truth poses), positive definite.  Nothing
// outside tests/ builds or loads it.
#include "stub.hpp"

#include <cmath>

namespace {
stub::Records<> g_calls;
bool finite(const double* x, int n) {
  for (int i = 0; i < n; ++i)
    if (!std::isfinite(x[i])) return false;
  return true;
}
bool quaternion(const double* q) { return q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0; }
// truth_imu: p, v, b_g, b_a, g (ignored), q_IG; truth_poses: [M][7] p, q
int check(const msckf_b200_engine* e, const double* imu, const double* poses) {
  if (!imu || !finite(imu, 12) || !finite(imu + 15, 4) || !quaternion(imu + 15)) return stub::fail(MSCKF_B200_ERR_ARG, "stub: bad truth_imu");
  if (poses)
    for (int k = 0; k < e->M; ++k)
      if (!finite(poses + 7 * k, 7) || !quaternion(poses + 7 * k + 3)) return stub::fail(MSCKF_B200_ERR_ARG, "stub: bad truth_poses");
  if (e->pending) return stub::fail(MSCKF_B200_ERR_STATE, "stub: previous update not fetched");
  return 0;
}
void answer(const msckf_b200_engine* e, const double* poses, msckf_b200_nees_result* out) {
  *out = msckf_b200_nees_result{0.0, 0.0, 0.0, 0.0, poses ? 0.0 : NAN, poses ? 15 + 6 * e->M : 0, -1};
  g_calls.last(e);
}
}  // namespace

extern "C" {
int msckf_b200_nees(msckf_b200_engine* e, const double* truth_imu, const double* truth_poses, msckf_b200_nees_result* out) {
  if (!e || !out) return stub::fail(MSCKF_B200_ERR_ARG, "stub: null argument");
  if (int rc = check(e, truth_imu, truth_poses)) return rc;
  answer(e, truth_poses, out);
  g_calls.engine[e].single++;
  return 0;
}
int msckf_b200_batch_nees(msckf_b200_batch* b, const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out) {
  if (!b || !truth_imu || !out) return stub::fail(MSCKF_B200_ERR_ARG, "stub: null argument");
  for (size_t i = 0; i < b->es.size(); ++i)
    if (int rc = check(b->es[i], truth_imu[i], truth_poses ? truth_poses[i] : nullptr)) return rc;
  for (size_t i = 0; i < b->es.size(); ++i) {
    answer(b->es[i], truth_poses ? truth_poses[i] : nullptr, out + i);
    g_calls.engine[b->es[i]].batch++;
  }
  g_calls.batch[b]++;
  return 0;
}
// test hooks: out3 = single calls, batched calls naming e, IMU readings handed over before its last NEES call; the batched
// calls made on b
void msckf_b200_stub_nees_calls(const msckf_b200_engine* e, long long* out3) { g_calls.counts(e, out3); }
long long msckf_b200_stub_batch_nees_calls(const msckf_b200_batch* b) { return g_calls.of(b); }
}
