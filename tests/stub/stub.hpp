// tests/stub/stub.hpp -- TEST INFRASTRUCTURE ONLY.
// What the sources of the recording fake of the C-ABI (include/msckf_b200.h, tests/stub/stub_*.cpp) share: the one definition
// of its engine and batch handles, its error text, and the per-engine and per-batch records its call families keep.  The
// sources link into one complete fake: every msckf_b200_* entry point and every msckf_b200_stub_* test hook is defined in
// exactly one of them.  Nothing outside tests/ builds or loads it.
#pragma once
#include <msckf_b200.h>

#include <map>
#include <vector>

struct msckf_b200_engine {
  int dtype = 0, M = 0, max_clones = 0;
  double imu[19] = {0};
  std::vector<int> last_len;  // observations per track of the pending batch
  std::vector<int> buf_off, buf_idx;  // msckf_b200_input_buffer: host arrays the caller packs into
  std::vector<double> buf_obs, buf_pfg;
  long long imu_readings = 0;
  int pending = 0, mode = 0;
  long long updates = 0, launches = 0;
};
struct msckf_b200_batch { std::vector<msckf_b200_engine*> es; long long launches = 0; };

namespace stub {
// sets msckf_b200_last_error() and returns code
int fail(int code, const char* msg);

// What every call family records per engine: its single calls, the batched calls naming the engine, and the IMU readings the
// engine had been handed by its last call.  A family extends it with what it records of that call.
struct Calls { long long single = 0, batch = 0, readings_at_last = -1; };

// One family's records, keyed by handle address.  They outlive their handle (a freed handle's address may come back), so the
// tests compare counts before and after a call.
template <class R = Calls>
struct Records {
  std::map<const msckf_b200_engine*, R> engine;
  std::map<const msckf_b200_batch*, long long> batch;  // batched calls made on each batch
  // the record of e's latest call, its readings_at_last set
  R& last(const msckf_b200_engine* e) {
    R& r = engine[e];
    r.readings_at_last = e->imu_readings;
    return r;
  }
  R of(const msckf_b200_engine* e) const {
    auto it = engine.find(e);
    return it == engine.end() ? R() : it->second;
  }
  long long of(const msckf_b200_batch* b) const {
    auto it = batch.find(b);
    return it == batch.end() ? 0 : it->second;
  }
  // out3 = single calls, batched calls naming e, IMU readings handed over before its last call
  void counts(const msckf_b200_engine* e, long long* out3) const {
    const R r = of(e);
    out3[0] = r.single; out3[1] = r.batch; out3[2] = r.readings_at_last;
  }
};
}  // namespace stub

extern "C" {
// defined in stub_aid_stack.cpp, read by the standstill hooks (the at-rest class forms reach the engine as stacked calls)
int msckf_b200_stub_aid_stack_calls(const msckf_b200_engine* e, long long* out3, double* fde33, double* rec, int cap);
}
