// msckf_mono_b200/csrc/engine.cu -- host side of the H100 engine and the C-ABI of include/msckf_b200.h.
// One handle = one filter: device-resident covariance / clone poses / IMU state and workspaces.  Updates run through a
// launch context (Ctx): one stream, one packed pinned + device input arena ([UpdArgs per filter | track batches]), one packed
// report arena, a small cache of captured CUDA graphs.  Every engine has a private context; a msckf_b200_batch is a context
// shared by several engines -- the same kernels with the filter index in blockIdx.z.  No CPU fallback anywhere.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/msckf_b200.h"
#include "aid_kernels.cuh"
#include "common.cuh"
#include "feature_kernels.cuh"
#include "gram_kernels.cuh"
#include "landmark_kernels.cuh"
#include "consensus_kernels.cuh"
#include "nees_kernels.cuh"
#include "state_kernels.cuh"
#include "tail_kernels.cuh"
#include "tail_cluster.cuh"
#include "tail_fused.cuh"

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(MSCKF_B200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));        \
  } while (0)
#define RC(call) do { int rc_ = (call); if (rc_ != 0) return rc_; } while (0)

using mb::kMaxSplit;  // split-K chunks of the Gram products (gram_kernels.cuh)
constexpr int kJacBatchGroup = 32;  // k_jac threads per track in a device batch (DESIGN.md 4.2)
constexpr int kTailCluster = 8;  // portable cluster size: the serial EKF tail runs on 8 SMs of one GPC
constexpr size_t kSmemBudget = 220 * 1024;  // dynamic shared memory per CTA, under H100's 227 KB opt-in limit
// k_aid: W^T and dx in dynamic shared memory up to this many bytes, else in the global workspace (both forms of the kernel;
// with the FDE form's static shared memory this passes the default 48 KB per CTA, so set_func_attrs raises the limit)
constexpr size_t kAidSmemMax = 32 * 1024;
constexpr int kStandstillMaxReadings = 4096;  // IMU readings of one standstill window
constexpr int kMaxClonesHard = mb::kMaxKeep;  // the keep list of prune() travels as a kernel argument
constexpr int kMaxGraphs = 8;

static const double kChi2_005[99] = {
#include "chi2_table.inc"
};

inline size_t up16(size_t x) { return (x + 15) & ~(size_t)15; }
inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

// SMs of a device (cached per ordinal): caps the grids of the grid-stride element-wise kernels at a few CTAs per SM
inline int num_sms(int dev) {
  static int n[64] = {};
  if (dev < 0 || dev >= 64) return 132;
  if (n[dev] == 0 && cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n[dev] = 132;
  return n[dev];
}

// pinned host + device buffer pair that grows on demand
struct Arena {
  unsigned char *d = nullptr, *h = nullptr;
  size_t cap = 0;
  int ensure(size_t need, cudaStream_t s) {
    if (need <= cap) return 0;
    if (s) CK(cudaStreamSynchronize(s));
    release();
    size_t c = std::max(need, cap * 2);
    c = up256(c);
    CK(cudaMalloc(&d, c));
    CK(cudaMallocHost(&h, c));
    memset(h, 0, c);
    // zeroed on the stream that uses the arena: cudaMemset would run on the legacy default stream, which the engine's
    // non-blocking streams do not wait for, so it could land after the first input copy into the arena or after the first
    // kernels wrote their reports there (a device batch's first update then read back m = 0 for a member)
    CK(cudaMemsetAsync(d, 0, c, s));
    if (!s) CK(cudaStreamSynchronize(nullptr));
    cap = c;
    return 0;
  }
  void release() {
    if (d) cudaFree(d);
    if (h) cudaFreeHost(h);
    d = h = nullptr; cap = 0;
  }
  ~Arena() { release(); }
};

// device-only workspace that grows on demand (at least x2); the stream is synchronised before the old block is freed
struct DevBuf {
  unsigned char* d = nullptr;
  size_t cap = 0;
  int ensure(size_t need, cudaStream_t s) {
    if (need <= cap) return 0;
    const size_t c = std::max(need, 2 * cap);
    CK(cudaStreamSynchronize(s));
    release();
    CK(cudaMalloc(&d, c));
    cap = c;
    return 0;
  }
  void release() {
    if (d) cudaFree(d);
    d = nullptr; cap = 0;
  }
  ~DevBuf() { release(); }
};

inline bool finite(const double* v, size_t k) {
  for (size_t i = 0; i < k; ++i) if (!std::isfinite(v[i])) return false;
  return true;
}

// the outcome of an aided or landmark update whose first member with a non-finite delta-x or covariance entry is `member` (-1: none)
int numeric_error(const char* what, int member) {
  if (member < 0) return 0;
  return fail(MSCKF_B200_ERR_NUMERIC, std::string(what) + ": non-finite delta-x or covariance entry (member " + std::to_string(member) + "); the update was applied");
}

// One member's aided update as k_aid takes it: up to 8 model items stacked into m rows (a single-model call or a LINEAR
// update is one item), each with its z and its own block of the block-diagonal R.  n_items = 0: the member is left alone.
struct AidJob {
  int m = 0, n_items = 0;
  mb::AidItem item[mb::kAidMaxItems] = {};
  const double* z[mb::kAidMaxItems] = {};  // (LINEAR: the residual r)
  int nz[mb::kAidMaxItems] = {};
  const double* R[mb::kAidMaxItems] = {};  // [rows][rows] of the item, row-major, lower triangle read
  const double* H = nullptr;               // LINEAR: [m][n]
  double chi2_max = 0.0;
};

// Checks one item of a stacked aided update against a window of M clones and appends it to j, its rows after j's: the check
// of every stack item and of msckf_b200_aid_update's four item models.  0, or MSCKF_B200_ERR_ARG.
int aid_append(AidJob& j, const msckf_b200_aid_item& q, int M, const std::string& w, const std::string& who) {
  int m = 0, nz = 3;
  switch (q.model) {
    case MSCKF_B200_AID_VELOCITY: case MSCKF_B200_AID_POSITION: m = 3; break;
    case MSCKF_B200_AID_POSE: m = 6; nz = 7; break;
    case MSCKF_B200_AID_CLONE_POSE:
      if (q.a < 0 || q.a >= M) return fail(MSCKF_B200_ERR_ARG, w + ": clone outside the window" + who);
      m = 6; nz = 7;
      break;
    case MSCKF_B200_AID_BODY_VELOCITY:
      if (q.a < 1 || q.a > 7) return fail(MSCKF_B200_ERR_ARG, w + ": the row mask must select rows 0..2" + who);
      m = (q.a & 1) + ((q.a >> 1) & 1) + ((q.a >> 2) & 1);
      break;
    case MSCKF_B200_AID_RELATIVE_POSE:
      if (q.a < 0 || q.a >= M || q.b < 0 || q.b >= M) return fail(MSCKF_B200_ERR_ARG, w + ": clone outside the window" + who);
      if (q.a == q.b) return fail(MSCKF_B200_ERR_ARG, w + ": a relative pose needs two different clones" + who);
      m = 6; nz = 7;
      break;
    case MSCKF_B200_AID_ANTENNA_POSITION: case MSCKF_B200_AID_CLONE_ANTENNA_POSITION:
    case MSCKF_B200_AID_HEADING: case MSCKF_B200_AID_CLONE_HEADING: {  // (the a / b they do not use must be 0)
      const bool clone = q.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION || q.model == MSCKF_B200_AID_CLONE_HEADING;
      const bool heading = q.model == MSCKF_B200_AID_HEADING || q.model == MSCKF_B200_AID_CLONE_HEADING;
      if (clone && (q.a < 0 || q.a >= M)) return fail(MSCKF_B200_ERR_ARG, w + ": clone outside the window" + who);
      const int mask = heading ? 1 : clone ? q.b : q.a;
      if (mask < 1 || mask > 7) return fail(MSCKF_B200_ERR_ARG, w + ": the row mask must select rows 0..2" + who);
      if ((!clone && heading && q.a != 0) || (q.model != MSCKF_B200_AID_CLONE_ANTENNA_POSITION && q.b != 0))
        return fail(MSCKF_B200_ERR_ARG, w + ": a / b the model does not use must be 0" + who);
      m = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);
      nz = heading ? 4 : 6;
      break;
    }
    case MSCKF_B200_AID_RANGE: case MSCKF_B200_AID_CLONE_RANGE:
    case MSCKF_B200_AID_PLANE_RANGE: case MSCKF_B200_AID_CLONE_PLANE_RANGE: {  // one row each (b and the IMU forms' a must be 0)
      const bool clone = q.model == MSCKF_B200_AID_CLONE_RANGE || q.model == MSCKF_B200_AID_CLONE_PLANE_RANGE;
      if (clone && (q.a < 0 || q.a >= M)) return fail(MSCKF_B200_ERR_ARG, w + ": clone outside the window" + who);
      if ((!clone && q.a != 0) || q.b != 0) return fail(MSCKF_B200_ERR_ARG, w + ": a / b the model does not use must be 0" + who);
      m = 1;
      nz = q.model == MSCKF_B200_AID_RANGE || q.model == MSCKF_B200_AID_CLONE_RANGE ? 7 : 8;
      break;
    }
    case MSCKF_B200_AID_GYRO_AT_REST: case MSCKF_B200_AID_ACCEL_AT_REST:  // three rows each (a and b must be 0)
      if (q.a != 0 || q.b != 0) return fail(MSCKF_B200_ERR_ARG, w + ": a / b the model does not use must be 0" + who);
      m = 3;
      break;
    default: return fail(MSCKF_B200_ERR_ARG, w + ": model not allowed in a stack" + who);
  }
  if (j.m + m > mb::kAidMaxRows) return fail(MSCKF_B200_ERR_ARG, w + ": more than 32 rows" + who);
  if (!q.z || !finite(q.z, nz)) return fail(MSCKF_B200_ERR_ARG, w + ": missing or non-finite z" + who);
  const bool pose = q.model == MSCKF_B200_AID_POSE || q.model == MSCKF_B200_AID_CLONE_POSE || q.model == MSCKF_B200_AID_RELATIVE_POSE;
  const bool heading = q.model == MSCKF_B200_AID_HEADING || q.model == MSCKF_B200_AID_CLONE_HEADING;
  const bool plane = q.model == MSCKF_B200_AID_PLANE_RANGE || q.model == MSCKF_B200_AID_CLONE_PLANE_RANGE;
  if (pose && !(q.z[3] * q.z[3] + q.z[4] * q.z[4] + q.z[5] * q.z[5] + q.z[6] * q.z[6] > 0.0))
    return fail(MSCKF_B200_ERR_ARG, w + ": zero quaternion" + who);
  if (heading && !(q.z[1] * q.z[1] + q.z[2] * q.z[2] + q.z[3] * q.z[3] > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": zero heading axis" + who);
  if (plane && !(q.z[5] * q.z[5] + q.z[6] * q.z[6] + q.z[7] * q.z[7] > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": zero beam axis" + who);
  if (!q.R) return fail(MSCKF_B200_ERR_ARG, w + ": missing R" + who);
  for (int r = 0; r < m; ++r)
    if (!finite(q.R + (size_t)r * m, r + 1)) return fail(MSCKF_B200_ERR_ARG, w + ": non-finite R" + who);
  const int k = j.n_items++;
  j.item[k] = {(short)q.model, (short)(q.model >= MSCKF_B200_AID_CLONE_POSE ? q.a : 0),  // (LINEAR is not an item model)
               (short)(q.model == MSCKF_B200_AID_RELATIVE_POSE || q.model == MSCKF_B200_AID_CLONE_ANTENNA_POSITION ? q.b : 0), (short)j.m};
  j.z[k] = q.z; j.nz[k] = nz; j.R[k] = q.R; j.m += m;
  return 0;
}

// tail kernel choice (engine option 3 / window size)
inline size_t tail_legacy_smem(int n, int NB) {
  const int ldt = (n + 3) & ~3;
  return sizeof(double) * ((size_t)2 * NB * (NB + 1) + 2 + (size_t)2 * NB * ldt + ((n + 1) & ~1) + 2 * NB) + 64;
}
inline int pick_tail(int n, bool no_fused) {
  const bool fused = (n + 1 + kTailCluster - 2) / (kTailCluster - 1) <= 32 &&  // (right-hand-side columns per worker CTA)
                     mb::tail_fused_smem_bytes(n) <= kSmemBudget && !no_fused;
  if (fused) return 0;
  if (tail_legacy_smem(n, 32) <= kSmemBudget) return 1;
  if (tail_legacy_smem(n, 16) <= kSmemBudget) return 2;
  return -1;
}
inline size_t tail_smem(int n, int kind) { return kind == 0 ? mb::tail_fused_smem_bytes(n) : tail_legacy_smem(n, kind == 1 ? 32 : 16); }

// grid / shared-memory shape of one (batched) update: what a captured graph is valid for
struct LaunchShape {
  int nf, mode, tri_gx, jac_gx, bd_gx, gram_gx, gram_gy, asm_gx, rows_gx, gemm_g, syrk_gx, tail_mask, pdl, gram_mma, jac_g, tail_nch,
      stop;  // option 8: the sequence ends after the compression
  unsigned tri_smem, jac_smem, rows_smem, inj_smem, tail_smem[3];
  const void* args;  // device address of the UpdArgs array (moves only when the input arena is re-allocated)
  bool operator==(const LaunchShape& o) const { return memcmp(this, &o, sizeof(*this)) == 0; }
};

struct EngineBase;
struct CtxBase {
  virtual ~CtxBase() {}
  virtual int stage(int mode, const msckf_b200_tracks* tracks, int threads) = 0;
  virtual int launch() = 0;
  virtual int launch_timed(float* ms) = 0;
  virtual int fetch(msckf_b200_report* reports) = 0;
  virtual int kernel_times(float* ms, const char** names, int cap) = 0;
  virtual void detach(EngineBase* e) = 0;
  virtual int count() const = 0;
  virtual EngineBase* member(int i) const = 0;
  // the state calls of every member as one launch per kernel (msckf_b200_batch_propagate_n / _augment / _prune / _get_state)
  virtual int propagate_n(const void* const* readings, const int* k) = 0;
  virtual int augment(const int* which) = 0;
  virtual int prune(const int* const* keep, const int* n_keep) = 0;
  virtual int get_state(void* const* imu, void* const* poses) = 0;
  // NEES of every member against caller-given truth (msckf_b200_nees / _batch_nees): read-only, one synchronisation
  virtual int nees(const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out) = 0;
  // aided measurement updates of the members (msckf_b200_aid_update / _batch_aid_update, and the stacked
  // msckf_b200_aid_stack_update / _batch_aid_stack_update): one launch per 32, one synchronisation
  virtual int aid(const msckf_b200_aid* in, msckf_b200_aid_result* out) = 0;
  // iter: the iterated form (msckf_b200_aid_stack_update_iter / ..._fde_iter and their batch forms), iter[i] and iout[i] per
  // member; nullptr: one linearisation
  virtual int aid_stack(const msckf_b200_aid_item* const* items, const int* n_items, double chi2_max, msckf_b200_aid_result* out,
                        const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) = 0;
  // the stacked form with fault detection and exclusion over the items (msckf_b200_aid_stack_update_fde / _batch_..._fde)
  virtual int aid_stack_fde(const msckf_b200_aid_item* const* items, const int* n_items, const msckf_b200_aid_fde* fde,
                            msckf_b200_aid_fde_result* out, const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) = 0;
  // standstill detection and the 9-row zero-motion stack (msckf_b200_standstill_update / _batch_standstill_update): the scatter
  // test on the host, then one launch per 32 members at rest, one synchronisation (none when no member is at rest)
  virtual int standstill(const void* const* readings, const int* k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out) = 0;
  // mapped-landmark updates of the members (msckf_b200_landmark_update / _batch_landmark_update): three launches per 32, one synchronisation
  // (cons, cout: the consensus of each member, or NULL)
  virtual int landmarks(const msckf_b200_landmarks* in, const msckf_b200_landmark_map* map, msckf_b200_landmark_result* out,
                        const msckf_b200_landmark_consensus* cons = nullptr, msckf_b200_landmark_consensus_result* cout = nullptr) = 0;
  cudaStream_t stream = nullptr;
  long long launches = 0;
  bool pending = false;
  // k_jac at the last launch's shape: threads per track, dynamic shared memory, CTAs resident per SM (msckf_b200_batch_jac_occupancy)
  int jac_g = 0, jac_ctas = 0;
  unsigned jac_smem = 0;
};

struct EngineBase {
  virtual ~EngineBase() {}
  virtual int initialize(const void*, const void*, const void*, const void*) = 0;
  virtual int propagate_n(const void*, int) = 0;
  virtual int augment() = 0;
  virtual int prune(const int*, int) = 0;
  virtual int get_state(void*, void*) = 0;
  virtual int get_covariance(void*) = 0;
  virtual int set_covariance(const void*) = 0;
  virtual int get_counters(long long*) = 0;
  virtual int last_dx(double*, int) = 0;
  virtual int rank_pivots(double*, int) = 0;
  virtual int stage_buffer(int, void*, int) = 0;
  virtual int copy_from(const EngineBase*) = 0;
  virtual int sync() = 0;
  virtual int input_buffer(int, int, msckf_b200_tracks*) = 0;
  virtual int tail_profile(unsigned long long* out, int cap) = 0;
  virtual CtxBase* solo_ctx() = 0;
  virtual void drop_graphs() = 0;
  void set_stream(cudaStream_t s) { stream = s; solo_ctx()->stream = s; }
  bool profile = false;
  bool use_graph = true;
  bool use_pdl = true;
  bool gram_mma = true;        // option 5: Gram products on the FP64 tensor-core path (DMMA) instead of SIMT DFMA tiles
  bool no_fused_tail = false;  // option 3 = 0: substitution as a separate sweep even where the fused form fits
  int tail_chains = 0;         // option 7: CTAs running the tail's chains of diagonal blocks (1, 2; 0 = 2 where the device takes clusters of 9)
  int jac_group = 0;           // option 6: threads per track in k_jac (32 / 64 / 128; 0 = by batch size)
  bool stop_after_compression = false;  // option 8: an update ends with T'', R'', r'' (msckf_b200_stage_buffer reads them)
  // the last launched update's sizes, for msckf_b200_stage_buffer (M < 0: none, or its buffers have been re-staged or reallocated
  // since); accept lives in the launching context's report arena
  struct StageRec { int N, O, M; const int* accept; } last_stage = {0, 0, -1, nullptr};
  int dtype = 0, device = 0, Mmax = 0, Tmax = 0, Omax = 0;
  int M = 0;
  double rank_thr = 1e-9;
  long long launches = 0;
  cudaStream_t stream = nullptr, own_stream = nullptr;
  CtxBase* group = nullptr;  // the batch this engine belongs to (nullptr: none)
  CtxBase* busy = nullptr;   // the context holding an un-fetched update of this engine
};

template <class S> struct Engine;

// per-filter slice of the packed arenas for one update
template <class S>
struct Plan {
  int N = 0, O = 0, Lmax = 0;
  size_t in_off = 0, rep_off = 0;
  int *h_off = nullptr, *h_idx = nullptr, *d_off = nullptr, *d_idx = nullptr;
  S *h_obs = nullptr, *h_pfg_in = nullptr, *d_obs = nullptr, *d_pfg_in = nullptr;
  int *h_mr = nullptr, *h_cmeff = nullptr, *h_cm = nullptr, *h_tri = nullptr, *h_valid = nullptr, *h_accept = nullptr;
  int *d_mr = nullptr, *d_cmeff = nullptr, *d_cm = nullptr, *d_tri = nullptr, *d_valid = nullptr, *d_accept = nullptr;
  S *h_pfg = nullptr, *h_gamma = nullptr, *d_pfg = nullptr, *d_gamma = nullptr;
  static size_t in_bytes(int N, int O) {
    return up16(sizeof(int) * ((size_t)N + 1)) + up16(sizeof(int) * (size_t)O) + up16(sizeof(S) * 2 * (size_t)O) + up16(sizeof(S) * 3 * (size_t)N);
  }
  static size_t rep_bytes(int N) {
    return up16(sizeof(int) * 4) + 5 * up16(sizeof(int) * (size_t)N) + up16(sizeof(S) * 3 * (size_t)N) + up16(sizeof(S) * (size_t)N);
  }
  void carve(const Arena& in, const Arena& rep) {
    size_t o = in_off;
    auto take = [&](const Arena& a, size_t bytes, void** hp, void** dp) { *hp = a.h + o; *dp = a.d + o; o += up16(bytes); };
    take(in, sizeof(int) * ((size_t)N + 1), (void**)&h_off, (void**)&d_off);
    take(in, sizeof(int) * (size_t)O, (void**)&h_idx, (void**)&d_idx);
    take(in, sizeof(S) * 2 * (size_t)O, (void**)&h_obs, (void**)&d_obs);
    take(in, sizeof(S) * 3 * (size_t)N, (void**)&h_pfg_in, (void**)&d_pfg_in);
    o = rep_off;
    take(rep, sizeof(int) * 4, (void**)&h_mr, (void**)&d_mr);  // m, rank, status, pad
    take(rep, sizeof(int) * (size_t)N, (void**)&h_cmeff, (void**)&d_cmeff);
    take(rep, sizeof(int) * (size_t)N, (void**)&h_cm, (void**)&d_cm);
    take(rep, sizeof(int) * (size_t)N, (void**)&h_tri, (void**)&d_tri);
    take(rep, sizeof(int) * (size_t)N, (void**)&h_valid, (void**)&d_valid);
    take(rep, sizeof(int) * (size_t)N, (void**)&h_accept, (void**)&d_accept);
    take(rep, sizeof(S) * 3 * (size_t)N, (void**)&h_pfg, (void**)&d_pfg);
    take(rep, sizeof(S) * (size_t)N, (void**)&h_gamma, (void**)&d_gamma);
  }
};

// A few persistent host threads that share the validation / packing of a batch's track arrays (spawning std::threads per call
// costs more than packing eight 100 KB batches).
struct WorkerPool {
  std::vector<std::thread> th;
  std::mutex mu;
  std::condition_variable cv_go, cv_done;
  std::function<void(int)> fn;
  int n_items = 0, next = 0, active = 0, gen = 0;
  bool quit = false;
  void start(int n) {
    for (int i = (int)th.size(); i < n; ++i) th.emplace_back([this] { loop(); });
  }
  void loop() {
    int seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> lk(mu);
      cv_go.wait(lk, [&] { return quit || gen != seen; });
      if (quit) return;
      seen = gen;
      while (next < n_items) {
        const int i = next++;
        lk.unlock();
        fn(i);
        lk.lock();
      }
      if (--active == 0) cv_done.notify_all();
    }
  }
  // run f(0..n-1) on the pool's threads plus the caller
  void run(int n, const std::function<void(int)>& f) {
    {
      std::lock_guard<std::mutex> lk(mu);
      fn = f; n_items = n; next = 0; active = (int)th.size(); gen++;
    }
    cv_go.notify_all();
    for (;;) {
      int i;
      { std::lock_guard<std::mutex> lk(mu); if (next >= n_items) break; i = next++; }
      f(i);
    }
    std::unique_lock<std::mutex> lk(mu);
    cv_done.wait(lk, [&] { return active == 0; });
  }
  ~WorkerPool() {
    { std::lock_guard<std::mutex> lk(mu); quit = true; }
    cv_go.notify_all();
    for (auto& t : th) t.join();
  }
};

// RAII guard: a failure between BeginCapture and EndCapture must not leave the stream in capture mode
struct CaptureGuard {
  cudaStream_t s;
  bool active = false;
  explicit CaptureGuard(cudaStream_t st) : s(st) {}
  int begin() {
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    active = true;
    return 0;
  }
  int end(cudaGraph_t* g) {
    active = false;
    CK(cudaStreamEndCapture(s, g));
    return 0;
  }
  ~CaptureGuard() {
    if (active) {
      cudaGraph_t g = nullptr;
      cudaStreamEndCapture(s, &g);
      if (g) cudaGraphDestroy(g);
      cudaGetLastError();
    }
  }
};

template <class S>
struct Ctx : CtxBase {
  std::vector<Engine<S>*> eng;
  std::vector<Plan<S>> plan;
  // The update's inputs and reports: a staged or launched update lives in them across calls (and the class packs its tracks
  // into `in` through msckf_b200_input_buffer before stage), so no other call may use them.
  Arena in, rep;
  // The side calls (get_state, nees, aid, landmarks) copy in, launch, copy back and synchronise before they return, so no two
  // are ever live at once: they share one pinned block for their inputs and results, and one device workspace.
  Arena io;
  DevBuf ws;
  size_t in_used = 0, rep_used = 0;
  int device = 0;
  bool owns_stream = false;
  cudaStream_t stream2 = nullptr, stream3 = nullptr;  // side branches of the update (k_blockdiag, k_rows run beside k_gram)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_join2 = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  int st_mode = -1;
  bool staged = false, timed_region = false, st_stop = false;  // st_stop: option 8 of every member
  WorkerPool pool;
  // graph cache
  struct Cached { LaunchShape shape; cudaGraphExec_t exec; int nodes; unsigned long long stamp; };
  std::vector<Cached> graphs;
  std::vector<LaunchShape> seen;  // shapes launched directly once: captured the second time
  unsigned long long tick = 0;
  // optional per-kernel CUDA-event profile of the last launch (option key 1 of the first member)
  static constexpr int kMaxEv = 24;
  cudaEvent_t ev[kMaxEv] = {};
  const char* ev_name[kMaxEv] = {};
  int n_ev = 0;

  int init(int dev) {
    device = dev;
    CK(cudaSetDevice(device));
    CK(cudaStreamCreateWithFlags(&stream2, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&stream3, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_join2, cudaEventDisableTiming));
    return 0;
  }
  ~Ctx() override {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    drop_graphs();
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (ev_join2) cudaEventDestroy(ev_join2);
    if (ev_t0) cudaEventDestroy(ev_t0);
    if (ev_t1) cudaEventDestroy(ev_t1);
    if (stream2) cudaStreamDestroy(stream2);
    if (stream3) cudaStreamDestroy(stream3);
    if (owns_stream && stream) cudaStreamDestroy(stream);
  }
  void drop_graphs() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.exec);
    graphs.clear(); seen.clear();
  }
  int count() const override { return (int)eng.size(); }
  EngineBase* member(int i) const override;
  void detach(EngineBase* e) override;
  bool profile() const;
  void mark(const char* name) {
    if (!profile() || n_ev >= kMaxEv) return;
    if (!ev[n_ev]) cudaEventCreate(&ev[n_ev]);
    cudaEventRecord(ev[n_ev], stream);
    ev_name[n_ev] = name;
    n_ev++;
  }
  size_t args_bytes() const { return up256(sizeof(mb::UpdArgs<S>) * eng.size()); }
  mb::UpdArgs<S>* h_args() const { return reinterpret_cast<mb::UpdArgs<S>*>(in.h); }
  mb::UpdArgs<S>* d_args() const { return reinterpret_cast<mb::UpdArgs<S>*>(in.d); }

  int layout(const std::vector<std::pair<int, int>>& NO);
  int stage(int mode, const msckf_b200_tracks* tracks, int threads) override;
  int launch() override;
  int run_kernels(const LaunchShape& sh);
  int launch_timed(float* ms) override;
  int fetch(msckf_b200_report* reports) override;
  int members_ready(const char* what) const;
  // the launching halves of the state calls, for a batch and for the single filter's own calls (each checks its arguments first)
  int enqueue_propagate_n(const void* const* readings, const int* k);
  int enqueue_augment(const std::vector<int>& idx);
  int enqueue_prune(const std::vector<int>& idx, const int* const* keep, const int* n_keep);
  int read_state(void* const* imu, void* const* poses);
  // The one launch path of the per-member kernels.  args(i) gives member i's arguments; launch(a, nm) launches once for an
  // mb::Members<Args, NM> a filled with nm members.  NM = 1 when the context has one member (a single filter, or a batch of
  // one), else mb::kBatchMembers with one launch per chunk of that many.  counted: every launch counts on the context and on
  // the engine of each member it runs (the state calls).
  template <class ArgsOf, class Launch>
  void per_member(const std::vector<int>& idx, bool counted, ArgsOf&& args, Launch&& launch) {
    if (eng.size() == 1) chunks<1>(idx, counted, args, launch);
    else chunks<mb::kBatchMembers>(idx, counted, args, launch);
  }
  template <int NM, class ArgsOf, class Launch>
  void chunks(const std::vector<int>& idx, bool counted, ArgsOf& args, Launch& launch) {
    for (size_t c = 0; c < idx.size(); c += NM) {
      const int nm = (int)std::min<size_t>(NM, idx.size() - c);
      mb::Members<decltype(args(0)), NM> a;
      for (int j = 0; j < nm; ++j) {
        a.m[j] = args(idx[c + j]);
        if (counted) eng[idx[c + j]]->launches++;
      }
      launch(a, nm);
      if (counted) launches++;
    }
  }
  int propagate_n(const void* const* readings, const int* k) override;
  int augment(const int* which) override;
  int prune(const int* const* keep, const int* n_keep) override;
  int get_state(void* const* imu, void* const* poses) override;
  int nees(const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out) override;
  int aid(const msckf_b200_aid* in, msckf_b200_aid_result* out) override;
  int aid_stack(const msckf_b200_aid_item* const* items, const int* n_items, double chi2_max, msckf_b200_aid_result* out,
                const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) override;
  int aid_stack_fde(const msckf_b200_aid_item* const* items, const int* n_items, const msckf_b200_aid_fde* fde,
                    msckf_b200_aid_fde_result* out, const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) override;
  int aid_stack_jobs(const msckf_b200_aid_item* const* items, const int* n_items, const std::string& w, std::vector<AidJob>& job,
                     const msckf_b200_aid_iter* iter);
  int standstill(const void* const* readings, const int* k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out) override;
  int aid_run(const std::vector<AidJob>& job, msckf_b200_aid_result* out, const char* what, const msckf_b200_aid_fde* fde = nullptr,
              msckf_b200_aid_fde_result* fout = nullptr, const msckf_b200_aid_iter* iter = nullptr,
              msckf_b200_aid_iter_result* iout = nullptr);
  int landmarks(const msckf_b200_landmarks* in, const msckf_b200_landmark_map* map, msckf_b200_landmark_result* out,
                const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_consensus_result* cout) override;
  int kernel_times(float* ms, const char** names, int cap) override {
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    int k = 0;
    for (int i = 1; i < n_ev && k < cap; ++i, ++k) {
      CK(cudaEventElapsedTime(&ms[k], ev[i - 1], ev[i]));
      names[k] = ev_name[i];
    }
    return k;
  }
};

template <class S>
struct Engine : EngineBase {
  // resident state
  mb::DevState<S>* d_st = nullptr;
  S *d_P = nullptr, *d_P2 = nullptr, *d_poses = nullptr, *d_poses2 = nullptr;
  // workspaces
  int *d_src = nullptr, *d_rows = nullptr, *d_rowoff = nullptr, *d_keep = nullptr;
  unsigned long long* d_csnap = nullptr;
  unsigned long long* d_prof = nullptr;
  unsigned* d_done = nullptr;  // k_jac's CTA ticket counter
  S *d_Xg = nullptr, *d_rg = nullptr, *d_Vg = nullptr, *d_taug = nullptr;
  double *d_Z = nullptr, *d_Yq = nullptr, *d_ur = nullptr, *d_G1p = nullptr, *d_G2p = nullptr, *d_D1 = nullptr, *d_D2 = nullptr,
         *d_bb = nullptr, *d_T2 = nullptr, *d_R2 = nullptr, *d_r2 = nullptr, *d_TP = nullptr, *d_S2 = nullptr, *d_W = nullptr, *d_G = nullptr,
         *d_y = nullptr, *d_dx = nullptr, *d_idiag = nullptr, *d_pivr = nullptr;
  mb::DevState<S>* h_st = nullptr;
  int nmax = 0, ldp = 0, ld = 0;
  mutable int pivr_n = 0;  // dimension of the last update that made a rank decision (msckf_b200_rank_pivots)
  bool initialized = false;
  Ctx<S> solo;

  CtxBase* solo_ctx() override { return &solo; }
  void drop_graphs() override { solo.drop_graphs(); if (group) static_cast<Ctx<S>*>(group)->drop_graphs(); }

  static int& tail9_clusters() { static int v = 0; return v; }  // co-resident clusters of 9 (0: not available)
  // CTAs of k_jac with g threads per track resident per SM at `smem` bytes of dynamic shared memory (0: not available)
  static int jac_ctas_per_sm(int g, unsigned smem) {
    auto kj = g == 32 ? mb::k_jac<S, 32> : (g == 64 ? mb::k_jac<S, 64> : mb::k_jac<S, 128>);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kj, g == 32 ? 64 : 128, smem) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
  }
  static int set_func_attrs(int dev) {
    static bool done[64] = {};  // (per scalar type and device: function attributes belong to the device's context)
    if (dev < 0 || dev >= 64) return fail(MSCKF_B200_ERR_ARG, "device index");
    if (done[dev]) return 0;
    CK(cudaFuncSetAttribute(mb::k_tri<S, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_jac<S, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_jac<S, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_jac<S, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    // k_jac's occupancy is set by shared memory: ask for the largest carveout, not just enough for one CTA
    CK(cudaFuncSetAttribute(mb::k_jac<S, 128>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CK(cudaFuncSetAttribute(mb::k_jac<S, 64>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CK(cudaFuncSetAttribute(mb::k_jac<S, 32>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CK(cudaFuncSetAttribute(mb::k_tail_fused<S, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_tail_fused<S, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    // the two-chain form runs in clusters of 9 (2 chain CTAs + 7 workers): a non-portable size; use it where the device takes it
    if (cudaFuncSetAttribute(mb::k_tail_fused<S, 2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(kTailCluster + 1, 1, 1); cfg.blockDim = dim3(mb::kTailThreads); cfg.dynamicSmemBytes = kSmemBudget;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = kTailCluster + 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int ncl = 0;
      if (cudaOccupancyMaxActiveClusters(&ncl, mb::k_tail_fused<S, 2>, &cfg) == cudaSuccess && ncl > 0) tail9_clusters() = ncl;
    }
    cudaGetLastError();
    CK(cudaFuncSetAttribute(mb::k_tail<S, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_tail<S, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    CK(cudaFuncSetAttribute(mb::k_aid<S, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid<S, mb::kBatchMembers>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid<S, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid<S, mb::kBatchMembers, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid_iter<S, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid_iter<S, mb::kBatchMembers>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid_iter<S, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    CK(cudaFuncSetAttribute(mb::k_aid_iter<S, mb::kBatchMembers, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAidSmemMax));
    done[dev] = true;
    return 0;
  }

  // ---- allocation: resident state (sized by Mmax), per-window workspaces (Mmax), per-batch workspaces (Tmax, Omax, Mmax)
  void free_window() {
    for (double** p : {&d_T2, &d_R2, &d_TP, &d_S2, &d_W, &d_G, &d_r2, &d_idiag, &d_pivr, &d_y, &d_dx, &d_D1, &d_D2, &d_bb}) { if (*p) cudaFree(*p); *p = nullptr; }
    if (d_keep) { cudaFree(d_keep); d_keep = nullptr; }
  }
  void free_batchws() {
    for (int** p : {&d_src, &d_rows, &d_rowoff}) { if (*p) cudaFree(*p); *p = nullptr; }
    for (S** p : {&d_Xg, &d_rg, &d_Vg, &d_taug}) { if (*p) cudaFree(*p); *p = nullptr; }
    for (double** p : {&d_Z, &d_Yq, &d_ur, &d_G1p, &d_G2p}) { if (*p) cudaFree(*p); *p = nullptr; }
  }
  int alloc_window() {
    for (double** p : {&d_T2, &d_R2, &d_TP, &d_S2, &d_W}) CK(cudaMalloc(p, sizeof(double) * (size_t)ld * nmax));
    // Gamma / the tail kernel's L2 scratch (double-buffered 32 x 34 inverses + two transposed 32-row panels): at least that big
    CK(cudaMalloc(&d_G, sizeof(double) * std::max((size_t)ld * nmax, (size_t)4 * 32 * 34 + (size_t)64 * (ld + 4))));
    CK(cudaMalloc(&d_r2, sizeof(double) * nmax));
    CK(cudaMalloc(&d_idiag, sizeof(double) * 2 * nmax));
    CK(cudaMalloc(&d_pivr, sizeof(double) * 2 * nmax));  // pivots | original diagonal
    CK(cudaMemsetAsync(d_pivr, 0, sizeof(double) * 2 * nmax, stream));
    CK(cudaMalloc(&d_y, sizeof(double) * nmax));
    CK(cudaMalloc(&d_dx, sizeof(double) * nmax));
    CK(cudaMemsetAsync(d_dx, 0, sizeof(double) * nmax, stream));
    CK(cudaMalloc(&d_D1, sizeof(double) * 36 * Mmax));
    CK(cudaMalloc(&d_D2, sizeof(double) * 36 * Mmax));
    CK(cudaMalloc(&d_bb, sizeof(double) * 6 * Mmax));
    CK(cudaMalloc(&d_keep, sizeof(int) * nmax));
    return 0;
  }
  int alloc_batchws() {
    const size_t T = Tmax, O = Omax, cmax = 6 * (size_t)Mmax;
    for (int** p : {&d_src, &d_rows}) CK(cudaMalloc(p, sizeof(int) * T));
    CK(cudaMalloc(&d_rowoff, sizeof(int) * (T + 1)));
    CK(cudaMalloc(&d_Xg, sizeof(S) * 12 * O));
    CK(cudaMalloc(&d_rg, sizeof(S) * 2 * O));
    CK(cudaMalloc(&d_Vg, sizeof(S) * 6 * O));
    CK(cudaMalloc(&d_taug, sizeof(S) * 3 * T));
    CK(cudaMalloc(&d_Z, sizeof(double) * 3 * T * cmax));
    CK(cudaMalloc(&d_Yq, sizeof(double) * 3 * T * cmax));
    CK(cudaMalloc(&d_ur, sizeof(double) * 3 * T));
    CK(cudaMalloc(&d_G1p, sizeof(double) * kMaxSplit * cmax * cmax));
    CK(cudaMalloc(&d_G2p, sizeof(double) * (kMaxSplit * cmax * cmax + kMaxSplit * cmax)));  // + the Z^T u partials
    return 0;
  }
  void set_dims() {
    nmax = 15 + 6 * Mmax;
    ldp = (nmax + 3) & ~3;
    ld = (nmax + 1) & ~1;
  }
  int alloc() {
    set_dims();
    CK(cudaSetDevice(device));
    CK(cudaStreamCreateWithFlags(&own_stream, cudaStreamNonBlocking));
    stream = own_stream;
    RC(solo.init(device));
    solo.stream = stream;
    solo.eng.assign(1, this);
    solo.plan.resize(1);
    CK(cudaMalloc(&d_st, sizeof(mb::DevState<S>)));
    CK(cudaMalloc(&d_P, sizeof(S) * (size_t)ldp * nmax));
    CK(cudaMalloc(&d_P2, sizeof(S) * (size_t)ldp * nmax));
    CK(cudaMalloc(&d_poses, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1)));
    CK(cudaMalloc(&d_poses2, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1)));
    CK(cudaMemsetAsync(d_P, 0, sizeof(S) * (size_t)ldp * nmax, stream));
    CK(cudaMemsetAsync(d_P2, 0, sizeof(S) * (size_t)ldp * nmax, stream));
    CK(cudaMemsetAsync(d_poses, 0, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1), stream));
    CK(cudaMemsetAsync(d_poses2, 0, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1), stream));
    CK(cudaMalloc(&d_csnap, sizeof(unsigned long long)));
    CK(cudaMalloc(&d_prof, sizeof(unsigned long long) * 80));
    CK(cudaMalloc(&d_done, sizeof(unsigned)));
    CK(cudaMemsetAsync(d_done, 0, sizeof(unsigned), stream));
    CK(cudaMemsetAsync(d_prof, 0, sizeof(unsigned long long) * 80, stream));
    RC(alloc_window());
    RC(alloc_batchws());
    // the private context's packed arenas, sized for a full batch and a full window (no pinned allocation inside the first
    // update or get_state)
    RC(solo.in.ensure(solo.args_bytes() + up256(Plan<S>::in_bytes(Tmax, Omax)), nullptr));
    RC(solo.rep.ensure(up256(Plan<S>::rep_bytes(Tmax)), nullptr));
    RC(solo.io.ensure(up16(sizeof(S) * mb::kPoseStride * Mmax), nullptr));
    CK(cudaMallocHost(&h_st, sizeof(mb::DevState<S>)));
    memset(h_st, 0, sizeof(mb::DevState<S>));
    RC(set_func_attrs(device));
    CK(cudaStreamSynchronize(stream));
    return 0;
  }
  ~Engine() override {
    cudaSetDevice(device);
    if (group) group->detach(this);
    if (stream) cudaStreamSynchronize(stream);
    if (own_stream) cudaStreamSynchronize(own_stream);
    free_window(); free_batchws();
    void* dv[] = {d_st, d_P, d_P2, d_poses, d_poses2, d_csnap, d_prof, d_done};
    for (void* p : dv) if (p) cudaFree(p);
    if (h_st) cudaFreeHost(h_st);
    solo.stream = nullptr;  // owned here
    if (own_stream) cudaStreamDestroy(own_stream);
  }

  // the reference's window is an unbounded std::vector: grow instead of failing (ADVICE r01)
  int ensure_clones(int need) {
    if (need <= Mmax) return 0;
    if (need > kMaxClonesHard) return fail(MSCKF_B200_ERR_CAPACITY, "sliding window exceeds the engine's hard limit of " + std::to_string(kMaxClonesHard) + " clones");
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    const int old_ldp = ldp, old_nmax = nmax, old_M = Mmax;
    last_stage.M = -1;
    Mmax = std::min(kMaxClonesHard, std::max(need, 2 * Mmax));
    set_dims();
    S *nP = nullptr, *nP2 = nullptr, *nposes = nullptr, *nposes2 = nullptr;
    CK(cudaMalloc(&nP, sizeof(S) * (size_t)ldp * nmax));
    CK(cudaMalloc(&nP2, sizeof(S) * (size_t)ldp * nmax));
    CK(cudaMalloc(&nposes, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1)));
    CK(cudaMalloc(&nposes2, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1)));
    CK(cudaMemsetAsync(nP, 0, sizeof(S) * (size_t)ldp * nmax, stream));
    CK(cudaMemsetAsync(nP2, 0, sizeof(S) * (size_t)ldp * nmax, stream));
    CK(cudaMemsetAsync(nposes, 0, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1), stream));
    CK(cudaMemsetAsync(nposes2, 0, sizeof(S) * mb::kPoseStride * (size_t)(Mmax + 1), stream));
    CK(cudaMemcpy2DAsync(nP, sizeof(S) * ldp, d_P, sizeof(S) * old_ldp, sizeof(S) * old_nmax, old_nmax, cudaMemcpyDeviceToDevice, stream));
    CK(cudaMemcpyAsync(nposes, d_poses, sizeof(S) * mb::kPoseStride * (size_t)(old_M + 1), cudaMemcpyDeviceToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    cudaFree(d_P); cudaFree(d_P2); cudaFree(d_poses); cudaFree(d_poses2);
    d_P = nP; d_P2 = nP2; d_poses = nposes; d_poses2 = nposes2;
    free_window(); free_batchws();
    RC(alloc_window());
    RC(alloc_batchws());
    CK(cudaStreamSynchronize(stream));
    return 0;
  }
  int ensure_tracks(int T, int O) {
    if (T <= Tmax && O <= Omax) return 0;
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    if (T > Tmax) Tmax = std::max(T, 2 * Tmax);
    if (O > Omax) Omax = std::max(O, 2 * Omax);
    last_stage.M = -1;
    free_batchws();
    RC(alloc_batchws());
    return 0;
  }
  // option 8: every compression workspace NaN (bytes 0xFF), so that an element no kernel of the update writes reads as NaN
  int poison_compression(cudaStream_t s) {
    const size_t T = Tmax, cmax = 6 * (size_t)Mmax;
    const std::pair<double*, size_t> ws[] = {
        {d_Z, 3 * T * cmax}, {d_Yq, 3 * T * cmax}, {d_ur, 3 * T}, {d_G1p, kMaxSplit * cmax * cmax},
        {d_G2p, kMaxSplit * cmax * cmax + kMaxSplit * cmax} /* + bzp */, {d_D1, 36 * (size_t)Mmax}, {d_D2, 36 * (size_t)Mmax},
        {d_bb, 6 * (size_t)Mmax}, {d_T2, (size_t)ld * nmax}, {d_R2, (size_t)ld * nmax}, {d_r2, (size_t)nmax}};
    for (const auto& w : ws) CK(cudaMemsetAsync(w.first, 0xFF, sizeof(double) * w.second, s));
    return 0;
  }

  int initialize(const void* cam_, const void* noise_, const void* params_, const void* imu_) override {
    const S* cam = (const S*)cam_; const S* nz = (const S*)noise_; const S* pr = (const S*)params_; const S* im = (const S*)imu_;
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    mb::DevState<S>& s = *h_st;
    memset(&s, 0, sizeof(s));
    for (int i = 0; i < 4; ++i) s.q_CI[i] = cam[i];
    for (int i = 0; i < 3; ++i) s.p_C_I[i] = cam[4 + i];
    s.u_var = nz[0]; s.v_var = nz[1];
    for (int i = 0; i < 144; ++i) s.Q_imu[i] = nz[2 + i];
    s.max_gn_cost_norm = pr[0]; s.translation_threshold = pr[1];
    for (int i = 0; i < 3; ++i) {
      s.p_I_G[i] = im[i]; s.v_I_G[i] = im[3 + i]; s.b_g[i] = im[6 + i]; s.b_a[i] = im[9 + i]; s.g[i] = im[12 + i];
      s.p_I_G_null[i] = im[i]; s.v_I_G_null[i] = im[3 + i];
    }
    for (int i = 0; i < 4; ++i) { s.q_IG[i] = im[15 + i]; s.q_IG_null[i] = im[15 + i]; }
    for (int i = 0; i < 99; ++i) s.chi2[i] = (S)kChi2_005[i];  // msckf.h:91-95
    CK(cudaMemcpyAsync(d_st, h_st, sizeof(s), cudaMemcpyHostToDevice, stream));
    // imu_covar_ = initial_imu_covar (msckf.h:86)
    std::vector<S> P0((size_t)ldp * 15, S(0));
    for (int i = 0; i < 15; ++i)
      for (int j = 0; j < 15; ++j) P0[(size_t)i * ldp + j] = nz[146 + 15 * i + j];
    CK(cudaMemsetAsync(d_P, 0, sizeof(S) * (size_t)ldp * nmax, stream));
    CK(cudaMemcpyAsync(d_P, P0.data(), sizeof(S) * P0.size(), cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    M = 0;
    initialized = true;
    if (busy) { busy->pending = false; busy = nullptr; }
    return 0;
  }

  int propagate_n(const void* r_, int k) override {
    if (!initialized) return fail(MSCKF_B200_ERR_STATE, "propagate before initialize");
    if (k < 0 || (k > 0 && !r_)) return fail(MSCKF_B200_ERR_ARG, "propagate_n: bad arguments");
    return solo.enqueue_propagate_n(&r_, &k);
  }
  // k_propagate's arguments for readings k0 .. k0 + n - 1 of r (n <= kPropMax)
  mb::PropBatch<S> prop_args(const S* r, int k0, int n) const {
    mb::PropBatch<S> pb;
    pb.st = d_st; pb.P = d_P; pb.ldp = ldp; pb.M = M; pb.k = n; pb.pad_ = 0;
    pb.prof = profile ? d_prof : nullptr;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < 7; ++j) pb.r[i][j] = r[7 * (size_t)(k0 + i) + j];
    return pb;
  }

  int augment() override {
    if (!initialized) return fail(MSCKF_B200_ERR_STATE, "augment before initialize");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "augment with an un-fetched update pending");
    return solo.enqueue_augment({0});
  }
  mb::AugArgs<S> aug_args() const { return {d_st, d_P, d_poses, ldp, M}; }
  // k_nees's arguments; truth / W / out are device addresses in the calling context's buffers
  mb::NeesArgs<S> nees_args(const double* truth, bool full, double* W, mb::NeesOut* out) const {
    return {d_st, d_P, d_poses, truth, W, out, ldp, M, full ? 15 + 6 * M : 15, full ? 1 : 0};
  }
  // k_aid's arguments; in / ws / out are device addresses in the calling context's buffers (ws = nullptr: shared memory)
  mb::AidArgs<S> aid_args(const AidJob& q, const double* in, double* ws, mb::AidOut* out) const {
    mb::AidArgs<S> a = {d_st, d_P, d_poses, in, ws, out, q.chi2_max, ldp, M, q.m, q.n_items, {}};
    for (int k = 0; k < q.n_items; ++k) a.item[k] = q.item[k];
    return a;
  }
  // the landmark kernels' arguments except the device addresses, which the calling context fills in
  mb::LmkArgs<S> lmk_args(const msckf_b200_landmarks& q, int G, int ld) const {
    mb::LmkArgs<S> a;
    memset(&a, 0, sizeof(a));
    a.st = d_st; a.P = d_P; a.poses = d_poses;
    if (q.R) { a.R[0] = q.R[0]; a.R[1] = q.R[1]; a.R[2] = q.R[2]; a.use_R = 1; }
    a.chi2 = q.chi2_obs; a.ldp = ldp; a.M = M; a.G = G; a.ld = ld; a.ntiles = mb::lmk_tiles(15 + 6 * M);
    return a;
  }

  // everything the kernels need for this filter's slice of the update
  void fill_args(mb::UpdArgs<S>& a, const Plan<S>& p, int mode) const {
    memset(&a, 0, sizeof(a));
    a.n_tracks = p.N; a.M = M; a.Lmax = p.Lmax; a.ldp = ldp; a.ld = ld; a.n = 15 + 6 * M; a.mode = mode;
    a.K = 3 * p.N;
    int nsplit = std::max(1, std::min(kMaxSplit, a.K / 96));
    int kchunk = (a.K + nsplit - 1) / nsplit;
    kchunk = (kchunk + mb::GK - 1) / mb::GK * mb::GK;
    if (kchunk < mb::GK) kchunk = mb::GK;
    nsplit = std::max(1, (a.K + kchunk - 1) / kchunk);
    a.nsplit = nsplit; a.kchunk = kchunk;
    // FP64 tensor-core Gram products where they win (measured, DESIGN.md 4.4): >= 200 tracks.  The choice depends on the
    // filter's own batch only, never on how many filters share a launch: a device batch stays bit-identical to separate calls.
    a.gram_mma = (gram_mma && p.N >= 200) ? 1 : 0;
    a.tail_kind = pick_tail(a.n, no_fused_tail);
    a.rank_thr = rank_thr;
    a.obs_off = p.d_off; a.obs = p.d_obs; a.clone_idx = p.d_idx; a.pfg_given = p.d_pfg_in;
    a.poses = d_poses; a.P = d_P; a.st = d_st;
    a.m_out = p.d_mr; a.rank_out = p.d_mr + 1;
    a.cm_eff = p.d_cmeff; a.cm_ok = p.d_cm; a.tri_ok = p.d_tri; a.valid = p.d_valid; a.accept = p.d_accept; a.pfg = p.d_pfg; a.gamma = p.d_gamma;
    a.counter_snap = d_csnap; a.src = d_src; a.rows = d_rows; a.row_off = d_rowoff; a.done = d_done;
    a.Xg = d_Xg; a.rg = d_rg; a.Vg = d_Vg; a.taug = d_taug; a.Z = d_Z; a.Yq = d_Yq; a.ur = d_ur;
    a.G1p = d_G1p; a.G2p = d_G2p; a.bzp = d_G2p + (size_t)kMaxSplit * 6 * Mmax * 6 * Mmax; a.D1 = d_D1; a.D2 = d_D2; a.bb = d_bb;
    a.T2 = d_T2; a.R2 = d_R2; a.r2 = d_r2; a.TP = d_TP; a.S2 = d_S2; a.W = d_W; a.G = d_G; a.y = d_y; a.dx = d_dx; a.idiag = d_idiag; a.pivr = d_pivr;
    a.keep = d_keep;
    a.prof = profile ? d_prof : nullptr;
  }

  int input_buffer(int N, int O, msckf_b200_tracks* out) override {
    if (!out || N < 0 || O < 0) return fail(MSCKF_B200_ERR_ARG, "input_buffer: bad arguments");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "previous update not fetched");
    CK(cudaSetDevice(device));
    RC(solo.layout({{N, O}}));
    const Plan<S>& p = solo.plan[0];
    out->n_tracks = N; out->obs_offset = p.h_off; out->obs = p.h_obs; out->clone_index = p.h_idx; out->p_f_G = p.h_pfg_in;
    return 0;
  }

  int prune(const int* keep, int n_keep) override {
    RC(prune_check(keep, n_keep));
    if (n_keep == M) return 0;
    return solo.enqueue_prune({0}, &keep, &n_keep);
  }
  int prune_check(const int* keep, int n_keep) const {
    if (n_keep < 0 || n_keep > M) return fail(MSCKF_B200_ERR_ARG, "prune: bad keep count");
    if (n_keep > 0 && !keep) return fail(MSCKF_B200_ERR_ARG, "prune: null keep list");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "prune with an un-fetched update pending");
    for (int i = 0; i < n_keep; ++i)
      if (keep[i] < 0 || keep[i] >= M || (i && keep[i] <= keep[i - 1])) return fail(MSCKF_B200_ERR_ARG, "prune: keep[] must be ascending positions");
    return 0;
  }
  mb::GatherArgs<S> gather_args(const int* keep, int n_keep) const {
    mb::GatherArgs<S> g;
    g.Pold = d_P; g.Pnew = d_P2; g.poses_old = d_poses; g.poses_new = d_poses2;
    g.n_new = 15 + 6 * n_keep; g.ldp = ldp;
    g.kl.n = n_keep;
    for (int i = 0; i < n_keep; ++i) g.kl.idx[i] = keep[i];
    return g;
  }
  void prune_swap(int n_keep) {
    std::swap(d_P, d_P2);      // (buffer addresses ride in UpdArgs, not in captured kernel arguments:
    std::swap(d_poses, d_poses2);  //  no synchronisation, and captured graphs stay valid)
    M = n_keep;
  }

  int get_state(void* imu_, void* poses_) override { return solo.read_state(&imu_, &poses_); }
  // get_state in two halves: enqueue the copies (IMU state into h_st, kPoseStride * M clone-pose scalars into raw_poses),
  // and, once the stream has been synchronised, convert them into the C-ABI's layouts
  int state_copy(bool imu, S* raw_poses) {
    if (imu) CK(cudaMemcpyAsync(h_st, d_st, sizeof(mb::DevState<S>), cudaMemcpyDeviceToHost, stream));
    if (raw_poses && M > 0) CK(cudaMemcpyAsync(raw_poses, d_poses, sizeof(S) * mb::kPoseStride * M, cudaMemcpyDeviceToHost, stream));
    return 0;
  }
  void state_unpack(void* imu_, void* poses_, const S* raw_poses) const {
    if (imu_) {
      S* o = (S*)imu_;
      const mb::DevState<S>& s = *h_st;
      for (int i = 0; i < 3; ++i) {
        o[i] = s.p_I_G[i]; o[3 + i] = s.v_I_G[i]; o[6 + i] = s.b_g[i]; o[9 + i] = s.b_a[i]; o[12 + i] = s.g[i];
        o[19 + i] = s.p_I_G_null[i]; o[22 + i] = s.v_I_G_null[i];
      }
      for (int i = 0; i < 4; ++i) { o[15 + i] = s.q_IG[i]; o[25 + i] = s.q_IG_null[i]; }
    }
    if (poses_ && M > 0) {
      S* o = (S*)poses_;
      for (int k = 0; k < M; ++k) {
        const S* p = raw_poses + mb::kPoseStride * k;
        o[7 * k] = p[4]; o[7 * k + 1] = p[5]; o[7 * k + 2] = p[6];
        o[7 * k + 3] = p[0]; o[7 * k + 4] = p[1]; o[7 * k + 5] = p[2]; o[7 * k + 6] = p[3];
      }
    }
  }

  int get_covariance(void* out) override {
    CK(cudaSetDevice(device));
    const int n = 15 + 6 * M;
    CK(cudaMemcpy2DAsync(out, sizeof(S) * n, d_P, sizeof(S) * ldp, sizeof(S) * n, n, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    return n;
  }

  int set_covariance(const void* in) override {
    if (!in) return fail(MSCKF_B200_ERR_ARG, "null argument");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "set_covariance with an un-fetched update pending");
    CK(cudaSetDevice(device));
    const int n = 15 + 6 * M;
    CK(cudaMemcpy2DAsync(d_P, sizeof(S) * ldp, in, sizeof(S) * n, sizeof(S) * n, n, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));  // `in` is caller memory
    return 0;
  }

  int get_counters(long long* c) override {
    CK(cudaSetDevice(device));
    CK(cudaMemcpyAsync(h_st, d_st, sizeof(mb::DevState<S>), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    c[0] = (long long)h_st->num_residualized; c[1] = (long long)h_st->pfg_shifted; c[2] = (long long)h_st->pfg_oob;
    c[3] = (long long)h_st->n_updates; c[4] = h_st->last_m; c[5] = h_st->last_rank; c[6] = h_st->last_status; c[7] = 0;
    return 0;
  }

  int rank_pivots(double* out, int cap) override {
    CK(cudaSetDevice(device));
    const int n = pivr_n;  // dimension of the last update (0: none yet)
    if (n <= 0) return 0;
    std::vector<double> tmp(2 * (size_t)n);
    CK(cudaMemcpyAsync(tmp.data(), d_pivr, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    for (int i = 0; i < std::min(n, cap); ++i) out[i] = tmp[n + i] > 0.0 ? tmp[i] / tmp[n + i] : 0.0;
    return n;
  }
  int stage_buffer(int which, void* out, int cap) override {
    if (busy) return fail(MSCKF_B200_ERR_STATE, "stage_buffer with an un-fetched update pending");
    if (which < MSCKF_B200_STAGE_T2 || which > MSCKF_B200_STAGE_ROW_OFF) return fail(MSCKF_B200_ERR_ARG, "stage_buffer: unknown buffer");
    if (cap < 0 || (cap > 0 && !out)) return fail(MSCKF_B200_ERR_ARG, "stage_buffer: bad arguments");
    const StageRec& r = last_stage;
    if (r.M < 0) return 0;
    const int n = 15 + 6 * r.M, c = 6 * r.M, N = r.N, O = r.O;
    const void* src = nullptr;
    size_t count = 0, elem = sizeof(double);
    switch (which) {
      case MSCKF_B200_STAGE_T2: src = d_T2; count = (size_t)n * n; break;
      case MSCKF_B200_STAGE_R2: src = d_R2; count = (size_t)n * n; break;
      case MSCKF_B200_STAGE_R2_RHS: src = d_r2; count = n; break;
      case MSCKF_B200_STAGE_Z: src = d_Z; count = 3 * (size_t)N * c; break;
      case MSCKF_B200_STAGE_YQ: src = d_Yq; count = 3 * (size_t)N * c; break;
      case MSCKF_B200_STAGE_UR: src = d_ur; count = 3 * (size_t)N; break;
      case MSCKF_B200_STAGE_D1: src = d_D1; count = 36 * (size_t)r.M; break;
      case MSCKF_B200_STAGE_D2: src = d_D2; count = 36 * (size_t)r.M; break;
      case MSCKF_B200_STAGE_BB: src = d_bb; count = 6 * (size_t)r.M; break;
      case MSCKF_B200_STAGE_XG: src = d_Xg; count = 12 * (size_t)O; elem = sizeof(S); break;
      case MSCKF_B200_STAGE_RG: src = d_rg; count = 2 * (size_t)O; elem = sizeof(S); break;
      case MSCKF_B200_STAGE_VG: src = d_Vg; count = 6 * (size_t)O; elem = sizeof(S); break;
      case MSCKF_B200_STAGE_TAUG: src = d_taug; count = 3 * (size_t)N; elem = sizeof(S); break;
      case MSCKF_B200_STAGE_ACCEPT: src = r.accept; count = N; elem = sizeof(int); break;
      default: src = d_rowoff; count = (size_t)N + 1; elem = sizeof(int); break;
    }
    const size_t k = std::min(count, (size_t)cap);
    if (k > 0) {
      CK(cudaSetDevice(device));
      if (which == MSCKF_B200_STAGE_T2 || which == MSCKF_B200_STAGE_R2) {  // n x n, de-strided from ld
        const size_t rows = k / n;
        if (rows) CK(cudaMemcpy2DAsync(out, sizeof(double) * n, src, sizeof(double) * ld, sizeof(double) * n, rows, cudaMemcpyDeviceToHost, stream));
        if (k % n) CK(cudaMemcpyAsync((double*)out + rows * n, (const double*)src + rows * ld, sizeof(double) * (k % n), cudaMemcpyDeviceToHost, stream));
      } else {
        CK(cudaMemcpyAsync(out, src, elem * k, cudaMemcpyDeviceToHost, stream));
      }
      CK(cudaStreamSynchronize(stream));
    }
    return (int)count;
  }
  int last_dx(double* out, int cap) override {
    CK(cudaSetDevice(device));
    const int n = 15 + 6 * M;
    std::vector<double> tmp(n);
    CK(cudaMemcpyAsync(tmp.data(), d_dx, sizeof(double) * n, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    for (int i = 0; i < std::min(n, cap); ++i) out[i] = tmp[i];
    return n;
  }

  int copy_from(const EngineBase* src_) override {
    const Engine<S>* src = dynamic_cast<const Engine<S>*>(src_);
    if (!src || src->device != device) return fail(MSCKF_B200_ERR_ARG, "copy_state: incompatible engines");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "copy_state with an un-fetched update pending");
    CK(cudaSetDevice(device));
    RC(ensure_clones(src->M));
    CK(cudaStreamSynchronize(src->stream));
    const int n = 15 + 6 * src->M;
    CK(cudaMemcpyAsync(d_st, src->d_st, sizeof(mb::DevState<S>), cudaMemcpyDeviceToDevice, stream));
    CK(cudaMemcpy2DAsync(d_P, sizeof(S) * ldp, src->d_P, sizeof(S) * src->ldp, sizeof(S) * n, n, cudaMemcpyDeviceToDevice, stream));
    if (src->M > 0)
      CK(cudaMemcpyAsync(d_poses, src->d_poses, sizeof(S) * mb::kPoseStride * (size_t)src->M, cudaMemcpyDeviceToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    rank_thr = src->rank_thr;
    memcpy(h_st, src->h_st, sizeof(mb::DevState<S>));
    M = src->M;
    initialized = src->initialized;
    return 0;
  }

  int sync() override {
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    return 0;
  }

  int tail_profile(unsigned long long* out, int cap) override {
    CK(cudaSetDevice(device));
    CK(cudaStreamSynchronize(stream));
    CK(cudaMemcpy(out, d_prof, sizeof(unsigned long long) * std::min(cap, 80), cudaMemcpyDeviceToHost));
    return std::min(cap, 80);
  }
};

// ------------------------------------------------------------------------------------------------ Ctx implementation
template <class S> EngineBase* Ctx<S>::member(int i) const { return eng[i]; }
template <class S> bool Ctx<S>::profile() const { return !eng.empty() && eng[0]->profile; }
template <class S>
void Ctx<S>::detach(EngineBase* e) {
  // an engine leaves the batch (it is being destroyed): the batch becomes unusable for updates but stays destroyable
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  for (auto& p : eng)
    if (p == e) p = nullptr;
  e->group = nullptr;
  e->set_stream(e->own_stream);
  pending = false; staged = false;
  drop_graphs();
}

template <class S>
int Ctx<S>::layout(const std::vector<std::pair<int, int>>& NO) {
  size_t oi = args_bytes(), orp = 0;
  for (size_t i = 0; i < eng.size(); ++i) {
    Plan<S>& p = plan[i];
    p.N = NO[i].first; p.O = NO[i].second;
    p.in_off = oi; oi += up256(Plan<S>::in_bytes(p.N, p.O));
    p.rep_off = orp; orp += up256(Plan<S>::rep_bytes(p.N));
  }
  in_used = oi; rep_used = orp;
  for (auto* e : eng) e->last_stage.M = -1;
  const unsigned char* old = in.d;
  RC(in.ensure(in_used, stream));
  RC(rep.ensure(rep_used, stream));
  if (in.d != old) drop_graphs();  // captured kernel arguments hold the arena's address
  for (auto& p : plan) p.carve(in, rep);
  return 0;
}

template <class S>
int Ctx<S>::stage(int mode, const msckf_b200_tracks* tracks, int threads) {
  const int nf = (int)eng.size();
  if (mode < 0 || mode > 2) return fail(MSCKF_B200_ERR_ARG, "bad mode");
  staged = false;
  for (auto* e : eng) {
    if (!e) return fail(MSCKF_B200_ERR_STATE, "a member engine of this batch was destroyed");
    if (!e->initialized) return fail(MSCKF_B200_ERR_STATE, "update before initialize");
    if (e->busy) return fail(MSCKF_B200_ERR_STATE, "previous update not fetched");
    if (e->stop_after_compression != eng[0]->stop_after_compression)
      return fail(MSCKF_B200_ERR_ARG, "option 8 (stop after the compression) must be the same for every member of a batch");
  }
  CK(cudaSetDevice(device));
  std::vector<std::pair<int, int>> NO(nf);
  std::vector<int> Lmax(nf, 0);
  std::vector<int> rc(nf, 0);
  std::vector<std::string> err(nf);
  // ---- validation (per filter; the index range check reads every observation once)
  auto validate = [&](int i) -> int {
    const msckf_b200_tracks& tr = tracks[i];
    Engine<S>* e = eng[i];
    const int N = tr.n_tracks;
    if (N < 0) return fail(MSCKF_B200_ERR_ARG, "negative track count");
    if (N == 0) { NO[i] = {0, 0}; return 0; }
    if (!tr.obs_offset || !tr.obs || !tr.clone_index) return fail(MSCKF_B200_ERR_ARG, "null track arrays");
    if (e->M < 1) return fail(MSCKF_B200_ERR_STATE, "update without clones");
    if (tr.obs_offset[0] != 0) return fail(MSCKF_B200_ERR_ARG, "obs_offset[0] must be 0");
    const int O = tr.obs_offset[N];
    int lm = 0;
    for (int t = 0; t < N; ++t) {
      const int L = tr.obs_offset[t + 1] - tr.obs_offset[t];
      if (L < 1 || L > 98) return fail(MSCKF_B200_ERR_ARG, "track length must be in [1,98] (chi-square table, msckf.h:91)");
      lm = std::max(lm, L);
    }
    const int Mi = e->M;
    // one observation per clone and track: MSCKF sees a feature once per image, and k_jac writes a track's compact Gram
    // outputs one clone column per observation, so a clone named twice would keep only one of its observations' terms
    std::vector<int> seen(Mi, -1);
    for (int t = 0; t < N; ++t)
      for (int o = tr.obs_offset[t]; o < tr.obs_offset[t + 1]; ++o) {
        const int k = tr.clone_index[o];
        if ((unsigned)k >= (unsigned)Mi) return fail(MSCKF_B200_ERR_ARG, "clone_index out of range");
        if (seen[k] == t) return fail(MSCKF_B200_ERR_ARG, "a track names one clone twice");
        seen[k] = t;
      }
    if (mode == MSCKF_B200_RESIDUALIZE && !tr.p_f_G) return fail(MSCKF_B200_ERR_ARG, "RESIDUALIZE needs p_f_G");
    NO[i] = {N, O};
    Lmax[i] = lm;
    return 0;
  };
  // Staging threads: `threads` is an upper bound.  Spreading the pack over several threads shortens the pack itself but
  // lengthens the time until the results are back -- the copy engine reads lines left dirty in several cores' caches -- so
  // a batch only gets a second thread from 8 MB of observations on (scripts/e2e_breakdown.py measures both parts).
  size_t in_bytes_est = 0;
  for (int i = 0; i < nf; ++i)
    if (tracks[i].n_tracks > 0 && tracks[i].obs_offset) in_bytes_est += (size_t)tracks[i].obs_offset[tracks[i].n_tracks] * (2 * sizeof(S) + sizeof(int));
  const int T = std::max(1, std::min({threads, nf, 1 + (int)(in_bytes_est >> 23)}));
  auto for_all = [&](auto&& fn) -> int {
    if (T == 1) {
      for (int i = 0; i < nf; ++i) { const int r = fn(i); if (r != 0) return r; }
      return 0;
    }
    pool.start(T - 1);
    pool.run(nf, [&](int i) { rc[i] = fn(i); if (rc[i] != 0) err[i] = g_err; });
    for (int i = 0; i < nf; ++i) if (rc[i] != 0) return fail(rc[i], err[i]);
    return 0;
  };
  RC(for_all(validate));
  for (int i = 0; i < nf; ++i) RC(eng[i]->ensure_tracks(NO[i].first, NO[i].second));
  // ---- packed layout; copy the batches into the pinned arena (skipped where the caller packed in place)
  const msckf_b200_tracks* t0 = tracks;
  const bool in_place = nf == 1 && plan[0].N == NO[0].first && plan[0].O == NO[0].second && t0->obs_offset == plan[0].h_off && in.h != nullptr;
  if (!in_place) RC(layout(NO));
  auto pack = [&](int i) -> int {
    Plan<S>& p = plan[i];
    p.Lmax = Lmax[i];
    const msckf_b200_tracks& tr = tracks[i];
    if (p.N > 0 && tr.obs_offset != p.h_off) {
      memcpy(p.h_off, tr.obs_offset, sizeof(int) * ((size_t)p.N + 1));
      memcpy(p.h_idx, tr.clone_index, sizeof(int) * (size_t)p.O);
      memcpy(p.h_obs, tr.obs, sizeof(S) * 2 * (size_t)p.O);
      if (mode == MSCKF_B200_RESIDUALIZE) memcpy(p.h_pfg_in, tr.p_f_G, sizeof(S) * 3 * (size_t)p.N);
    }
    eng[i]->fill_args(h_args()[i], p, mode);
    if (p.N > 0 && mode != MSCKF_B200_TRIANGULATE && h_args()[i].tail_kind < 0) return fail(MSCKF_B200_ERR_CAPACITY, "window too large for the tail kernel's shared memory");
    return 0;
  };
  RC(for_all(pack));
  CK(cudaMemcpyAsync(in.d, in.h, in_used, cudaMemcpyHostToDevice, stream));
  st_mode = mode;
  st_stop = eng[0]->stop_after_compression;
  staged = true;
  return 0;
}

template <class S>
int Ctx<S>::launch() {
  if (!staged) return fail(MSCKF_B200_ERR_STATE, "launch without a staged batch");
  staged = false;
  const int nf = (int)eng.size(), mode = st_mode;
  CK(cudaSetDevice(device));
  pending = true;
  for (auto* e : eng) e->busy = this;
  n_ev = 0;
  // ---- shape of the launch: every grid is sized for the largest member, rounded so that similar batches share a graph
  LaunchShape sh;
  memset(&sh, 0, sizeof(sh));
  sh.nf = nf; sh.mode = mode; sh.args = d_args();
  sh.stop = st_stop && mode != MSCKF_B200_TRIANGULATE ? 1 : 0;
  int Nmax = 0, Mmax_ = 0, Lm = 0, nmax_ = 0, nsplit = 1, jac_L = 0, jac_M = 0;
  for (int i = 0; i < nf; ++i) {
    const Plan<S>& p = plan[i];
    if (p.N == 0) continue;
    const mb::UpdArgs<S>& a = h_args()[i];
    Nmax = std::max(Nmax, p.N); Mmax_ = std::max(Mmax_, a.M); Lm = std::max(Lm, p.Lmax); nmax_ = std::max(nmax_, a.n);
    nsplit = std::max(nsplit, a.nsplit);
    sh.tri_smem = std::max<unsigned>(sh.tri_smem, (unsigned)(16 + sizeof(S) * mb::kPoseStride * (size_t)a.M + sizeof(S) * 4 * 14 * (size_t)p.Lmax));
    jac_L = std::max(jac_L, p.Lmax); jac_M = std::max(jac_M, a.M);
    sh.gram_mma |= a.gram_mma ? 2 : 1;  // which Gram kernels the batch needs
    if (mode != MSCKF_B200_TRIANGULATE) {
      sh.tail_mask |= 1 << a.tail_kind;
      sh.tail_smem[a.tail_kind] = std::max<unsigned>(sh.tail_smem[a.tail_kind], (unsigned)tail_smem(a.n, a.tail_kind));
    }
  }
  if (Nmax == 0) return 0;  // nothing to do on the device
  // k_jac: threads per track.  One filter: the whole CTA per track (latency).  A device batch: a warp per track, two tracks
  // per 64-thread CTA (throughput: a track's serial sections no longer idle its CTA), widened while the CTA's groups do not fit.
  sh.jac_g = eng[0]->jac_group ? eng[0]->jac_group : (nf > 1 ? kJacBatchGroup : 128);
  while (sh.jac_g < 128 && mb::jac_smem_bytes<S>(jac_L, jac_M, sh.jac_g) > kSmemBudget) sh.jac_g *= 2;
  sh.jac_smem = (unsigned)mb::jac_smem_bytes<S>(jac_L, jac_M, sh.jac_g);
  if (sh.tri_smem > kSmemBudget) return fail(MSCKF_B200_ERR_CAPACITY, "k_tri shared memory");
  if (mode != MSCKF_B200_TRIANGULATE && sh.jac_smem > kSmemBudget) return fail(MSCKF_B200_ERR_CAPACITY, "k_jac shared memory");
  // the dimension of the update whose rank decision msckf_b200_rank_pivots reports: set once the launch is committed, so that
  // a stage or launch that fails on a capacity leaves the last update's diagnostics alone; the window may shrink before they
  // are asked for
  if (mode != MSCKF_B200_TRIANGULATE)
    for (int i = 0; i < nf; ++i) {
      if (plan[i].N == 0) continue;
      Engine<S>* e = eng[i];
      e->last_stage = {plan[i].N, plan[i].O, e->M, plan[i].d_accept};
      if (sh.stop) RC(e->poison_compression(stream));  // (ahead of the graph: never captured)
      else e->pivr_n = h_args()[i].n;
    }
  const int Nr = (Nmax + 15) & ~15;  // rounded track count: kernels exit on blockIdx >= their filter's own N
  // (k_jac's at the SM's allocation granularity of 128 B: a whole KB would cost a batch of 8 config-B filters its tenth CTA per SM)
  sh.tri_smem = (sh.tri_smem + 1023) & ~1023u; sh.jac_smem = (sh.jac_smem + 127) & ~127u;
  if (sh.tri_smem > kSmemBudget) sh.tri_smem = (unsigned)kSmemBudget;
  if (sh.jac_smem > kSmemBudget) sh.jac_smem = (unsigned)kSmemBudget;
  if (mode != MSCKF_B200_TRIANGULATE && (sh.jac_g != jac_g || sh.jac_smem != jac_smem)) {
    jac_g = sh.jac_g; jac_smem = sh.jac_smem;
    jac_ctas = Engine<S>::jac_ctas_per_sm(jac_g, jac_smem);
  }
  sh.tri_gx = (Nr + 3) / 4; sh.jac_gx = Nr / (sh.jac_g == 128 ? 1 : 2); sh.rows_gx = Nr; sh.bd_gx = Mmax_;
  const int c = nmax_ - mb::kImuDim, ntile = (c + mb::GT - 1) / mb::GT;
  sh.gram_gx = ntile * (ntile + 1) / 2; sh.gram_gy = nsplit;
  sh.asm_gx = mb::asm_ctas(c);
  sh.rows_smem = (unsigned)(sizeof(double) * mb::rows_smem_doubles((Lm + 7) & ~7));
  sh.gemm_g = (nmax_ + 31) / 32;
  sh.syrk_gx = sh.gemm_g * (sh.gemm_g + 1) / 2;  // lower 32 x 32 tile pairs (k_gemm_s, k_syrk)
  sh.inj_smem = (unsigned)(sizeof(double) * nmax_);
  sh.pdl = (eng[0]->use_pdl && !profile()) ? 1 : 0;
  sh.tail_nch = (eng[0]->tail_chains == 1 || Engine<S>::tail9_clusters() == 0) ? 1 : 2;
  const bool want_graph = eng[0]->use_graph && !profile();
  if (want_graph) {
    for (auto& g : graphs)
      if (g.shape == sh) {
        g.stamp = ++tick;
        CK(cudaGraphLaunch(g.exec, stream));
        launches += g.nodes;
        for (auto* e : eng) e->launches += g.nodes;
        goto report;
      }
    bool second = false;
    for (auto& s : seen) if (s == sh) second = true;
    if (second) {
      const long long before = launches;
      cudaGraph_t graph = nullptr;
      {
        CaptureGuard cap(stream);
        RC(cap.begin());
        RC(run_kernels(sh));
        RC(cap.end(&graph));
      }
      cudaGraphExec_t exec = nullptr;
      cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
      cudaGraphDestroy(graph);
      if (ie != cudaSuccess) return fail(MSCKF_B200_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ie));
      if ((int)graphs.size() >= kMaxGraphs) {  // evict the least recently used
        size_t lru = 0;
        for (size_t k = 1; k < graphs.size(); ++k) if (graphs[k].stamp < graphs[lru].stamp) lru = k;
        cudaGraphExecDestroy(graphs[lru].exec);
        graphs.erase(graphs.begin() + lru);
      }
      graphs.push_back({sh, exec, (int)(launches - before), ++tick});
      CK(cudaGraphLaunch(exec, stream));
      for (auto* e : eng) e->launches += launches - before;
      goto report;
    }
    if (seen.size() >= 16) seen.erase(seen.begin());
    seen.push_back(sh);
  }
  {
    const long long before = launches;
    RC(run_kernels(sh));
    for (auto* e : eng) e->launches += launches - before;
  }
report:
  CK(cudaGetLastError());
  if (timed_region) CK(cudaEventRecord(ev_t1, stream));
  CK(cudaMemcpyAsync(rep.h, rep.d, rep_used, cudaMemcpyDeviceToHost, stream));  // one copy of all packed reports
  return 0;
}

// One launch: k = kernel, g = grid, b = block, smem; attrs: programmatic dependent launch (the kernel's prologue overlaps the
// tail of its predecessor; every kernel begins with griddepcontrol.wait before touching its predecessor's outputs).
template <class... Params, class... Args>
static cudaError_t launch_k(void (*k)(Params...), dim3 g, dim3 b, size_t smem, cudaStream_t s, bool pdl, int cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = g; cfg.blockDim = b; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    na++;
  }
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    na++;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, k, args...);
}

template <class S>
int Ctx<S>::run_kernels(const LaunchShape& sh) {
  const mb::UpdArgs<S>* A = d_args();
  const unsigned nf = (unsigned)sh.nf;
  const bool pdl = sh.pdl != 0;
  mark("begin");
  if (sh.mode != MSCKF_B200_RESIDUALIZE) {
    CK(launch_k(mb::k_tri<S, 4>, dim3(sh.tri_gx, 1, nf), dim3(128), sh.tri_smem, stream, false, 1, A));
    launches++;
    mark("k_tri");
  }
  if (sh.mode != MSCKF_B200_TRIANGULATE) {
    auto kj = sh.jac_g == 32 ? mb::k_jac<S, 32> : (sh.jac_g == 64 ? mb::k_jac<S, 64> : mb::k_jac<S, 128>);
    CK(launch_k(kj, dim3(sh.jac_gx, 1, nf), dim3(sh.jac_g == 32 ? 64 : 128), sh.jac_smem, stream, pdl && sh.mode != MSCKF_B200_RESIDUALIZE, 1, A));
    launches++;
    mark("k_jac");
    // k_blockdiag and k_gram both depend on k_jac only: two branches (a fork / join in the captured graph)
    const bool fork = !profile();  // per-kernel event timing keeps everything on one stream
    cudaStream_t sb = fork ? stream2 : stream, sr = fork ? stream3 : stream;
    if (fork) { CK(cudaEventRecord(ev_fork, stream)); CK(cudaStreamWaitEvent(stream2, ev_fork, 0)); CK(cudaStreamWaitEvent(stream3, ev_fork, 0)); }
    CK(launch_k(mb::k_blockdiag<S>, dim3(sh.bd_gx, 1, nf), dim3(128), 0, sb, false, 1, A));
    launches++;
    mark("k_blockdiag");
    if (fork) CK(cudaEventRecord(ev_join, stream2));
    // the explicit head rows only need k_jac's outputs and own their part of T'', R'', r'': a branch of their own, joined before T''P
    CK(launch_k(mb::k_rows<S>, dim3(sh.rows_gx, 1, nf), dim3(128), sh.rows_smem, sr, false, 1, A));
    launches++;
    mark("k_rows");
    if (fork) CK(cudaEventRecord(ev_join2, stream3));
    if (sh.gram_mma & 2) { CK(launch_k(mb::k_gram_mma<S>, dim3(sh.gram_gx, sh.gram_gy, nf), dim3(128), 0, stream, false, 1, A)); if (sh.gram_mma & 1) launches++; }  // FP64 tensor cores (DMMA)
    if (sh.gram_mma & 1) CK(launch_k(mb::k_gram<S>, dim3(sh.gram_gx, sh.gram_gy, nf), dim3(256), 0, stream, false, 1, A));
    launches++;
    mark("k_gram");
    if (fork) CK(cudaStreamWaitEvent(stream, ev_join, 0));
    CK(launch_k(mb::k_assemble<S>, dim3(sh.asm_gx, 1, nf), dim3(mb::kAsmThreads), 0, stream, false, 1, A));
    launches++;
    mark("k_assemble");
    if (fork) CK(cudaStreamWaitEvent(stream, ev_join2, 0));
    if (sh.stop) return 0;
    CK(launch_k(mb::k_gemm_tp<S>, dim3(sh.gemm_g, sh.gemm_g, nf), dim3(mb::kGemmThreads), 0, stream, false, 1, A));
    mark("k_gemm_tp");
    CK(launch_k(mb::k_gemm_s<S>, dim3(sh.syrk_gx, 1, nf), dim3(mb::kGemmThreads), 0, stream, pdl, 1, A));  // lower tile pairs of S''
    mark("k_gemm_s");
    launches += 2;
    // rank decision + Cholesky + substitution: one thread-block cluster per filter (kernels of a kind no member uses are skipped)
    if (sh.tail_mask & 1) {
      if (sh.tail_nch == 2) CK(launch_k(mb::k_tail_fused<S, 2>, dim3(kTailCluster + 1, 1, nf), dim3(mb::kTailThreads), sh.tail_smem[0], stream, pdl, kTailCluster + 1, A));
      else CK(launch_k(mb::k_tail_fused<S, 1>, dim3(kTailCluster, 1, nf), dim3(mb::kTailThreads), sh.tail_smem[0], stream, pdl, kTailCluster, A));
      launches++;
    }
    if (sh.tail_mask & 2) { CK(launch_k(mb::k_tail<S, 32>, dim3(kTailCluster, 1, nf), dim3(mb::kTailThreads), sh.tail_smem[1], stream, pdl, kTailCluster, A)); launches++; }
    if (sh.tail_mask & 4) { CK(launch_k(mb::k_tail<S, 16>, dim3(kTailCluster, 1, nf), dim3(mb::kTailThreads), sh.tail_smem[2], stream, pdl, kTailCluster, A)); launches++; }
    mark("k_tail");
    CK(launch_k(mb::k_syrk<S>, dim3(sh.syrk_gx, 1, nf), dim3(mb::kGemmThreads), 0, stream, pdl, 1, A));  // + dx = W^T y + state injection
    launches++;
    mark("k_syrk");
  }
  return 0;
}

// launch() bracketed by CUDA events on this context's stream; the staged inputs are already in HBM.
// The report copy is queued after the stop event, so the time is kernels only.
template <class S>
int Ctx<S>::launch_timed(float* ms) {
  CK(cudaSetDevice(device));
  if (!ev_t0) { CK(cudaEventCreate(&ev_t0)); CK(cudaEventCreate(&ev_t1)); }
  CK(cudaStreamSynchronize(stream));
  timed_region = true;
  CK(cudaEventRecord(ev_t0, stream));
  CK(cudaEventRecord(ev_t1, stream));  // (re-recorded after the kernels; recorded here so that an empty batch reads 0)
  int rc = launch();
  timed_region = false;
  if (rc != 0) return rc;
  CK(cudaStreamSynchronize(stream));
  CK(cudaEventElapsedTime(ms, ev_t0, ev_t1));
  return 0;
}

template <class S>
int Ctx<S>::fetch(msckf_b200_report* reports) {
  if (!pending) return fail(MSCKF_B200_ERR_STATE, "fetch without a pending update");
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(stream));
  pending = false;
  const int mode = st_mode;
  int status = 0;
  for (size_t i = 0; i < eng.size(); ++i) {
    if (eng[i]) eng[i]->busy = nullptr;
    const Plan<S>& p = plan[i];
    const int N = p.N;
    if (N > 0 && mode != MSCKF_B200_TRIANGULATE && p.h_mr[2] != 0) status = MSCKF_B200_ERR_NUMERIC;
    if (!reports) continue;
    msckf_b200_report* rep = &reports[i];
    rep->m = 0; rep->rank = 0;
    if (N == 0) continue;
    if (mode != MSCKF_B200_RESIDUALIZE) {
      if (rep->cm_ok) memcpy(rep->cm_ok, mode == MSCKF_B200_MARGINALIZE ? p.h_cmeff : p.h_cm, sizeof(int) * N);
      if (rep->tri_ok) memcpy(rep->tri_ok, p.h_tri, sizeof(int) * N);
      if (rep->p_f_G) memcpy(rep->p_f_G, p.h_pfg, sizeof(S) * 3 * (size_t)N);
    }
    if (mode != MSCKF_B200_TRIANGULATE) {
      if (rep->valid) memcpy(rep->valid, p.h_valid, sizeof(int) * N);
      if (rep->accepted) memcpy(rep->accepted, p.h_accept, sizeof(int) * N);
      if (rep->gamma) memcpy(rep->gamma, p.h_gamma, sizeof(S) * N);
      rep->m = p.h_mr[0];
      rep->rank = st_stop ? 0 : p.h_mr[1];  // (option 8: no rank decision was made)
    }
  }
  if (status != 0) return fail(status, "non-finite delta-x or covariance after the update (the update has been applied, like msckf.h:1369-1418 would), or the tail kernel's two chain CTAs lost their hand-off");
  return 0;
}

// ---- state calls.  A batch validates every member before anything is launched, so a bad argument changes no member; then it
// and the single filter's calls launch through the same enqueue_* and per_member, so a member runs exactly the kernel body and
// arguments of its single-filter call.  Arguments travel by value: no staging buffer, no host synchronisation.
template <class S>
int Ctx<S>::members_ready(const char* what) const {
  for (auto* e : eng) {
    if (!e) return fail(MSCKF_B200_ERR_STATE, "a member engine of this batch was destroyed");
    if (!e->initialized) return fail(MSCKF_B200_ERR_STATE, std::string(what) + " before initialize");
    if (e->busy) return fail(MSCKF_B200_ERR_STATE, std::string(what) + " with an un-fetched update pending");
  }
  return 0;
}

template <class S>
int Ctx<S>::propagate_n(const void* const* readings, const int* k) {
  RC(members_ready("batch_propagate_n"));
  for (int i = 0; i < (int)eng.size(); ++i) {
    const int ki = k ? k[i] : 0;
    if (ki < 0 || (ki > 0 && (!readings || !readings[i]))) return fail(MSCKF_B200_ERR_ARG, "batch_propagate_n: bad arguments");
  }
  return enqueue_propagate_n(readings, k);
}
template <class S>
int Ctx<S>::enqueue_propagate_n(const void* const* readings, const int* k) {
  const int nf = (int)eng.size();
  int kmax = 0;
  for (int i = 0; i < nf; ++i) kmax = std::max(kmax, k ? k[i] : 0);
  CK(cudaSetDevice(device));
  std::vector<int> idx;
  // kPropMax readings per launch: step k0 runs every member with more than k0 readings
  for (int k0 = 0; k0 < kmax; k0 += mb::kPropMax) {
    idx.clear();
    for (int i = 0; i < nf; ++i) if (k[i] > k0) idx.push_back(i);
    per_member(idx, true, [&](int i) { return eng[i]->prop_args((const S*)readings[i], k0, std::min(mb::kPropMax, k[i] - k0)); },
               [&](const auto& a, int nm) { mb::k_propagate<<<nm, 256, 0, stream>>>(a); });
  }
  CK(cudaGetLastError());
  return 0;
}

template <class S>
int Ctx<S>::augment(const int* which) {
  RC(members_ready("batch_augment"));
  std::vector<int> idx;
  for (int i = 0; i < (int)eng.size(); ++i) {
    if (which && !which[i]) continue;
    if (eng[i]->M + 1 > kMaxClonesHard) return fail(MSCKF_B200_ERR_CAPACITY, "sliding window exceeds the engine's hard limit of " + std::to_string(kMaxClonesHard) + " clones");
    idx.push_back(i);
  }
  return enqueue_augment(idx);
}
template <class S>
int Ctx<S>::enqueue_augment(const std::vector<int>& idx) {
  for (int i : idx) RC(eng[i]->ensure_clones(eng[i]->M + 1));
  CK(cudaSetDevice(device));
  per_member(idx, true, [&](int i) { return eng[i]->aug_args(); },
             [&](const auto& a, int nm) { mb::k_augment<<<nm, 256, 0, stream>>>(a); });
  CK(cudaGetLastError());
  for (int i : idx) eng[i]->M += 1;
  return 0;
}

template <class S>
int Ctx<S>::prune(const int* const* keep, const int* n_keep) {
  RC(members_ready("batch_prune"));
  if (!n_keep) return fail(MSCKF_B200_ERR_ARG, "batch_prune: null n_keep");
  std::vector<int> idx;  // members whose window changes
  for (int i = 0; i < (int)eng.size(); ++i) {
    if (n_keep[i] < 0 || n_keep[i] == eng[i]->M) continue;
    RC(eng[i]->prune_check(keep ? keep[i] : nullptr, n_keep[i]));
    idx.push_back(i);
  }
  return enqueue_prune(idx, keep, n_keep);
}
template <class S>
int Ctx<S>::enqueue_prune(const std::vector<int>& idx, const int* const* keep, const int* n_keep) {
  CK(cudaSetDevice(device));
  per_member(idx, true, [&](int i) { return eng[i]->gather_args(keep ? keep[i] : nullptr, n_keep[i]); },
             [&](const auto& a, int nm) {
               int gx = 1;  // the largest member's grid; smaller members' CTAs past their own grid-stride range exit at once
               for (int j = 0; j < nm; ++j) gx = std::max(gx, std::min(2 * num_sms(device), (a.m[j].n_new * a.m[j].n_new + 255) / 256));
               mb::k_gather<<<dim3(gx, nm), 256, 0, stream>>>(a);
             });
  CK(cudaGetLastError());
  for (int i : idx) eng[i]->prune_swap(n_keep[i]);
  return 0;
}

template <class S>
int Ctx<S>::get_state(void* const* imu, void* const* poses) {
  RC(members_ready("batch_get_state"));
  return read_state(imu, poses);
}
// every member's copies into the pinned I/O block, one synchronisation, then the C-ABI's layouts
template <class S>
int Ctx<S>::read_state(void* const* imu, void* const* poses) {
  const int nf = (int)eng.size();
  std::vector<size_t> off(nf + 1, 0);
  for (int i = 0; i < nf; ++i) off[i + 1] = off[i] + (poses && poses[i] ? up16(sizeof(S) * mb::kPoseStride * eng[i]->M) : 0);
  CK(cudaSetDevice(device));
  RC(io.ensure(off[nf], stream));
  for (int i = 0; i < nf; ++i)
    RC(eng[i]->state_copy(imu && imu[i], off[i + 1] > off[i] ? reinterpret_cast<S*>(io.h + off[i]) : nullptr));
  CK(cudaStreamSynchronize(stream));  // one synchronisation for the whole batch
  for (int i = 0; i < nf; ++i)
    eng[i]->state_unpack(imu ? imu[i] : nullptr, off[i + 1] > off[i] ? poses[i] : nullptr, reinterpret_cast<S*>(io.h + off[i]));
  return 0;
}

// Truth travels in the I/O block ([19] IMU + [M][7] poses per member) with one host-to-device copy; k_nees runs through
// per_member (NM = 1 with one member in the context); the results come back with one copy and one synchronisation.  Nothing of
// the filters is written (P, state, poses, graphs, launch counts).
static_assert(sizeof(mb::NeesOut) == sizeof(msckf_b200_nees_result) && offsetof(msckf_b200_nees_result, first_bad_pivot) == 44,
              "mb::NeesOut must have the layout of msckf_b200_nees_result");
template <class S>
int Ctx<S>::nees(const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out) {
  if (!truth_imu || !out) return fail(MSCKF_B200_ERR_ARG, "nees: null argument");
  RC(members_ready("nees"));
  const int nf = (int)eng.size();
  auto unit_ok = [](const double* q) { return q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0; };
  std::vector<size_t> off(nf + 1, 0), woff(nf + 1, 0);
  std::vector<int> idx;
  for (int i = 0; i < nf; ++i) {
    const double* ti = truth_imu[i];
    const double* tp = truth_poses ? truth_poses[i] : nullptr;
    const int M = eng[i]->M;
    if (!ti || !finite(ti, mb::kNeesTruthImu) || !unit_ok(ti + 15)) return fail(MSCKF_B200_ERR_ARG, "nees: missing or malformed truth_imu of member " + std::to_string(i));
    if (tp) {
      if (!finite(tp, 7 * M)) return fail(MSCKF_B200_ERR_ARG, "nees: malformed truth_poses of member " + std::to_string(i));
      for (int k = 0; k < M; ++k)
        if (!unit_ok(tp + 7 * k + 3)) return fail(MSCKF_B200_ERR_ARG, "nees: zero truth quaternion in member " + std::to_string(i));
    }
    const int n = tp ? 15 + 6 * M : 15;
    off[i + 1] = off[i] + up16(sizeof(double) * (mb::kNeesTruthImu + (tp ? 7 * (size_t)M : 0)));
    woff[i + 1] = woff[i] + up256(sizeof(double) * (size_t)(n + 1) * n);
    idx.push_back(i);
  }
  const size_t res_off = up256(off[nf]);
  CK(cudaSetDevice(device));
  RC(io.ensure(res_off + sizeof(mb::NeesOut) * nf, stream));
  RC(ws.ensure(woff[nf], stream));
  for (int i = 0; i < nf; ++i) {
    double* h = reinterpret_cast<double*>(io.h + off[i]);
    memcpy(h, truth_imu[i], sizeof(double) * mb::kNeesTruthImu);
    if (truth_poses && truth_poses[i] && eng[i]->M > 0) memcpy(h + mb::kNeesTruthImu, truth_poses[i], sizeof(double) * 7 * eng[i]->M);
  }
  CK(cudaMemcpyAsync(io.d, io.h, off[nf], cudaMemcpyHostToDevice, stream));
  per_member(idx, false,
             [&](int i) {
               return eng[i]->nees_args(reinterpret_cast<const double*>(io.d + off[i]), truth_poses && truth_poses[i],
                                        reinterpret_cast<double*>(ws.d + woff[i]), reinterpret_cast<mb::NeesOut*>(io.d + res_off) + i);
             },
             [&](const auto& a, int nm) { mb::k_nees<<<nm, 256, 0, stream>>>(a); });
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(io.h + res_off, io.d + res_off, sizeof(mb::NeesOut) * nf, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));  // one synchronisation for the whole batch
  memcpy(out, io.h + res_off, sizeof(mb::NeesOut) * nf);
  return 0;
}

// Aided updates: every updated member's inputs travel in the I/O block ([8][8] z of its items (LINEAR: r), the block-diagonal
// R [m][m], H [m][n] for LINEAR), k_aid runs through per_member (NM = 1 with one member in the context), the results come back
// with one copy and one synchronisation.  W^T and dx (n (m + 1) doubles) sit in dynamic shared memory up to kAidSmemMax bytes,
// else in the workspace.  Nothing is launched unless every member is valid: aid and aid_stack check their arguments and
// build one AidJob per member, aid_run launches them.
static_assert(offsetof(mb::AidOut, status) == offsetof(msckf_b200_aid_result, status), "mb::AidOut must start like msckf_b200_aid_result");
static_assert(offsetof(mb::AidFdeOut, stack) == 0 && sizeof(mb::AidFdeOut) % alignof(double) == 0, "mb::AidFdeOut must start with mb::AidOut");
static_assert((int)MSCKF_B200_AID_BODY_VELOCITY == (int)mb::kAidBodyVelocity && (int)MSCKF_B200_AID_RELATIVE_POSE == (int)mb::kAidRelativePose &&
                  (int)MSCKF_B200_AID_ANTENNA_POSITION == (int)mb::kAidAntennaPosition &&
                  (int)MSCKF_B200_AID_CLONE_ANTENNA_POSITION == (int)mb::kAidCloneAntennaPosition &&
                  (int)MSCKF_B200_AID_HEADING == (int)mb::kAidHeading && (int)MSCKF_B200_AID_CLONE_HEADING == (int)mb::kAidCloneHeading &&
                  (int)MSCKF_B200_AID_RANGE == (int)mb::kAidRange && (int)MSCKF_B200_AID_CLONE_RANGE == (int)mb::kAidCloneRange &&
                  (int)MSCKF_B200_AID_PLANE_RANGE == (int)mb::kAidPlaneRange &&
                  (int)MSCKF_B200_AID_CLONE_PLANE_RANGE == (int)mb::kAidClonePlaneRange &&
                  (int)MSCKF_B200_AID_GYRO_AT_REST == (int)mb::kAidGyroAtRest && (int)MSCKF_B200_AID_ACCEL_AT_REST == (int)mb::kAidAccelAtRest,
              "msckf_b200_aid_model and mb::AidModel differ");
template <class S>
int Ctx<S>::aid(const msckf_b200_aid* in, msckf_b200_aid_result* out) {
  if (!in || !out) return fail(MSCKF_B200_ERR_ARG, "aid_update: null argument");
  RC(members_ready("aid_update"));
  const int nf = (int)eng.size();
  std::vector<AidJob> job(nf);
  for (int i = 0; i < nf; ++i) {
    const msckf_b200_aid& q = in[i];
    if (q.model < 0) continue;
    const std::string who = " (member " + std::to_string(i) + ")";
    const int M = eng[i]->M, n = 15 + 6 * M;
    if (q.model > MSCKF_B200_AID_LINEAR) return fail(MSCKF_B200_ERR_ARG, "aid_update: unknown model" + who);
    if (std::isnan(q.chi2_max)) return fail(MSCKF_B200_ERR_ARG, "aid_update: chi2_max is NaN" + who);
    AidJob& j = job[i];
    j.chi2_max = q.chi2_max;
    if (q.model != MSCKF_B200_AID_LINEAR) {  // one item of the stacked form (a = the clone of CLONE_POSE; ignored otherwise)
      RC(aid_append(j, msckf_b200_aid_item{q.model, q.clone, 0, q.z, q.R}, M, "aid_update", who));
      if ((q.m != 0 && q.m != j.m) || (q.n != 0 && q.n != n)) return fail(MSCKF_B200_ERR_ARG, "aid_update: m / n do not match the model and the window" + who);
      continue;
    }
    const int m = q.m;  // LINEAR: the caller's r and H
    if (m < 1 || m > mb::kAidMaxRows || q.n != n) return fail(MSCKF_B200_ERR_ARG, "aid_update: m / n do not match the model and the window" + who);
    if (!q.z || !finite(q.z, m)) return fail(MSCKF_B200_ERR_ARG, "aid_update: missing or non-finite z" + who);
    if (!q.R) return fail(MSCKF_B200_ERR_ARG, "aid_update: missing R" + who);
    for (int r = 0; r < m; ++r)
      if (!finite(q.R + (size_t)r * m, r + 1)) return fail(MSCKF_B200_ERR_ARG, "aid_update: non-finite R" + who);
    if (!q.H || !finite(q.H, (size_t)m * n)) return fail(MSCKF_B200_ERR_ARG, "aid_update: missing or non-finite H" + who);
    j.m = m; j.n_items = 1; j.item[0] = {(short)q.model, 0, 0, 0};
    j.z[0] = q.z; j.nz[0] = m; j.R[0] = q.R; j.H = q.H;
  }
  return aid_run(job, out, "aid_update");
}

template <class S>
int Ctx<S>::aid_stack(const msckf_b200_aid_item* const* items, const int* n_items, double chi2_max, msckf_b200_aid_result* out,
                      const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) {
  const char* w = iter ? "aid_stack_update_iter" : "aid_stack_update";
  if (!items || !n_items || !out) return fail(MSCKF_B200_ERR_ARG, std::string(w) + ": null argument");
  RC(members_ready(w));
  if (std::isnan(chi2_max)) return fail(MSCKF_B200_ERR_ARG, std::string(w) + ": chi2_max is NaN");
  std::vector<AidJob> job;
  RC(aid_stack_jobs(items, n_items, w, job, iter));
  for (AidJob& j : job) j.chi2_max = chi2_max;
  return aid_run(job, out, w, nullptr, nullptr, iter, iout);
}

template <class S>
int Ctx<S>::aid_stack_fde(const msckf_b200_aid_item* const* items, const int* n_items, const msckf_b200_aid_fde* fde,
                          msckf_b200_aid_fde_result* out, const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) {
  const std::string w = iter ? "aid_stack_update_fde_iter" : "aid_stack_update_fde";
  if (!items || !n_items || !fde || !out) return fail(MSCKF_B200_ERR_ARG, w + ": null argument");
  RC(members_ready(w.c_str()));
  for (int d = 0; d < mb::kAidMaxRows; ++d)
    if (!(std::isfinite(fde->chi2[d]) && fde->chi2[d] > 0.0))
      return fail(MSCKF_B200_ERR_ARG, w + ": chi2[" + std::to_string(d) + "] is not finite and > 0");
  if (fde->max_exclude < 0 || fde->max_exclude > mb::kAidMaxItems - 1) return fail(MSCKF_B200_ERR_ARG, w + ": max_exclude outside 0..7");
  std::vector<AidJob> job;
  RC(aid_stack_jobs(items, n_items, w, job, iter));
  return aid_run(job, nullptr, w.c_str(), fde, out, iter, iout);
}

// one AidJob per member of a stacked call (n_items[i] = 0: member i is left alone), iter[i] checked for the members updated
// (iter given); 0, or MSCKF_B200_ERR_ARG
template <class S>
int Ctx<S>::aid_stack_jobs(const msckf_b200_aid_item* const* items, const int* n_items, const std::string& w, std::vector<AidJob>& job,
                           const msckf_b200_aid_iter* iter) {
  const int nf = (int)eng.size();
  job.assign(nf, AidJob{});
  for (int i = 0; i < nf; ++i) {
    if (n_items[i] == 0) continue;
    const std::string who = " (member " + std::to_string(i) + ")";
    if (n_items[i] < 0 || n_items[i] > mb::kAidMaxItems) return fail(MSCKF_B200_ERR_ARG, w + ": 1 to 8 items per stack" + who);
    if (!items[i]) return fail(MSCKF_B200_ERR_ARG, w + ": null item list" + who);
    if (iter && (iter[i].max_iter < 0 || iter[i].max_iter > mb::kAidMaxIter))
      return fail(MSCKF_B200_ERR_ARG, w + ": max_iter outside 0..16" + who);
    if (iter && !(std::isfinite(iter[i].tol) && iter[i].tol >= 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": tol is not finite and >= 0" + who);
    for (int k = 0; k < n_items[i]; ++k) {
      const std::string wk = " (member " + std::to_string(i) + ", item " + std::to_string(k) + ")";
      RC(aid_append(job[i], items[i][k], eng[i]->M, w, wk));
      // the iterate (mb::AidIterate) carries no biases: the at-rest rows are linear in b_g and b_a and nearly so in the attitude
      if (iter && (items[i][k].model == MSCKF_B200_AID_GYRO_AT_REST || items[i][k].model == MSCKF_B200_AID_ACCEL_AT_REST))
        return fail(MSCKF_B200_ERR_ARG, w + ": the at-rest models are not iterated" + wk);
    }
  }
  return 0;
}

// A standstill window's statistics (msckf_b200_standstill_update, DESIGN.md 4.18), in fp64 and in reading order: T = sum dT_j,
// the dT-weighted means of omega and a (the at-rest items' z), their R = s^2 R0 / T, the zero-velocity R and the scatter
// sigma / (6 (k - 1)) of the readings about their means under s^2 R0 (R0: Q_imu's gyro block, rows / columns 0..2, and
// accelerometer block, 6..8).  0, or MSCKF_B200_ERR_ARG.
struct StandstillStats {
  double T = 0.0, w[3] = {0.0, 0.0, 0.0}, a[3] = {0.0, 0.0, 0.0}, scatter = 0.0;
  double Rv[9] = {}, Rg[9] = {}, Ra[9] = {};
};
template <class S>
int standstill_stats(const S* r, int k, const S* Q, const msckf_b200_standstill& cfg, StandstillStats& o, const std::string& who) {
  const std::string w = "standstill_update";
  for (int j = 0; j < k; ++j) {
    for (int i = 0; i < 7; ++i)
      if (!std::isfinite((double)r[7 * j + i])) return fail(MSCKF_B200_ERR_ARG, w + ": non-finite reading" + who);
    if (!((double)r[7 * j + 6] > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": a dT that is not > 0" + who);
  }
  double sw[3] = {0.0, 0.0, 0.0}, sa[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < k; ++j) {
    const double dT = r[7 * j + 6];
    o.T += dT;
    for (int i = 0; i < 3; ++i) { sw[i] += dT * (double)r[7 * j + i]; sa[i] += dT * (double)r[7 * j + 3 + i]; }
  }
  for (int i = 0; i < 3; ++i) { o.w[i] = sw[i] / o.T; o.a[i] = sa[i] / o.T; }
  // R0's two blocks and their Cholesky factors (lower triangle read)
  double L[2][9] = {};
  const double s2 = cfg.noise_scale * cfg.noise_scale;
  for (int b = 0; b < 2; ++b) {
    const int c0 = b == 0 ? 0 : 6;
    double* R = b == 0 ? o.Rg : o.Ra;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[3 * i + j] = s2 * (double)Q[12 * (c0 + i) + c0 + j] / o.T;
    for (int j = 0; j < 3; ++j) {
      double d = Q[12 * (c0 + j) + c0 + j];
      for (int m = 0; m < j; ++m) d -= L[b][3 * j + m] * L[b][3 * j + m];
      if (!(d > 0.0) || !std::isfinite(d))
        return fail(MSCKF_B200_ERR_ARG, w + ": Q_imu's " + (b == 0 ? "gyro" : "accelerometer") + " block is not positive definite" + who);
      L[b][3 * j + j] = std::sqrt(d);
      for (int i = j + 1; i < 3; ++i) {
        double t = Q[12 * (c0 + i) + c0 + j];
        for (int m = 0; m < j; ++m) t -= L[b][3 * i + m] * L[b][3 * j + m];
        L[b][3 * i + j] = t / L[b][3 * j + j];
      }
    }
  }
  double sig = 0.0;
  for (int j = 0; j < k; ++j) {
    double q = 0.0;
    for (int b = 0; b < 2; ++b) {  // |L^-1 (y_j - y^)|^2 of the block
      const double* m = b == 0 ? o.w : o.a;
      double x[3];
      for (int i = 0; i < 3; ++i) {
        double t = (double)r[7 * j + 3 * b + i] - m[i];
        for (int c = 0; c < i; ++c) t -= L[b][3 * i + c] * x[c];
        x[i] = t / L[b][3 * i + i];
        q += x[i] * x[i];
      }
    }
    sig += (double)r[7 * j + 6] * q;
  }
  o.scatter = sig / s2 / (6.0 * (k - 1));
  const double v2 = cfg.sigma_v * cfg.sigma_v;
  for (int i = 0; i < 3; ++i) o.Rv[4 * i] = v2;
  return 0;
}

template <class S>
int Ctx<S>::standstill(const void* const* readings, const int* k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out) {
  const std::string w = "standstill_update";
  if (!readings || !k || !cfg || !out) return fail(MSCKF_B200_ERR_ARG, w + ": null argument");
  RC(members_ready(w.c_str()));
  if (!(std::isfinite(cfg->noise_scale) && cfg->noise_scale >= 1.0)) return fail(MSCKF_B200_ERR_ARG, w + ": noise_scale is not finite and >= 1");
  if (!(std::isfinite(cfg->sigma_v) && cfg->sigma_v > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": sigma_v is not finite and > 0");
  if (!(std::isfinite(cfg->scatter_max) && cfg->scatter_max > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": scatter_max is not finite and > 0");
  if (!(std::isfinite(cfg->chi2_max) && cfg->chi2_max > 0.0)) return fail(MSCKF_B200_ERR_ARG, w + ": chi2_max is not finite and > 0");
  const int nf = (int)eng.size();
  std::vector<StandstillStats> st(nf);
  for (int i = 0; i < nf; ++i) {
    if (k[i] == 0) continue;
    const std::string who = " (member " + std::to_string(i) + ")";
    if (k[i] < 2 || k[i] > kStandstillMaxReadings) return fail(MSCKF_B200_ERR_ARG, w + ": 2 to 4096 readings" + who);
    if (!readings[i]) return fail(MSCKF_B200_ERR_ARG, w + ": null readings" + who);
    RC(standstill_stats((const S*)readings[i], k[i], eng[i]->h_st->Q_imu, *cfg, st[i], who));
  }
  // the members at rest by their scatter: the 9-row stack, gated on chi2_max
  static const double kZero[3] = {0.0, 0.0, 0.0};
  std::vector<AidJob> job(nf);
  for (int i = 0; i < nf; ++i) {
    if (k[i] == 0 || st[i].scatter > cfg->scatter_max) continue;
    const std::string who = " (member " + std::to_string(i) + ")";
    RC(aid_append(job[i], {MSCKF_B200_AID_VELOCITY, 0, 0, kZero, st[i].Rv}, eng[i]->M, w, who));
    RC(aid_append(job[i], {MSCKF_B200_AID_GYRO_AT_REST, 0, 0, st[i].w, st[i].Rg}, eng[i]->M, w, who));
    RC(aid_append(job[i], {MSCKF_B200_AID_ACCEL_AT_REST, 0, 0, st[i].a, st[i].Ra}, eng[i]->M, w, who));
    job[i].chi2_max = cfg->chi2_max;
  }
  std::vector<msckf_b200_aid_result> res(nf);
  const int rc = aid_run(job, res.data(), w.c_str());
  if (rc != 0 && rc != MSCKF_B200_ERR_NUMERIC) return rc;
  for (int i = 0; i < nf; ++i) {
    if (k[i] == 0) continue;
    msckf_b200_standstill_result& o = out[i];
    o.scatter = st[i].scatter;
    if (job[i].n_items == 0) {
      o.stack = msckf_b200_aid_result{std::nan(""), 0.0, 0, 0, 0};
      o.outcome = 1;
    } else {
      o.stack = res[i];
      o.outcome = res[i].status == 1 ? -1 : res[i].applied ? 0 : 2;
    }
  }
  return rc;
}

template <class S>
int Ctx<S>::aid_run(const std::vector<AidJob>& job, msckf_b200_aid_result* out, const char* what, const msckf_b200_aid_fde* fde,
                    msckf_b200_aid_fde_result* fout, const msckf_b200_aid_iter* iter, msckf_b200_aid_iter_result* iout) {
  const int nf = (int)eng.size();
  // FDE: the item block follows the plain result; iter: then AidIterOut
  const size_t obase = fde ? sizeof(mb::AidFdeOut) : sizeof(mb::AidOut), osz = obase + (iter ? sizeof(mb::AidIterOut) : 0);
  const size_t in_tail = (fde ? mb::kAidFdeIn : 0) + (iter ? 2 : 0);  // doubles after R (and H)
  std::vector<int> idx;
  std::vector<size_t> off(nf + 1, 0), woff(nf + 1, 0);
  for (int i = 0; i < nf; ++i) {
    const int m = job[i].m, n = 15 + 6 * eng[i]->M;
    off[i + 1] = off[i];
    woff[i + 1] = woff[i];
    if (job[i].n_items == 0) continue;
    idx.push_back(i);
    off[i + 1] = off[i] + up16(sizeof(double) * (mb::kAidZ + (size_t)m * m + (job[i].H ? (size_t)m * n : 0) + in_tail));
    if (mb::aid_ws_bytes(n, m) > kAidSmemMax) woff[i + 1] = woff[i] + up256(mb::aid_ws_bytes(n, m));
  }
  if (idx.empty()) return 0;
  const size_t res_off = up256(off[nf]);
  CK(cudaSetDevice(device));
  RC(io.ensure(res_off + osz * nf, stream));
  RC(ws.ensure(woff[nf], stream));
  for (int i : idx) {
    const AidJob& q = job[i];
    const int m = q.m, n = 15 + 6 * eng[i]->M;
    double* h = reinterpret_cast<double*>(io.h + off[i]);
    memset(h, 0, sizeof(double) * (mb::kAidZ + (size_t)m * m));
    double* R = h + mb::kAidZ;
    for (int k = 0; k < q.n_items; ++k) {
      memcpy(h + mb::kAidItemZ * k, q.z[k], sizeof(double) * q.nz[k]);
      const int r0 = q.item[k].row, mk = (k + 1 < q.n_items ? q.item[k + 1].row : m) - r0;
      for (int r = 0; r < mk; ++r) memcpy(R + (size_t)(r0 + r) * m + r0, q.R[k] + (size_t)r * mk, sizeof(double) * mk);
    }
    if (q.H) memcpy(h + mb::kAidZ + m * m, q.H, sizeof(double) * m * n);
    if (fde) {
      memcpy(R + m * m, fde->chi2, sizeof(double) * mb::kAidMaxRows);
      R[m * m + mb::kAidMaxRows] = fde->max_exclude;
    }
    if (iter) {
      double* t = R + m * m + (fde ? mb::kAidFdeIn : 0);
      t[0] = iter[i].max_iter; t[1] = iter[i].tol;
    }
  }
  CK(cudaMemcpyAsync(io.d, io.h, off[nf], cudaMemcpyHostToDevice, stream));
  per_member(idx, false,
             [&](int i) {
               const bool global = woff[i + 1] > woff[i];
               return eng[i]->aid_args(job[i], reinterpret_cast<const double*>(io.d + off[i]),
                                       global ? reinterpret_cast<double*>(ws.d + woff[i]) : nullptr,
                                       reinterpret_cast<mb::AidOut*>(io.d + res_off + osz * i));
             },
             [&](const auto& a, int nm) {
               constexpr int NM = (int)std::extent<decltype(std::decay_t<decltype(a)>::m)>::value;
               size_t smem = 0;  // the largest need of the members whose W^T and dx are in shared memory
               for (int j = 0; j < nm; ++j)
                 if (!a.m[j].ws) smem = std::max(smem, mb::aid_ws_bytes(15 + 6 * a.m[j].M, a.m[j].m));
               if (fde && iter) mb::k_aid_iter<S, NM, true><<<nm, mb::kAidThreads, smem, stream>>>(a);
               else if (fde) mb::k_aid<S, NM, true><<<nm, mb::kAidThreads, smem, stream>>>(a);
               else if (iter) mb::k_aid_iter<S, NM><<<nm, mb::kAidThreads, smem, stream>>>(a);
               else mb::k_aid<<<nm, mb::kAidThreads, smem, stream>>>(a);
             });
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(io.h + res_off, io.d + res_off, osz * nf, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));  // one synchronisation for the whole batch
  int numeric = -1;
  for (int i : idx) {
    const mb::AidOut& o = *reinterpret_cast<const mb::AidOut*>(io.h + res_off + osz * i);
    msckf_b200_aid_result& r = fde ? fout[i].stack : out[i];
    r.nis = o.nis; r.dx_norm = o.dx_norm; r.dof = o.dof; r.applied = o.applied; r.status = o.status;
    if (fde) {
      const mb::AidFdeOut& g = *reinterpret_cast<const mb::AidFdeOut*>(&o);
      fout[i].outcome = g.outcome; fout[i].n_excluded = g.n_excluded;
      for (int k = 0; k < mb::kAidMaxItems; ++k)
        fout[i].item[k] = k < job[i].n_items ? msckf_b200_aid_item_result{g.item[k].nis, g.item[k].test, g.item[k].state, g.item[k].round}
                                             : msckf_b200_aid_item_result{std::nan(""), std::nan(""), -1, -1};
    }
    if (iter) {
      const mb::AidIterOut& g = *reinterpret_cast<const mb::AidIterOut*>(io.h + res_off + osz * i + obase);
      iout[i] = msckf_b200_aid_iter_result{g.iterations, g.converged, g.step};
    }
    if (o.numeric && numeric < 0) numeric = i;
  }
  return numeric_error(what, numeric);
}

// Mapped-landmark updates: every member with observations sends its observations (grouped by clone in window order, input
// order kept inside a clone), its clone table and (Sigma_L given) its map in the I/O block with one host-to-device copy;
// results, gamma and flags come back with one copy and one synchronisation.  Each per_member chunk (NM = 1 with one member in
// the context) launches clone, [set], gain, (step, clone, [set], gain) x (K - 1), downdate, K its largest max_iter and set only
// with a Sigma_L member, whatever the observations turn out to be.  Nothing is launched unless every member is valid.
static_assert(offsetof(mb::LmkOut, status) == offsetof(msckf_b200_landmark_result, status) &&
                  offsetof(mb::LmkOut, iterations) == offsetof(msckf_b200_landmark_result, iterations) &&
                  offsetof(mb::LmkOut, converged) == offsetof(msckf_b200_landmark_result, converged) &&
                  offsetof(mb::LmkOut, step) == offsetof(msckf_b200_landmark_result, step),
              "mb::LmkOut must have msckf_b200_landmark_result's fields at their offsets");
static_assert(sizeof(mb::LmkConsOut) == sizeof(msckf_b200_landmark_consensus_result) &&
                  offsetof(mb::LmkConsOut, refit) == offsetof(msckf_b200_landmark_consensus_result, refit) &&
                  offsetof(mb::LmkConsOut, yaw) == offsetof(msckf_b200_landmark_consensus_result, yaw) &&
                  offsetof(mb::LmkConsOut, pivot) == offsetof(msckf_b200_landmark_consensus_result, pivot),
              "mb::LmkConsOut must be msckf_b200_landmark_consensus_result");
// one member's call, planned on the host
struct LmkPlan {
  std::vector<int> perm, grp;  // packed observation j is input observation perm[j]; [G][3] clone, first observation, count
  int M = 0, G = 0, ld = 0;    // clones in the window; touched clones; rows of the compressed system, at most
  // Sigma_L given: the map, the clone-set groups, each observation's pair (-1: a one-clone landmark), the groups' landmarks
  const msckf_b200_landmark_map* map = nullptr;
  std::vector<int> sdesc, pair_of, lms;
  int H = 0, pairs = 0;
  size_t E_len = 0, B_len = 0;
  // consensus: the member runs one; its sampled observation pairs (packed order) and each observation's group
  bool cons = false;
  std::vector<int> hpair, ogrp;
};

// splitmix64's output function (DESIGN.md 4.17)
inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// the consensus's hypotheses of a member with no observations and its pairs: hypothesis h samples input observations
// i = u mod n and j = v mod (n - 1), j += 1 when j >= i, with u = splitmix64(seed + 2h), v = splitmix64(seed + 2h + 1), and the
// pair goes to the device in packed order (fewer than 2 observations: no pair, so no valid hypothesis)
int lmk_cons_plan(const msckf_b200_landmarks& q, const msckf_b200_landmark_consensus& c, const std::string& who, LmkPlan& p) {
  if (c.hypotheses < 0 || c.hypotheses > mb::kLmkMaxHyp) return fail(MSCKF_B200_ERR_ARG, "landmark_update: hypotheses outside 0 .. 1024" + who);
  if (c.hypotheses == 0) return 0;
  if (!std::isfinite(c.thresh) || !(c.thresh > 0.0)) return fail(MSCKF_B200_ERR_ARG, "landmark_update: consensus thresh is not finite and > 0" + who);
  if (c.min_inliers < 2) return fail(MSCKF_B200_ERR_ARG, "landmark_update: consensus min_inliers < 2" + who);
  p.cons = true;
  const int n = q.n_obs;
  if (n < 2) return 0;
  std::vector<int> inv(n);
  for (int j = 0; j < n; ++j) inv[p.perm[j]] = j;
  p.hpair.resize(2 * (size_t)c.hypotheses);
  for (int h = 0; h < c.hypotheses; ++h) {
    const uint64_t u = splitmix64(c.seed + 2 * (uint64_t)h), v = splitmix64(c.seed + 2 * (uint64_t)h + 1);
    const int i = (int)(u % (uint64_t)n);
    int j = (int)(v % (uint64_t)(n - 1));
    if (j >= i) ++j;
    p.hpair[2 * h] = inv[i]; p.hpair[2 * h + 1] = inv[j];
  }
  p.ogrp.resize(n);
  for (int g = 0; g < p.G; ++g)
    for (int k = 0; k < p.grp[3 * g + 2]; ++k) p.ogrp[p.grp[3 * g + 1] + k] = g;
  return 0;
}

// Sigma_L given: check the landmark ids and covariances, count the one-clone landmarks' observations per clone (single),
// and group the landmarks seen from 2 .. 8 clones by their exact clone set (sets in ascending order, landmarks ascending)
int lmk_map_plan(const msckf_b200_landmarks& q, const msckf_b200_landmark_map& mq, const std::string& who, LmkPlan& p,
                 std::vector<int>& single) {
  const int nl = mq.n_landmarks, no = q.n_obs;
  if (!mq.landmark || nl < 1) return fail(MSCKF_B200_ERR_ARG, "landmark_update: Sigma_L without landmark ids" + who);
  if (!finite(mq.Sigma_L, 6 * (size_t)nl)) return fail(MSCKF_B200_ERR_ARG, "landmark_update: non-finite Sigma_L" + who);
  // positive definite with room to spare: every squared pivot of the Cholesky factor >= 1e-30 m^2 and >= 1e-12 x the largest
  // diagonal entry, so that k_lmk_set's L^-1 (entries up to 1e15 / m) is finite and meaningful
  for (int l = 0; l < nl; ++l) {
    const double* s = mq.Sigma_L + 6 * (size_t)l;
    const double a = s[0], b = s[2] - s[1] * s[1] / a;
    const double c = s[4] - s[3] * s[1] / a;
    const double d = s[5] - s[3] * s[3] / a - c * c / b, floor = std::max(1e-30, 1e-12 * std::max(s[0], std::max(s[2], s[5])));
    if (!(a >= floor) || !(b >= floor) || !(d >= floor))
      return fail(MSCKF_B200_ERR_ARG, "landmark_update: Sigma_L of landmark " + std::to_string(l) +
                                          " is not positive definite (pivots >= 1e-30 and >= 1e-12 x its largest variance)" + who);
  }
  std::vector<std::vector<int>> of(nl);  // observations of each landmark, in input order
  for (int j = 0; j < no; ++j) {
    if (mq.landmark[j] < 0 || mq.landmark[j] >= nl) return fail(MSCKF_B200_ERR_ARG, "landmark_update: landmark id outside 0 .. n_landmarks - 1" + who);
    of[mq.landmark[j]].push_back(j);
  }
  std::map<std::vector<int>, std::vector<int>> sets;
  for (int l = 0; l < nl; ++l) {
    if (of[l].empty()) continue;
    std::vector<int> cs;
    for (int j : of[l]) {
      if (memcmp(q.p_L_G + 3 * (size_t)j, q.p_L_G + 3 * (size_t)of[l][0], sizeof(double) * 3) != 0)
        return fail(MSCKF_B200_ERR_ARG, "landmark_update: p_L_G differs within landmark " + std::to_string(l) + who);
      cs.push_back(q.clone[j]);
    }
    std::sort(cs.begin(), cs.end());
    if (std::adjacent_find(cs.begin(), cs.end()) != cs.end())
      return fail(MSCKF_B200_ERR_ARG, "landmark_update: landmark " + std::to_string(l) + " observed twice from one clone" + who);
    if ((int)cs.size() > mb::kLmkMapClones) return fail(MSCKF_B200_ERR_ARG, "landmark_update: a landmark seen from more than 8 clones" + who);
    if (cs.size() == 1) ++single[cs[0]];
    else sets[cs].push_back(l);
  }
  if ((int)sets.size() > mb::kLmkMaxSets) return fail(MSCKF_B200_ERR_ARG, "landmark_update: more than 256 clone sets" + who);
  p.pair_of.assign(no, -1);
  for (const auto& [cs, ls] : sets) {
    const int c = (int)cs.size(), nlg = (int)ls.size();
    if (c * nlg > mb::kLmkMaxPerSet) return fail(MSCKF_B200_ERR_ARG, "landmark_update: more than 256 observations in one clone set" + who);
    std::vector<int> d(mb::kLmkSetDesc, 0);
    d[0] = c; d[1] = nlg; d[2] = p.pairs; d[3] = (int)p.lms.size(); d[4] = (int)p.E_len; d[5] = (int)p.B_len;
    std::copy(cs.begin(), cs.end(), d.begin() + 8);
    p.sdesc.insert(p.sdesc.end(), d.begin(), d.end());
    for (int jl = 0; jl < nlg; ++jl)
      for (int j : of[ls[jl]]) p.pair_of[j] = p.pairs + jl * c + (int)(std::lower_bound(cs.begin(), cs.end(), q.clone[j]) - cs.begin());
    p.lms.insert(p.lms.end(), ls.begin(), ls.end());
    p.ld += std::min(2 * c * nlg, 6 * c);  // the group's rows, at most
    p.pairs += c * nlg;
    p.E_len += (size_t)nlg * (3 + 2 * c) * (6 * c + 4);
    p.B_len += (size_t)2 * c * nlg * (6 * c + 1);
    ++p.H;
  }
  return 0;
}

// Checks one member's call (mq: its map, or NULL) against a window of M clones and plans it.  A member without observations
// is only checked.
int lmk_plan(const msckf_b200_landmarks& q, const msckf_b200_landmark_map* mq, int M, const std::string& who, LmkPlan& p) {
  if (q.n_obs < 0 || q.n_obs > mb::kLmkMaxObs) return fail(MSCKF_B200_ERR_ARG, "landmark_update: n_obs outside 0 .. 4096" + who);
  if (q.max_iter < 0 || q.max_iter > mb::kLmkMaxIter) return fail(MSCKF_B200_ERR_ARG, "landmark_update: max_iter outside 0 .. 16" + who);
  if (!std::isfinite(q.tol) || q.tol < 0.0) return fail(MSCKF_B200_ERR_ARG, "landmark_update: tol is not finite and >= 0" + who);
  if (q.n_obs == 0) return 0;
  const int no = q.n_obs;
  if (!q.clone || !q.z || !q.p_L_G) return fail(MSCKF_B200_ERR_ARG, "landmark_update: missing clone, z or p_L_G" + who);
  std::vector<int> cnt(M, 0);
  for (int j = 0; j < no; ++j) {
    if (q.clone[j] < 0 || q.clone[j] >= M) return fail(MSCKF_B200_ERR_ARG, "landmark_update: clone outside the window" + who);
    if (++cnt[q.clone[j]] > mb::kLmkMaxPerClone) return fail(MSCKF_B200_ERR_ARG, "landmark_update: more than 256 observations of one clone" + who);
  }
  if (!finite(q.z, 2 * (size_t)no) || !finite(q.p_L_G, 3 * (size_t)no)) return fail(MSCKF_B200_ERR_ARG, "landmark_update: non-finite z or p_L_G" + who);
  if (q.R && (!finite(q.R, 3) || !(q.R[0] > 0.0) || !(q.R[0] * q.R[2] - q.R[1] * q.R[1] > 0.0)))
    return fail(MSCKF_B200_ERR_ARG, "landmark_update: R is not finite and positive definite" + who);
  if (std::isnan(q.chi2_obs)) return fail(MSCKF_B200_ERR_ARG, "landmark_update: chi2_obs is NaN" + who);
  p.M = M; p.map = mq;
  std::vector<int> single(M, 0);  // observations of one-clone landmarks per clone (all of them without Sigma_L)
  if (mq) RC(lmk_map_plan(q, *mq, who, p, single));
  else single = cnt;
  p.perm.resize(no);
  std::vector<int> first(M + 1, 0);
  for (int k = 0; k < M; ++k) first[k + 1] = first[k] + cnt[k];
  std::vector<int> fill(first.begin(), first.end() - 1);
  for (int j = 0; j < no; ++j) p.perm[fill[q.clone[j]]++] = j;  // stable: input order inside a clone
  for (int k = 0; k < M; ++k)
    if (cnt[k]) { p.grp.insert(p.grp.end(), {k, first[k], cnt[k]}); p.ld += std::min(2 * single[k], 6); }
  p.G = (int)p.grp.size() / 3;
  if (p.ld > mb::kLmkMaxRows)
    return fail(MSCKF_B200_ERR_ARG, "landmark_update: the compressed system may exceed " + std::to_string(mb::kLmkMaxRows) + " rows" + who);
  return 0;
}

// one member's host addresses in the I/O block: the inputs the host packs and the results it reads back
struct LmkHost {
  double *obs, *sig, *lsig, *gamma;
  int *grp, *wrow, *sdesc, *flag, *pairs, *ogrp, *score;
  mb::LmkOut* out;
  mb::LmkConsOut* cres;
};
struct LmkSizes { size_t in = 0, res = 0, io = 0, ws = 0; };  // bytes of inputs; offset of the results; I/O block; workspace

// The landmark call's buffers.  The I/O block holds every member's inputs, then (from a 256-byte boundary) every member's
// results; the workspace holds each member's slots, [S ; (T P)^T ; rho], dx and control words, then its iterated form's and
// its map's regions, each region 256-byte aligned.  With null bases this only sizes the blocks; with the allocated bases it
// also gives each member's host addresses (h) and its arguments' device addresses (a).
template <class S>
LmkSizes lmk_layout(const std::vector<int>& idx, const msckf_b200_landmarks* in, const std::vector<LmkPlan>& pl, unsigned char* ioh,
                    unsigned char* iod, unsigned char* wsd, std::vector<LmkHost>& h, std::vector<mb::LmkConsArgs<S>>& a) {
  LmkSizes z;
  size_t o = 0, w = 0;  // the cursors in the I/O block and in the workspace
  const auto io = [&](auto& hp, auto& dp, size_t bytes) {  // the next `bytes` of the I/O block, then 16-byte aligned
    if (ioh) {
      hp = reinterpret_cast<std::remove_reference_t<decltype(hp)>>(ioh + o);
      dp = reinterpret_cast<std::remove_reference_t<decltype(dp)>>(iod + o);
    }
    o += up16(bytes);
  };
  const auto take = [&](auto& dp, size_t bytes) { if (wsd) dp = reinterpret_cast<std::remove_reference_t<decltype(dp)>>(wsd + w); w += bytes; };
  for (int i : idx) {
    const LmkPlan& p = pl[i];
    const size_t no = p.perm.size(), n = 15 + 6 * (size_t)p.M;
    io(h[i].obs, a[i].obs, sizeof(double) * 5 * no);
    io(h[i].grp, a[i].grp, sizeof(int) * p.grp.size());
    if (p.map) {  // Sigma of each observation's landmark, its pair, the group table, Sigma of the groups' landmarks
      io(h[i].sig, a[i].sig, sizeof(double) * 6 * no);
      io(h[i].wrow, a[i].wrow, sizeof(int) * no);
      io(h[i].sdesc, a[i].sdesc, sizeof(int) * p.sdesc.size());
      io(h[i].lsig, a[i].lsig, sizeof(double) * 6 * p.lms.size());
    }
    if (p.cons) {  // the sampled pairs and each observation's group
      io(h[i].pairs, a[i].pairs, sizeof(int) * p.hpair.size());
      io(h[i].ogrp, a[i].ogrp, sizeof(int) * p.ogrp.size());
    }
    take(a[i].slot, sizeof(double) * mb::kLmkSlot * p.G);
    take(a[i].A, sizeof(double) * (p.ld + n + 1) * p.ld);
    take(a[i].dx, sizeof(double) * n);
    take(a[i].ctl, sizeof(mb::LmkCtl));
    w = up256(w);
    if (in[i].max_iter > 1) {  // the iterate table, delta_i and the iteration's control words
      take(a[i].xi, sizeof(double) * 7 * p.M); take(a[i].d, sizeof(double) * n); take(a[i].it, sizeof(mb::LmkIt));
      w = up256(w);
    }
    if (p.map) {  // the pairs, the elimination and group rows, the groups' slots
      take(a[i].pair, sizeof(double) * mb::kLmkPair * p.pairs); take(a[i].E, sizeof(double) * p.E_len);
      take(a[i].B, sizeof(double) * p.B_len); take(a[i].sslot, sizeof(double) * mb::kLmkSetSlot * p.H);
      w = up256(w);
    }
    if (p.cons) {  // the hypotheses' fits and counts
      take(a[i].hyp, sizeof(mb::LmkHyp) * p.hpair.size() / 2);
      w = up256(w);
    }
  }
  z.in = o;
  o = z.res = up256(o);
  for (int i : idx) {
    const size_t no = pl[i].perm.size();
    io(h[i].out, a[i].out, sizeof(mb::LmkOut));
    io(h[i].gamma, a[i].gamma, sizeof(double) * no);
    io(h[i].flag, a[i].flag, sizeof(int) * no);
    if (pl[i].cons) {
      io(h[i].cres, a[i].cres, sizeof(mb::LmkConsOut));
      io(h[i].score, a[i].score, sizeof(int) * pl[i].hpair.size() / 2);
    }
  }
  z.io = o; z.ws = w;
  return z;
}

template <class S>
int Ctx<S>::landmarks(const msckf_b200_landmarks* in, const msckf_b200_landmark_map* map, msckf_b200_landmark_result* out,
                      const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_consensus_result* cout) {
  if (!in || !out) return fail(MSCKF_B200_ERR_ARG, "landmark_update: null argument");
  RC(members_ready("landmark_update"));
  const int nf = (int)eng.size();
  std::vector<LmkPlan> pl(nf);
  std::vector<LmkHost> h(nf);
  std::vector<mb::LmkConsArgs<S>> args(nf);  // zeroed; the layout fills in the addresses
  std::vector<int> idx;
  bool any_cons = false;
  for (int i = 0; i < nf; ++i) {
    const std::string who = " (member " + std::to_string(i) + ")";
    RC(lmk_plan(in[i], map && map[i].Sigma_L ? &map[i] : nullptr, eng[i]->M, who, pl[i]));
    if (cons) RC(lmk_cons_plan(in[i], cons[i], who, pl[i]));
  }
  for (int i = 0; i < nf; ++i) {
    if (cout) {  // (a member whose consensus runs gets its result and scores below; without observations it fails)
      memset(&cout[i], 0, sizeof(cout[i]));
      cout[i].best = -1;
      if (pl[i].cons) cout[i].status = 1;
    }
    if (pl[i].cons && cons[i].scores)
      for (int k = 0; k < cons[i].hypotheses; ++k) cons[i].scores[k] = -1;
    if (!in[i].n_obs) continue;
    idx.push_back(i);
    static_cast<mb::LmkArgs<S>&>(args[i]) = eng[i]->lmk_args(in[i], pl[i].G, pl[i].ld);
    args[i].H = pl[i].H; args[i].max_iter = in[i].max_iter; args[i].tol = in[i].tol;
    if (pl[i].cons) {
      args[i].cons = 1; args[i].thresh = cons[i].thresh; args[i].min_inl = cons[i].min_inliers;
      args[i].n_obs = in[i].n_obs; args[i].nh = (int)pl[i].hpair.size() / 2;
      any_cons = true;
    }
  }
  if (idx.empty()) return 0;
  const LmkSizes z = lmk_layout<S>(idx, in, pl, nullptr, nullptr, nullptr, h, args);
  CK(cudaSetDevice(device));
  RC(io.ensure(z.io, stream));
  RC(ws.ensure(z.ws, stream));
  lmk_layout<S>(idx, in, pl, io.h, io.d, ws.d, h, args);
  for (int i : idx) {
    const msckf_b200_landmarks& q = in[i];
    const LmkPlan& p = pl[i];
    const LmkHost& hm = h[i];
    const msckf_b200_landmark_map* mq = p.map;
    for (int j = 0; j < q.n_obs; ++j) {
      const int s = p.perm[j];
      double* o = hm.obs + 5 * j;
      o[0] = q.z[2 * s]; o[1] = q.z[2 * s + 1];
      o[2] = q.p_L_G[3 * s]; o[3] = q.p_L_G[3 * s + 1]; o[4] = q.p_L_G[3 * s + 2];
      if (mq) { memcpy(hm.sig + 6 * j, mq->Sigma_L + 6 * (size_t)mq->landmark[s], sizeof(double) * 6); hm.wrow[j] = p.pair_of[s]; }
    }
    memcpy(hm.grp, p.grp.data(), sizeof(int) * p.grp.size());
    if (mq) {
      memcpy(hm.sdesc, p.sdesc.data(), sizeof(int) * p.sdesc.size());
      for (size_t l = 0; l < p.lms.size(); ++l) memcpy(hm.lsig + 6 * l, mq->Sigma_L + 6 * (size_t)p.lms[l], sizeof(double) * 6);
    }
    if (p.cons) {
      memcpy(hm.pairs, p.hpair.data(), sizeof(int) * p.hpair.size());
      memcpy(hm.ogrp, p.ogrp.data(), sizeof(int) * p.ogrp.size());
    }
  }
  CK(cudaMemcpyAsync(io.d, io.h, z.in, cudaMemcpyHostToDevice, stream));
  per_member(idx, false, [&](int i) { return args[i]; },
             [&](const auto& a, int nm) {
               constexpr int NM = (int)std::extent<decltype(std::decay_t<decltype(a)>::m)>::value;
               mb::Members<mb::LmkArgs<S>, NM> b;  // the single linearisation's arguments, as they always were
               mb::Members<mb::LmkItArgs<S>, NM> c;  // the iterated form's
               mb::Members<mb::LmkMapArgs<S>, NM> d;  // the map form's
               int gx = 1, tx = 1, K = 1, hx = 0, hy = 0;  // the largest member's grid; other members' CTAs past their own range exit at once
               for (int j = 0; j < nm; ++j) {
                 b.m[j] = a.m[j]; c.m[j] = a.m[j]; d.m[j] = a.m[j];
                 gx = std::max(gx, a.m[j].G);
                 tx = std::max(tx, a.m[j].ntiles);
                 K = std::max(K, a.m[j].max_iter);
                 if (a.m[j].sig) hx = std::max(hx, std::max(1, a.m[j].H));
                 if (a.m[j].cons) hy = std::max(hy, std::max(1, (a.m[j].nh + mb::kConsWarps - 1) / mb::kConsWarps));
               }
               // MAP (a member has Sigma_L): clone, set and gain take the map arguments; else b (linearisation 0) and c.
               // CONS (a member runs a consensus): k_lmk_hyp and k_lmk_cons, then linearisation 0's clone pre-set by them.
               const auto lin = [&](auto map, auto cs, const auto& x0, const auto& x1) {
                 constexpr bool MAP = decltype(map)::value, CONS = decltype(cs)::value;
                 if constexpr (CONS) {
                   mb::k_lmk_hyp<S, NM><<<dim3(hy, nm), mb::kConsWarps * 32, 0, stream>>>(a);
                   mb::k_lmk_cons<S, NM><<<nm, mb::kLmkThreads, 0, stream>>>(a);
                   mb::k_lmk_clone<S, NM, false, MAP, true><<<dim3(gx, nm), mb::kLmkThreads, 0, stream>>>(a);
                 } else {
                   mb::k_lmk_clone<S, NM, false, MAP><<<dim3(gx, nm), mb::kLmkThreads, 0, stream>>>(x0);
                 }
                 if constexpr (MAP) mb::k_lmk_set<S, NM><<<dim3(hx, nm), mb::kLmkThreads, 0, stream>>>(x0);
                 mb::k_lmk_gain<S, NM, false, MAP><<<nm, mb::kLmkThreads, 0, stream>>>(x0);
                 for (int it = 0; it + 1 < K; ++it) {
                   mb::k_lmk_step<S, NM><<<nm, mb::kLmkThreads, 0, stream>>>(c, it);
                   mb::k_lmk_clone<S, NM, true, MAP><<<dim3(gx, nm), mb::kLmkThreads, 0, stream>>>(x1);
                   if constexpr (MAP) mb::k_lmk_set<S, NM, true><<<dim3(hx, nm), mb::kLmkThreads, 0, stream>>>(x1);
                   mb::k_lmk_gain<S, NM, true, MAP><<<nm, mb::kLmkThreads, 0, stream>>>(x1);
                 }
               };
               if (hx == 0 && hy == 0) lin(std::false_type(), std::false_type(), b, c);
               else if (hx == 0) lin(std::false_type(), std::true_type(), b, c);
               else if (hy == 0) lin(std::true_type(), std::false_type(), d, d);
               else lin(std::true_type(), std::true_type(), d, d);
               mb::k_lmk_downdate<S, NM><<<dim3(tx, nm), mb::kLmkThreads, 0, stream>>>(b);
             });
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(io.h + z.res, io.d + z.res, z.io - z.res, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));  // one synchronisation for the whole batch
  int numeric = -1;
  for (int i : idx) {
    const msckf_b200_landmarks& q = in[i];
    const mb::LmkOut& o = *h[i].out;
    out[i].nis = o.nis; out[i].dx_norm = o.dx_norm; out[i].dof = o.dof; out[i].rows = o.rows; out[i].used = o.used;
    out[i].applied = o.applied; out[i].status = o.status;
    const bool it = q.max_iter > 1;  // (the single linearisation leaves these to the host)
    out[i].iterations = it ? o.iterations : o.applied; out[i].converged = it ? o.converged : 0; out[i].step = it ? o.step : 0.0;
    for (int j = 0; j < q.n_obs; ++j) {
      if (q.gamma) q.gamma[pl[i].perm[j]] = h[i].gamma[j];
      if (q.flag) q.flag[pl[i].perm[j]] = h[i].flag[j];
    }
    if (pl[i].cons) {
      if (cout) memcpy(&cout[i], h[i].cres, sizeof(cout[i]));
      if (cons[i].scores)
        for (int k = 0; k < cons[i].hypotheses; ++k) cons[i].scores[k] = k < (int)pl[i].hpair.size() / 2 ? h[i].score[k] : -1;
    }
    if (o.numeric && numeric < 0) numeric = i;
  }
  return numeric_error("landmark_update", numeric);
}
}  // namespace

struct msckf_b200_engine { EngineBase* impl; };
struct msckf_b200_batch { CtxBase* ctx; int dtype; };

namespace {
template <class S>
int make_batch(msckf_b200_engine** engines, int n, msckf_b200_batch** out) {
  auto* c = new Ctx<S>();
  Engine<S>* first = static_cast<Engine<S>*>(engines[0]->impl);
  int rc = c->init(first->device);
  if (rc != 0) { delete c; return rc; }
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return fail(MSCKF_B200_ERR_CUDA, "cudaStreamCreate"); }
  c->owns_stream = true;
  for (int i = 0; i < n; ++i) {
    Engine<S>* e = static_cast<Engine<S>*>(engines[i]->impl);
    e->sync();
    e->group = c;
    e->set_stream(c->stream);
    c->eng.push_back(e);
  }
  c->plan.resize(n);
  *out = new msckf_b200_batch{c, first->dtype};
  return 0;
}

// stage and launch an update of a filter's or a batch's context; update() also fetches
int update_async(CtxBase* c, int mode, const msckf_b200_tracks* tracks, int threads) {
  if (!tracks) return fail(MSCKF_B200_ERR_ARG, "null argument");
  RC(c->stage(mode, tracks, threads));
  return c->launch();
}
int update(CtxBase* c, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports, int threads) {
  const int rc = update_async(c, mode, tracks, threads);
  if (rc == 0) return c->fetch(reports);
  // keep the real cause: clean up a half-started update without touching the error message
  if (c->pending) { const std::string keep = g_err; c->fetch(nullptr); g_err = keep; }
  return rc;
}
}  // namespace

extern "C" {
const char* msckf_b200_last_error(void) { return g_err.c_str(); }

int msckf_b200_create(const msckf_b200_config* cfg, msckf_b200_engine** out) {
  if (!cfg || !out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(MSCKF_B200_ERR_NO_DEVICE, "no CUDA device: the engine has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(MSCKF_B200_ERR_ARG, "bad device ordinal");
  if (cfg->max_clones < 1 || cfg->max_tracks < 1 || cfg->max_obs < 1) return fail(MSCKF_B200_ERR_ARG, "bad capacities");
  if (cfg->max_clones > kMaxClonesHard) return fail(MSCKF_B200_ERR_CAPACITY, "max_clones above the engine's hard limit");
  EngineBase* b = nullptr;
  if (cfg->dtype == MSCKF_B200_F32) b = new Engine<float>();
  else if (cfg->dtype == MSCKF_B200_F64) b = new Engine<double>();
  else return fail(MSCKF_B200_ERR_ARG, "bad dtype");
  if (getenv("MSCKF_B200_NO_GRAPH")) b->use_graph = false;  // e.g. under ncu: profile plain launches
  if (getenv("MSCKF_B200_NO_PDL")) b->use_pdl = false;
  if (getenv("MSCKF_B200_NO_DMMA")) b->gram_mma = false;
  if (getenv("MSCKF_B200_NO_FUSED_TAIL")) b->no_fused_tail = true;
  if (const char* g = getenv("MSCKF_B200_TAIL_CHAINS")) { const int v = atoi(g); if (v == 1 || v == 2) b->tail_chains = v; }
  if (const char* g = getenv("MSCKF_B200_JAC_GROUP")) { const int v = atoi(g); if (v == 32 || v == 64 || v == 128) b->jac_group = v; }
  b->dtype = cfg->dtype; b->device = cfg->device; b->Mmax = cfg->max_clones; b->Tmax = cfg->max_tracks; b->Omax = cfg->max_obs;
  int rc = (cfg->dtype == MSCKF_B200_F32) ? static_cast<Engine<float>*>(b)->alloc() : static_cast<Engine<double>*>(b)->alloc();
  if (rc != 0) { delete b; return rc; }
  *out = new msckf_b200_engine{b};
  return 0;
}
int msckf_b200_destroy(msckf_b200_engine* e) {
  if (!e) return 0;
  delete e->impl;
  delete e;
  return 0;
}
int msckf_b200_initialize(msckf_b200_engine* e, const void* camera, const void* noise, const void* params, const void* imu_state) {
  return e->impl->initialize(camera, noise, params, imu_state);
}
int msckf_b200_propagate(msckf_b200_engine* e, const void* reading) { return e->impl->propagate_n(reading, 1); }
int msckf_b200_propagate_n(msckf_b200_engine* e, const void* readings, int k) { return e->impl->propagate_n(readings, k); }
int msckf_b200_augment(msckf_b200_engine* e) { return e->impl->augment(); }
int msckf_b200_input_buffer(msckf_b200_engine* e, int n_tracks, int n_obs, msckf_b200_tracks* out) { return e->impl->input_buffer(n_tracks, n_obs, out); }
int msckf_b200_stage(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks) {
  if (!tracks) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return e->impl->solo_ctx()->stage(mode, tracks, 1);
}
int msckf_b200_launch(msckf_b200_engine* e) { return e->impl->solo_ctx()->launch(); }
int msckf_b200_launch_timed(msckf_b200_engine* e, float* ms) { return e->impl->solo_ctx()->launch_timed(ms); }
int msckf_b200_update_async(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks) {
  return update_async(e->impl->solo_ctx(), mode, tracks, 1);
}
int msckf_b200_fetch(msckf_b200_engine* e, msckf_b200_report* report) { return e->impl->solo_ctx()->fetch(report); }
int msckf_b200_update(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* report) {
  return update(e->impl->solo_ctx(), mode, tracks, report, 1);
}

int msckf_b200_batch_create(msckf_b200_engine** engines, int n, msckf_b200_batch** out) {
  if (!engines || n <= 0 || !out) return fail(MSCKF_B200_ERR_ARG, "batch_create: bad arguments");
  for (int i = 0; i < n; ++i) {
    if (!engines[i]) return fail(MSCKF_B200_ERR_ARG, "batch_create: null engine");
    EngineBase* b = engines[i]->impl;
    if (b->dtype != engines[0]->impl->dtype || b->device != engines[0]->impl->device) return fail(MSCKF_B200_ERR_ARG, "batch_create: engines differ in dtype or device");
    if (b->group) return fail(MSCKF_B200_ERR_STATE, "batch_create: an engine already belongs to a batch");
    if (b->busy) return fail(MSCKF_B200_ERR_STATE, "batch_create: an engine has an un-fetched update");
    for (int j = 0; j < i; ++j) if (engines[j] == engines[i]) return fail(MSCKF_B200_ERR_ARG, "batch_create: duplicate engine");
  }
  return engines[0]->impl->dtype == MSCKF_B200_F32 ? make_batch<float>(engines, n, out) : make_batch<double>(engines, n, out);
}
int msckf_b200_batch_destroy(msckf_b200_batch* b) {
  if (!b) return 0;
  CtxBase* c = b->ctx;
  for (int i = 0; i < c->count(); ++i) {
    EngineBase* e = c->member(i);
    if (e) c->detach(e);  // synchronises, gives the engine its own stream back
  }
  delete c;
  delete b;
  return 0;
}
int msckf_b200_batch_stage(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, int threads) {
  if (!b || !tracks) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->stage(mode, tracks, threads);
}
int msckf_b200_batch_launch(msckf_b200_batch* b) { return b->ctx->launch(); }
int msckf_b200_batch_launch_timed(msckf_b200_batch* b, float* ms) { return b->ctx->launch_timed(ms); }
int msckf_b200_batch_update_async(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, int threads) {
  return b ? update_async(b->ctx, mode, tracks, threads) : fail(MSCKF_B200_ERR_ARG, "null argument");
}
int msckf_b200_batch_fetch(msckf_b200_batch* b, msckf_b200_report* reports) { return b->ctx->fetch(reports); }
int msckf_b200_batch_update(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports, int threads) {
  return b ? update(b->ctx, mode, tracks, reports, threads) : fail(MSCKF_B200_ERR_ARG, "null argument");
}
int msckf_b200_batch_kernel_times(msckf_b200_batch* b, float* ms, const char** names, int cap) { return b->ctx->kernel_times(ms, names, cap); }
long long msckf_b200_batch_launch_count(const msckf_b200_batch* b) { return b->ctx->launches; }
int msckf_b200_batch_jac_occupancy(const msckf_b200_batch* b) { return b->ctx->jac_ctas; }
int msckf_b200_jac_group(msckf_b200_engine* e) {
  const CtxBase* c = e->impl->group ? e->impl->group : e->impl->solo_ctx();
  return c->jac_g;
}
void* msckf_b200_batch_stream(msckf_b200_batch* b) { return (void*)b->ctx->stream; }
int msckf_b200_batch_propagate_n(msckf_b200_batch* b, const void* const* readings, const int* k) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->propagate_n(readings, k);
}
int msckf_b200_batch_augment(msckf_b200_batch* b, const int* which) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->augment(which);
}
int msckf_b200_batch_prune(msckf_b200_batch* b, const int* const* keep, const int* n_keep) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->prune(keep, n_keep);
}
int msckf_b200_batch_get_state(msckf_b200_batch* b, void* const* imu, void* const* clone_poses) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->get_state(imu, clone_poses);
}
int msckf_b200_batch_nees(msckf_b200_batch* b, const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->nees(truth_imu, truth_poses, out);
}
int msckf_b200_batch_aid_update(msckf_b200_batch* b, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->aid(aid, out);
}
int msckf_b200_batch_aid_stack_update(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                      double chi2_max, msckf_b200_aid_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->aid_stack(items, n_items, chi2_max, out, nullptr, nullptr);
}
int msckf_b200_batch_aid_stack_update_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                           double chi2_max, const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out,
                                           msckf_b200_aid_iter_result* iter_out) {
  if (!b || !iter || !iter_out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->aid_stack(items, n_items, chi2_max, out, iter, iter_out);
}
int msckf_b200_batch_standstill_update(msckf_b200_batch* b, const void* const* readings, const int* k, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->standstill(readings, k, cfg, out);
}
int msckf_b200_batch_aid_stack_update_fde(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                          const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->aid_stack_fde(items, n_items, fde, out, nullptr, nullptr);
}
int msckf_b200_batch_aid_stack_update_fde_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                               const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                               msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out) {
  if (!b || !iter || !iter_out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->aid_stack_fde(items, n_items, fde, out, iter, iter_out);
}
int msckf_b200_batch_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->landmarks(lm, nullptr, out);
}
int msckf_b200_batch_map_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         msckf_b200_landmark_result* out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->landmarks(lm, map, out);
}
int msckf_b200_batch_landmark_update_consensus(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                               const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                               msckf_b200_landmark_consensus_result* cons_out) {
  if (!b) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return b->ctx->landmarks(lm, map, out, cons, cons_out);
}

int msckf_b200_update_batch(msckf_b200_engine** engines, int n, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports,
                            int threads) {
  if (n <= 0) return 0;
  if (!engines || !tracks) return fail(MSCKF_B200_ERR_ARG, "null argument");
  // the engines already form a batch, in this order?
  CtxBase* g = engines[0] ? engines[0]->impl->group : nullptr;
  bool same = g && g->count() == n;
  for (int i = 0; same && i < n; ++i) same = engines[i] && g->member(i) == engines[i]->impl;
  if (same) {
    msckf_b200_batch tmp{g, engines[0]->impl->dtype};
    return msckf_b200_batch_update(&tmp, mode, tracks, reports, threads);
  }
  msckf_b200_batch* b = nullptr;
  int rc = msckf_b200_batch_create(engines, n, &b);
  if (rc != 0) return rc;
  rc = msckf_b200_batch_update(b, mode, tracks, reports, threads);
  const std::string keep = g_err;
  msckf_b200_batch_destroy(b);
  g_err = keep;
  return rc;
}
int msckf_b200_prune(msckf_b200_engine* e, const int* keep, int n_keep) { return e->impl->prune(keep, n_keep); }
int msckf_b200_num_clones(msckf_b200_engine* e) { return e->impl->M; }
int msckf_b200_get_state(msckf_b200_engine* e, void* imu, void* clone_poses) { return e->impl->get_state(imu, clone_poses); }
int msckf_b200_get_covariance(msckf_b200_engine* e, void* out) { return e->impl->get_covariance(out); }
int msckf_b200_nees(msckf_b200_engine* e, const double* truth_imu, const double* truth_poses, msckf_b200_nees_result* out) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return e->impl->solo_ctx()->nees(&truth_imu, &truth_poses, out);
}
int msckf_b200_aid_update(msckf_b200_engine* e, const msckf_b200_aid* aid, msckf_b200_aid_result* out) {
  if (!e || !aid) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (aid->model < 0) return fail(MSCKF_B200_ERR_ARG, "aid_update: unknown model");
  return e->impl->solo_ctx()->aid(aid, out);
}
int msckf_b200_aid_stack_update(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                msckf_b200_aid_result* out) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (n_items < 1) return fail(MSCKF_B200_ERR_ARG, "aid_stack_update: 1 to 8 items per stack");
  return e->impl->solo_ctx()->aid_stack(&items, &n_items, chi2_max, out, nullptr, nullptr);
}
int msckf_b200_aid_stack_update_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                     const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out, msckf_b200_aid_iter_result* iter_out) {
  if (!e || !iter || !iter_out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (n_items < 1) return fail(MSCKF_B200_ERR_ARG, "aid_stack_update_iter: 1 to 8 items per stack");
  return e->impl->solo_ctx()->aid_stack(&items, &n_items, chi2_max, out, iter, iter_out);
}
int msckf_b200_aid_stack_update_fde(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, const msckf_b200_aid_fde* fde,
                                    msckf_b200_aid_fde_result* out) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (n_items < 1) return fail(MSCKF_B200_ERR_ARG, "aid_stack_update_fde: 1 to 8 items per stack");
  return e->impl->solo_ctx()->aid_stack_fde(&items, &n_items, fde, out, nullptr, nullptr);
}
int msckf_b200_aid_stack_update_fde_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                         const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                         msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out) {
  if (!e || !iter || !iter_out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (n_items < 1) return fail(MSCKF_B200_ERR_ARG, "aid_stack_update_fde_iter: 1 to 8 items per stack");
  return e->impl->solo_ctx()->aid_stack_fde(&items, &n_items, fde, out, iter, iter_out);
}
int msckf_b200_standstill_update(msckf_b200_engine* e, const void* readings, int k, const msckf_b200_standstill* cfg,
                                 msckf_b200_standstill_result* out) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (k < 2 || k > kStandstillMaxReadings) return fail(MSCKF_B200_ERR_ARG, "standstill_update: 2 to 4096 readings");
  return e->impl->solo_ctx()->standstill(&readings, &k, cfg, out);
}
int msckf_b200_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out) {
  return msckf_b200_map_landmark_update(e, lm, nullptr, out);
}
// (an empty call with valid iteration settings only zeroes the result)
int msckf_b200_map_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                   msckf_b200_landmark_result* out) {
  if (!e || !lm || !out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  const bool it_ok = lm->max_iter >= 0 && lm->max_iter <= mb::kLmkMaxIter && std::isfinite(lm->tol) && lm->tol >= 0.0;
  if (lm->n_obs == 0 && it_ok) { memset(out, 0, sizeof(*out)); return 0; }
  return e->impl->solo_ctx()->landmarks(lm, map, out);
}
// (an empty call with valid settings zeroes the result; a consensus of no observations fails)
int msckf_b200_landmark_update_consensus(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                         msckf_b200_landmark_consensus_result* cons_out) {
  if (!e || !lm || !out) return fail(MSCKF_B200_ERR_ARG, "null argument");
  if (!cons || cons->hypotheses == 0) {
    if (cons_out) { memset(cons_out, 0, sizeof(*cons_out)); cons_out->best = -1; }
    return msckf_b200_map_landmark_update(e, lm, map, out);
  }
  if (lm->n_obs == 0) {
    LmkPlan p;
    RC(lmk_plan(*lm, nullptr, e->impl->M, "", p));
    RC(lmk_cons_plan(*lm, *cons, "", p));
    memset(out, 0, sizeof(*out));
    if (cons_out) { memset(cons_out, 0, sizeof(*cons_out)); cons_out->best = -1; cons_out->status = 1; }
    if (cons->scores)
      for (int k = 0; k < cons->hypotheses; ++k) cons->scores[k] = -1;
    return 0;
  }
  return e->impl->solo_ctx()->landmarks(lm, map, out, cons, cons_out);
}
int msckf_b200_set_covariance(msckf_b200_engine* e, const void* in) { return e->impl->set_covariance(in); }
int msckf_b200_get_counters(msckf_b200_engine* e, long long* counters) { return e->impl->get_counters(counters); }
int msckf_b200_last_delta_x(msckf_b200_engine* e, double* out, int cap) { return e->impl->last_dx(out, cap); }
int msckf_b200_rank_pivots(msckf_b200_engine* e, double* out, int cap) { return e->impl->rank_pivots(out, cap); }
int msckf_b200_stage_buffer(msckf_b200_engine* e, int which, void* out, int cap) {
  if (!e) return fail(MSCKF_B200_ERR_ARG, "null argument");
  return e->impl->stage_buffer(which, out, cap);
}
int msckf_b200_kernel_times(msckf_b200_engine* e, float* ms, const char** names, int cap) { return e->impl->solo_ctx()->kernel_times(ms, names, cap); }
int msckf_b200_tail_profile(msckf_b200_engine* e, unsigned long long* out, int cap) { return e->impl->tail_profile(out, cap); }
int msckf_b200_set_option(msckf_b200_engine* e, int key, double value) {
  if (key == 0) { e->impl->rank_thr = value; return 0; }  // (travels in UpdArgs: captured graphs stay valid)
  if (key == 1) { e->impl->profile = value != 0; return 0; }
  if (key == 2) { e->impl->use_graph = value != 0; e->impl->drop_graphs(); return 0; }
  if (key == 3) { e->impl->no_fused_tail = value == 0; return 0; }
  if (key == 4) { e->impl->use_pdl = value != 0; return 0; }
  if (key == 5) { e->impl->gram_mma = value != 0; return 0; }
  if (key == 8) { e->impl->stop_after_compression = value != 0; return 0; }  // (part of LaunchShape: graphs never mix the two)
  if (key == 7) {
    if (value != 0 && value != 1 && value != 2) return fail(MSCKF_B200_ERR_ARG, "option 7: 0, 1 or 2");
    e->impl->tail_chains = (int)value;
    return 0;
  }
  if (key == 6) {
    const int g = (int)value;
    if (g != 0 && g != 32 && g != 64 && g != 128) return fail(MSCKF_B200_ERR_ARG, "option 6: 0, 32, 64 or 128");
    e->impl->jac_group = g;
    return 0;
  }
  return fail(MSCKF_B200_ERR_ARG, "unknown option");
}
int msckf_b200_copy_state(msckf_b200_engine* dst, const msckf_b200_engine* src) { return dst->impl->copy_from(src->impl); }
long long msckf_b200_launch_count(const msckf_b200_engine* e) { return e->impl->launches; }
void* msckf_b200_stream(msckf_b200_engine* e) { return (void*)e->impl->stream; }
int msckf_b200_synchronize(msckf_b200_engine* e) { return e->impl->sync(); }
}
