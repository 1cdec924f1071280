// msckf_mono_b200/csrc/engine.cu -- host side of the H100 engine and the C-ABI of include/msckf_b200.h.
// One handle = one filter: device-resident covariance / clone poses / IMU state and workspaces.  Updates run through a
// launch context (Ctx): one stream, one packed pinned + device input arena ([UpdArgs per filter | track batches]), one packed
// report arena, a small cache of captured CUDA graphs.  Every engine has a private context; a msckf_b200_batch is a context
// shared by several engines -- the same kernels with the filter index in blockIdx.z.  No CPU fallback anywhere.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/msckf_b200.h"
#include "common.cuh"
#include "feature_kernels.cuh"
#include "gram_kernels.cuh"
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

constexpr int kMaxSplit = 16;
constexpr int kJacBatchGroup = 32;  // k_jac threads per track in a device batch (DESIGN.md 4.2)
constexpr int kTailCluster = 8;  // portable cluster size: the serial EKF tail runs on 8 SMs of one GPC
constexpr size_t kSmemBudget = 220 * 1024;  // dynamic shared memory per CTA, under H100's 227 KB opt-in limit
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
    CK(cudaMemset(d, 0, c));
    cap = c;
    return 0;
  }
  void release() {
    if (d) cudaFree(d);
    if (h) cudaFreeHost(h);
    d = h = nullptr; cap = 0;
  }
};

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
  int nf, mode, tri_gx, jac_gx, bd_gx, gram_gx, gram_gy, asm_gx, rows_gx, gemm_g, syrk_gx, tail_mask, pdl, gram_mma, jac_g, tail_nch;
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
  Arena in, rep;
  size_t in_used = 0, rep_used = 0;
  int device = 0;
  bool owns_stream = false;
  cudaStream_t stream2 = nullptr, stream3 = nullptr;  // side branches of the update (k_blockdiag, k_rows run beside k_gram)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_join2 = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  int st_mode = -1;
  bool staged = false, timed_region = false;
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
  int n_sm = 0;

  int init(int dev) {
    device = dev;
    CK(cudaSetDevice(device));
    CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
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
    in.release(); rep.release();
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
    // the private context's packed arenas, sized for a full batch (no pinned allocation inside the first update)
    RC(solo.in.ensure(solo.args_bytes() + up256(Plan<S>::in_bytes(Tmax, Omax)), nullptr));
    RC(solo.rep.ensure(up256(Plan<S>::rep_bytes(Tmax)), nullptr));
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
    free_batchws();
    RC(alloc_batchws());
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
    const S* r = (const S*)r_;
    CK(cudaSetDevice(device));
    for (int k0 = 0; k0 < k; k0 += mb::kPropMax) {
      mb::PropBatch<S> pb;
      pb.st = d_st; pb.P = d_P; pb.ldp = ldp; pb.M = M; pb.k = std::min(mb::kPropMax, k - k0); pb.pad_ = 0;
      pb.prof = profile ? d_prof : nullptr;
      for (int i = 0; i < pb.k; ++i)
        for (int j = 0; j < 7; ++j) pb.r[i][j] = r[7 * (size_t)(k0 + i) + j];
      mb::k_propagate<S><<<1, 256, 0, stream>>>(pb);
      launches++;
    }
    CK(cudaGetLastError());
    return 0;
  }

  int augment() override {
    if (!initialized) return fail(MSCKF_B200_ERR_STATE, "augment before initialize");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "augment with an un-fetched update pending");
    RC(ensure_clones(M + 1));
    CK(cudaSetDevice(device));
    mb::k_augment<S><<<1, 256, 0, stream>>>(d_st, d_P, ldp, M, d_poses);
    launches++;
    CK(cudaGetLastError());
    M += 1;
    return 0;
  }

  // everything the kernels need for this filter's slice of the update
  void fill_args(mb::UpdArgs<S>& a, const Plan<S>& p, int mode) const {
    memset(&a, 0, sizeof(a));
    a.n_tracks = p.N; a.M = M; a.Lmax = p.Lmax; a.ldp = ldp; a.ld = ld; a.n = 15 + 6 * M; a.mode = mode;
    if (p.N > 0 && mode != MSCKF_B200_TRIANGULATE) pivr_n = a.n;  // (the window may shrink before msckf_b200_rank_pivots is asked)
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
    if (n_keep < 0 || n_keep > M) return fail(MSCKF_B200_ERR_ARG, "prune: bad keep count");
    if (n_keep > 0 && !keep) return fail(MSCKF_B200_ERR_ARG, "prune: null keep list");
    if (busy) return fail(MSCKF_B200_ERR_STATE, "prune with an un-fetched update pending");
    for (int i = 0; i < n_keep; ++i)
      if (keep[i] < 0 || keep[i] >= M || (i && keep[i] <= keep[i - 1])) return fail(MSCKF_B200_ERR_ARG, "prune: keep[] must be ascending positions");
    if (n_keep == M) return 0;
    CK(cudaSetDevice(device));
    mb::KeepList kl;
    kl.n = n_keep;
    for (int i = 0; i < n_keep; ++i) kl.idx[i] = keep[i];
    const int n_new = 15 + 6 * n_keep;
    mb::k_gather<S><<<std::min(2 * num_sms(device), (n_new * n_new + 255) / 256), 256, 0, stream>>>(n_new, kl, d_P, d_P2, ldp, d_poses, d_poses2);
    launches++;
    CK(cudaGetLastError());
    std::swap(d_P, d_P2);      // (buffer addresses ride in UpdArgs, not in captured kernel arguments:
    std::swap(d_poses, d_poses2);  //  no synchronisation, and captured graphs stay valid)
    M = n_keep;
    return 0;
  }

  int get_state(void* imu_, void* poses_) override {
    CK(cudaSetDevice(device));
    std::vector<S> tmp;
    if (imu_) CK(cudaMemcpyAsync(h_st, d_st, sizeof(mb::DevState<S>), cudaMemcpyDeviceToHost, stream));
    if (poses_ && M > 0) {
      tmp.resize((size_t)mb::kPoseStride * M);
      CK(cudaMemcpyAsync(tmp.data(), d_poses, sizeof(S) * tmp.size(), cudaMemcpyDeviceToHost, stream));
    }
    CK(cudaStreamSynchronize(stream));  // one synchronisation for both copies
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
        const S* p = tmp.data() + mb::kPoseStride * k;
        o[7 * k] = p[4]; o[7 * k + 1] = p[5]; o[7 * k + 2] = p[6];
        o[7 * k + 3] = p[0]; o[7 * k + 4] = p[1]; o[7 * k + 5] = p[2]; o[7 * k + 6] = p[3];
      }
    }
    return 0;
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
    for (int o = 0; o < O; ++o)
      if ((unsigned)tr.clone_index[o] >= (unsigned)Mi) return fail(MSCKF_B200_ERR_ARG, "clone_index out of range");
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
  sh.asm_gx = std::min(4 * num_sms(device), (nmax_ * nmax_ + 255) / 256);
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
    CK(launch_k(mb::k_assemble<S>, dim3(sh.asm_gx, 1, nf), dim3(256), 0, stream, false, 1, A));
    launches++;
    mark("k_assemble");
    if (fork) CK(cudaStreamWaitEvent(stream, ev_join2, 0));
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
      rep->rank = p.h_mr[1];
    }
  }
  if (status != 0) return fail(status, "non-finite delta-x or covariance after the update (the update has been applied, like msckf.h:1369-1418 would), or the tail kernel's two chain CTAs lost their hand-off");
  return 0;
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
  int rc = msckf_b200_stage(e, mode, tracks);
  if (rc != 0) return rc;
  return e->impl->solo_ctx()->launch();
}
int msckf_b200_fetch(msckf_b200_engine* e, msckf_b200_report* report) { return e->impl->solo_ctx()->fetch(report); }
int msckf_b200_update(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* report) {
  int rc = msckf_b200_update_async(e, mode, tracks);
  if (rc != 0) {  // keep the real cause: clean up a half-started update without touching the error message
    CtxBase* c = e->impl->solo_ctx();
    if (c->pending) { const std::string keep = g_err; c->fetch(nullptr); g_err = keep; }
    return rc;
  }
  return e->impl->solo_ctx()->fetch(report);
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
  int rc = msckf_b200_batch_stage(b, mode, tracks, threads);
  if (rc != 0) return rc;
  return b->ctx->launch();
}
int msckf_b200_batch_fetch(msckf_b200_batch* b, msckf_b200_report* reports) { return b->ctx->fetch(reports); }
int msckf_b200_batch_update(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports, int threads) {
  int rc = msckf_b200_batch_update_async(b, mode, tracks, threads);
  if (rc != 0) {
    if (b->ctx->pending) { const std::string keep = g_err; b->ctx->fetch(nullptr); g_err = keep; }
    return rc;
  }
  return b->ctx->fetch(reports);
}
int msckf_b200_batch_kernel_times(msckf_b200_batch* b, float* ms, const char** names, int cap) { return b->ctx->kernel_times(ms, names, cap); }
long long msckf_b200_batch_launch_count(const msckf_b200_batch* b) { return b->ctx->launches; }
int msckf_b200_batch_jac_occupancy(const msckf_b200_batch* b) { return b->ctx->jac_ctas; }
void* msckf_b200_batch_stream(msckf_b200_batch* b) { return (void*)b->ctx->stream; }

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
int msckf_b200_set_covariance(msckf_b200_engine* e, const void* in) { return e->impl->set_covariance(in); }
int msckf_b200_get_counters(msckf_b200_engine* e, long long* counters) { return e->impl->get_counters(counters); }
int msckf_b200_last_delta_x(msckf_b200_engine* e, double* out, int cap) { return e->impl->last_dx(out, cap); }
int msckf_b200_rank_pivots(msckf_b200_engine* e, double* out, int cap) { return e->impl->rank_pivots(out, cap); }
int msckf_b200_kernel_times(msckf_b200_engine* e, float* ms, const char** names, int cap) { return e->impl->solo_ctx()->kernel_times(ms, names, cap); }
int msckf_b200_tail_profile(msckf_b200_engine* e, unsigned long long* out, int cap) { return e->impl->tail_profile(out, cap); }
int msckf_b200_set_option(msckf_b200_engine* e, int key, double value) {
  if (key == 0) { e->impl->rank_thr = value; return 0; }  // (travels in UpdArgs: captured graphs stay valid)
  if (key == 1) { e->impl->profile = value != 0; return 0; }
  if (key == 2) { e->impl->use_graph = value != 0; e->impl->drop_graphs(); return 0; }
  if (key == 3) { e->impl->no_fused_tail = value == 0; return 0; }
  if (key == 4) { e->impl->use_pdl = value != 0; return 0; }
  if (key == 5) { e->impl->gram_mma = value != 0; return 0; }
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
