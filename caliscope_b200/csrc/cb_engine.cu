// Host side of the caliscope_b200 bundle-adjustment engine: index build, the Levenberg-Marquardt
// driver and the C ABI declared in include/caliscope_b200.h.
//
// Replaces (behind the seam described in INTEGRATION.md) the call
//   scipy.optimize.least_squares(joint_residuals, x0, jac=joint_jacobian, method="trf", x_scale="jac", ...)
// at /root/reference/src/caliscope/core/capture_volume.py:387-411.  Termination tests and status
// codes follow scipy's (site-packages/scipy/optimize/_lsq/common.py:705-717, trf.py:466-475);
// the step itself is a damped Gauss-Newton step from the Schur-complement reduced camera system.
#include <cuda_runtime.h>
#include <dlfcn.h>
#if defined(__x86_64__)
#include <emmintrin.h>
#endif
#include <nvtx3/nvToolsExt.h>  // header-only; ranges show up in ncu / nsys timelines, no-ops otherwise

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <cub/cub.cuh>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/caliscope_b200.h"
#include "cb_kernels.cuh"
#include "cb_constraints.cuh"
#include "cb_triangulate.cuh"
#include "cb_bootstrap.cuh"
#include "cb_peer.cuh"

namespace {

thread_local std::string g_last_error;

struct NvtxRange {  // scoped NVTX range
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
std::atomic<long long> g_launches{0};

#define CB_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      g_last_error = std::string(#expr) + ": " + cudaGetErrorString(_e);                           \
      return CB_E_CUDA;                                                                            \
    }                                                                                              \
  } while (0)

#define CB_TRY(expr)                \
  do {                              \
    int _r = (expr);                \
    if (_r != CB_OK) return _r;     \
  } while (0)

#define CB_LAUNCH(kernel, grid, block, smem, stream, ...)                 \
  do {                                                                    \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);           \
    g_launches.fetch_add(1, std::memory_order_relaxed);                   \
  } while (0)

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------
// NCCL, resolved at run time from the libnccl the process already has loaded (torch's bundled copy):
// no link-time dependency, no second NCCL in the address space.
// ------------------------------------------------------------------------------------------
}  // namespace

// symmetric IPC buffer of one rank + the mapped views of its peers (cb_peer.cuh)
struct CbPeerGroup {
  int rank = 0, world = 1, device = 0;
  size_t cap = 0;  // doubles per data buffer
  size_t bytes = 0;
  void* base = nullptr;
  void* peer_base[cb::PEER_MAXW] = {};
  cb::PeerTable tab = {};
  unsigned long long epoch_big = 0, epoch_small = 0;
  bool connected = false;
  bool poisoned = false;  // a solve failed part-way: the ranks' epochs may be out of step, the group must be re-created
};

namespace {

struct NcclApi {
  bool ok = false;
  std::string err;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /* ncclUniqueId by value */ struct UidBlob, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
struct UidBlob { char internal[128]; };

NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = nullptr;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      h = dlopen(name, RTLD_NOW | RTLD_NOLOAD);  // only an already-loaded library
      if (h) break;
    }
    if (!h)
      for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
        h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
      }
    if (!h) { api.err = "libnccl.so.2 not found in the process (import torch first)"; return; }
    api.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void**, int, UidBlob, int))dlsym(h, "ncclCommInitRank");
    api.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(h, "ncclAllReduce");
    api.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.CommDestroy;
    if (!api.ok) api.err = "libnccl is missing ncclGetUniqueId / ncclCommInitRank / ncclAllReduce / ncclCommDestroy";
  });
  return api;
}

// sum-all-reduce of n doubles in place through whichever transport the options carry
int do_allreduce(const CbBaOptions* opt, double* buf, long long n, cudaStream_t st) {
  if (opt->peer_group) {
    CbPeerGroup* g = (CbPeerGroup*)opt->peer_group;
    if (n > cb::PEER_SMALL_N) { g_last_error = "peer transport: unexpected all-reduce length"; return CB_E_INVALID; }
    CB_LAUNCH(cb::peer_small_allreduce_kernel, 1, 32, 0, st, buf, (int)n, g->tab, ++g->epoch_small);
    return CB_OK;
  }
  if (opt->nccl_comm) {
    NcclApi& a = nccl();
    if (!a.ok) { g_last_error = a.err; return CB_E_UNSUPPORTED; }
    const int rc = a.AllReduce(buf, buf, (size_t)n, /*ncclFloat64*/ 8, /*ncclSum*/ 0, opt->nccl_comm, st);
    if (rc != 0) {
      g_last_error = std::string("ncclAllReduce: ") + (a.GetErrorString ? a.GetErrorString(rc) : "error");
      return CB_E_CALLBACK;
    }
    return CB_OK;
  }
  if (opt->allreduce(opt->allreduce_user, buf, n, (void*)st) != 0) {
    g_last_error = "all-reduce callback failed";
    return CB_E_CALLBACK;
  }
  return CB_OK;
}

inline bool sharded(const CbBaOptions* opt) { return opt && (opt->allreduce || opt->nccl_comm || opt->peer_group); }

// Process-wide caching allocator: repeated problem_create / destroy cycles (one per
// CaptureVolume.optimize call: linear -> soft_l1 -> filter -> linear) reuse device and pinned
// blocks instead of paying cudaMalloc / cudaFree / cudaMallocHost each time.
struct BlockCache {
  std::mutex mu;
  std::multimap<std::pair<int, size_t>, void*> free_dev;  // (device, bytes) -> ptr
  std::map<void*, std::pair<int, size_t>> live_dev;
  std::multimap<size_t, void*> free_host;
  std::map<void*, size_t> live_host;
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCached = 16ull << 30;
};
BlockCache g_cache;

size_t round_bytes(size_t b) { return (std::max<size_t>(b, 1) + 511) & ~(size_t)511; }

int cached_malloc(void** p, size_t bytes) {
  bytes = round_bytes(bytes);
  int dev = 0;
  cudaGetDevice(&dev);
  {
    std::lock_guard<std::mutex> lk(g_cache.mu);
    auto it = g_cache.free_dev.find({dev, bytes});
    if (it != g_cache.free_dev.end()) {
      *p = it->second;
      g_cache.free_dev.erase(it);
      g_cache.cached_bytes -= bytes;
      g_cache.live_dev[*p] = {dev, bytes};
      return CB_OK;
    }
  }
  cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) {
    // release the cache and retry once
    std::vector<void*> drop;
    {
      std::lock_guard<std::mutex> lk(g_cache.mu);
      for (auto& kv : g_cache.free_dev) drop.push_back(kv.second);
      g_cache.free_dev.clear();
      g_cache.cached_bytes = 0;
    }
    cudaGetLastError();
    for (void* q : drop) cudaFree(q);
    e = cudaMalloc(p, bytes);
  }
  if (e != cudaSuccess) {
    g_last_error = std::string("cudaMalloc: ") + cudaGetErrorString(e);
    cudaGetLastError();
    *p = nullptr;
    return CB_E_NOMEM;
  }
  std::lock_guard<std::mutex> lk(g_cache.mu);
  g_cache.live_dev[*p] = {dev, bytes};
  return CB_OK;
}

void cached_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_cache.mu);
  auto it = g_cache.live_dev.find(p);
  if (it == g_cache.live_dev.end()) { cudaFree(p); return; }
  auto key = it->second;
  g_cache.live_dev.erase(it);
  if (g_cache.cached_bytes + key.second > BlockCache::kMaxCached) { cudaFree(p); return; }
  g_cache.free_dev.insert({key, p});
  g_cache.cached_bytes += key.second;
}

int cached_malloc_host(void** p, size_t bytes) {
  bytes = round_bytes(bytes);
  {
    std::lock_guard<std::mutex> lk(g_cache.mu);
    auto it = g_cache.free_host.find(bytes);
    if (it != g_cache.free_host.end()) {
      *p = it->second;
      g_cache.free_host.erase(it);
      g_cache.live_host[*p] = bytes;
      return CB_OK;
    }
  }
  cudaError_t e = cudaMallocHost(p, bytes);
  if (e != cudaSuccess) {
    g_last_error = std::string("cudaMallocHost: ") + cudaGetErrorString(e);
    cudaGetLastError();
    *p = nullptr;
    return CB_E_NOMEM;
  }
  std::lock_guard<std::mutex> lk(g_cache.mu);
  g_cache.live_host[*p] = bytes;
  return CB_OK;
}

void cached_free_host(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_cache.mu);
  auto it = g_cache.live_host.find(p);
  if (it == g_cache.live_host.end()) { cudaFreeHost(p); return; }
  g_cache.free_host.insert({it->second, p});
  g_cache.live_host.erase(it);
}

struct ScopedFree {
  std::vector<void*> dev, host;
  ~ScopedFree() {
    for (void* q : dev) cached_free(q);
    for (void* q : host) cached_free_host(q);
  }
};

// memcpy into a pinned staging block with NON-TEMPORAL stores.  Lines written with ordinary stores sit dirty in the private
// caches of the staging threads, and the DMA engine that reads the block microseconds later has to snoop them out one by
// one, far slower than reading a block at rest; streaming stores go through the
// write-combining buffers straight to memory.  dst must be 16-byte aligned (pinned blocks are page aligned, units are
// multiples of 512 KB); src may be anything.
inline void stream_copy(void* dst, const void* src, size_t n) {
#if defined(__x86_64__) && defined(__SSE2__)
  if (((uintptr_t)dst & 15u) == 0) {
    char* d = (char*)dst;
    const char* s2 = (const char*)src;
    size_t i = 0;
    for (; i + 64 <= n; i += 64) {
      const __m128i a = _mm_loadu_si128((const __m128i*)(s2 + i)), b = _mm_loadu_si128((const __m128i*)(s2 + i + 16));
      const __m128i c = _mm_loadu_si128((const __m128i*)(s2 + i + 32)), e = _mm_loadu_si128((const __m128i*)(s2 + i + 48));
      _mm_stream_si128((__m128i*)(d + i), a);
      _mm_stream_si128((__m128i*)(d + i + 16), b);
      _mm_stream_si128((__m128i*)(d + i + 32), c);
      _mm_stream_si128((__m128i*)(d + i + 48), e);
    }
    if (i < n) std::memcpy(d + i, s2 + i, n - i);
    _mm_sfence();
    return;
  }
#endif
  std::memcpy(dst, src, n);
}

// A few long-lived host threads for staging copies.  Creating threads per call costs ~50 us each and a first CUDA call on
// a fresh thread binds the context again; the pool is started on first use and lives as long as the process.
class WorkerPool {
 public:
  static WorkerPool& get() {
    static WorkerPool* pool = new WorkerPool();  // never destroyed: workers may outlive static destruction order
    return *pool;
  }
  int size() const { return (int)threads_.size(); }
  void submit(std::function<void()> f) {
    {
      std::lock_guard<std::mutex> lk(mu_);
      q_.push_back(std::move(f));
    }
    cv_.notify_one();
  }

 private:
  WorkerPool() {
    unsigned hw = std::thread::hardware_concurrency();
    int n = (int)std::min<unsigned>(hw > 2 ? hw - 1 : 1, 12u);
    for (int i = 0; i < n; ++i) {
      threads_.emplace_back([this] {
        for (;;) {
          std::function<void()> f;
          {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [this] { return !q_.empty(); });
            f = std::move(q_.front());
            q_.pop_front();
          }
          f();
        }
      });
      threads_.back().detach();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_;
  std::deque<std::function<void()>> q_;
  std::vector<std::thread> threads_;
};

// Pageable host memory -> device at PCIe speed: cudaMemcpyAsync from pageable memory goes through one driver staging
// buffer, well below PCIe speed, so the caller's arrays (NumPy, pageable) are copied by pool threads into a pinned block in
// chunks; the calling thread queues each chunk's DMA in order as soon as it is staged (one thread talks to the driver)
// and copies chunks itself while it would otherwise wait.  Returns once the source has been read completely (the caller
// may free it); the pinned block must stay alive until `st` has drained (sf.host frees it at scope exit of the caller,
// which synchronises first).
int staged_h2d(void* d_dst, const void* h_src, size_t bytes, cudaStream_t st, ScopedFree& sf, int n_threads = 6) {
  if (bytes == 0) return CB_OK;
  void* pin = nullptr;
  CB_TRY(cached_malloc_host(&pin, bytes));
  sf.host.push_back(pin);
  // Two granularities.  Host threads copy 512 KB units (enough units to keep 6-8 threads busy on a 4 MB array); the DMA is
  // queued in 4 MB blocks: every cudaMemcpyAsync has a fixed copy-engine cost on top of its bytes, so small blocks
  // throttle the engine and large ones expose the staging.
  const size_t unit = (size_t)512 << 10, units_per_block = 8;
  const size_t n_units = (bytes + unit - 1) / unit;
  const size_t n_blocks = (n_units + units_per_block - 1) / units_per_block;
  struct Shared {
    std::atomic<size_t> next{0};
    std::vector<std::atomic<unsigned char>> done;
    explicit Shared(size_t n) : done(n) { for (auto& d : done) d.store(0, std::memory_order_relaxed); }
  };
  auto sh = std::make_shared<Shared>(n_units);
  auto copy_one = [sh, pin, h_src, bytes, unit, n_units]() -> bool {
    const size_t c = sh->next.fetch_add(1);
    if (c >= n_units) return false;
    const size_t off = c * unit, sz = std::min(unit, bytes - off);
    stream_copy((char*)pin + off, (const char*)h_src + off, sz);
    sh->done[c].store(1, std::memory_order_release);
    return true;
  };
  static const bool prof = std::getenv("CB_PROFILE_CREATE") != nullptr;
  const auto t0 = std::chrono::steady_clock::now();
  const int helpers = (int)std::min<size_t>((size_t)std::max(0, std::min(n_threads, WorkerPool::get().size())), n_units > 1 ? n_units - 1 : 0);
  for (int t = 0; t < helpers; ++t)
    WorkerPool::get().submit([copy_one] { while (copy_one()) {} });
  bool failed = false;
  double wait_ms = 0.0, issue_ms = 0.0;
  size_t own = 0;
  cudaEvent_t pe0 = nullptr, pe1 = nullptr;
  if (prof) { cudaEventCreate(&pe0); cudaEventCreate(&pe1); cudaEventRecord(pe0, st); }
  for (size_t blk = 0; blk < n_blocks; ++blk) {
    const size_t u0 = blk * units_per_block, u1 = std::min(n_units, u0 + units_per_block);
    const auto a = std::chrono::steady_clock::now();
    for (size_t c = u0; c < u1; ++c)
      while (!sh->done[c].load(std::memory_order_acquire)) {
        if (copy_one()) ++own; else std::this_thread::yield();
      }
    const auto b = std::chrono::steady_clock::now();
    const size_t off = u0 * unit, sz = std::min(bytes, u1 * unit) - off;
    if (!failed && cudaMemcpyAsync((char*)d_dst + off, (char*)pin + off, sz, cudaMemcpyHostToDevice, st) != cudaSuccess) failed = true;
    if (prof) {
      const auto e = std::chrono::steady_clock::now();
      wait_ms += std::chrono::duration<double, std::milli>(b - a).count();
      issue_ms += std::chrono::duration<double, std::milli>(e - b).count();
    }
  }
  if (prof) {
    const double host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    cudaEventRecord(pe1, st);
    cudaEventSynchronize(pe1);
    float dma_ms = 0.f;
    cudaEventElapsedTime(&dma_ms, pe0, pe1);
    const double all_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    cudaEventDestroy(pe0); cudaEventDestroy(pe1);
    std::fprintf(stderr, "[stage] %6.1f MB, %d helpers, %zu DMA blocks: host %.3f ms (units %.3f, %zu by the issuer; cudaMemcpyAsync calls %.3f); "
                         "device first->last copy %.3f ms = %.1f GB/s; staged + landed %.3f ms\n",
                 bytes / 1e6, helpers, n_blocks, host_ms, wait_ms, own, issue_ms, dma_ms, bytes / 1e6 / std::max(dma_ms, 1e-3f), all_ms);
  }
  if (failed) { g_last_error = std::string("staged host-to-device copy: ") + cudaGetErrorString(cudaGetLastError()); return CB_E_CUDA; }
  return CB_OK;
}

int select_device(int device) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    g_last_error = "no CUDA device";
    return CB_E_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { g_last_error = "device index out of range"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(device));
  return CB_OK;
}

template <typename T>
int dalloc(T** p, size_t n) {
  return cached_malloc((void**)p, std::max<size_t>(n, 1) * sizeof(T));
}

}  // namespace

// One captured LM trial (ensure_graph), keyed by everything that is baked into the captured launches.  A failure to build
// it is remembered for its key, so that later solves go straight to the fallback.
struct TrialGraph {
  struct Key {
    void *nccl, *peer; int rank, world;
    bool operator==(const Key& o) const { return nccl == o.nccl && peer == o.peer && rank == o.rank && world == o.world; }
  };
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  Key key = {};
  bool valid = false, failed = false;
  int n_kernels = 0;  // kernels of one trial
};

struct CbBaProblem {
  int device = 0, num_sms = 132;
  int n_cams = 0, n_pts = 0, P = 6, nP = 0, n_obs = 0, n_params = 0;
  int LD = 0, n_blk = 0, n_tiles = 0, n_split = 1, k_chunks = 0, K_pad = 0;
  int n_chunks = 0, pt_grid = 0, pt_lanes = 32, n_dups = 0;
  int cam_in_smem = 0;
  size_t pt_smem = 0, bs_smem = 0;
  std::vector<int> h_cam_off;   // caller's layout: x offset of caller camera c
  std::vector<int> h_perm, h_slot;  // internal slot i holds caller camera h_perm[i]; h_slot[c] = slot of caller camera c
  std::vector<int> h_iflags;    // flags by internal slot
  bool order_auto = false, order_identity = true;
  int ncp = 0;                  // total camera parameters in x
  int *d_cam_xoff = nullptr, *d_cam_slot = nullptr, *d_klist = nullptr;
  bool schur_sparse = false;
  double schur_flop_issued = 0.0;  // flops one schur_syrk_kernel launch issues (dense tiles or compacted lists)
  double schur_rows_dense = 0.0, schur_rows_listed = 0.0;  // weighted k rows the Schur product streams: all vs listed
  std::vector<void*> allocs;
  // problem tables
  int* d_cam_flags = nullptr;
  double* d_cam_const = nullptr;
  double2 *d_cm_xy = nullptr, *d_pm_xy = nullptr;
  int *d_cm_pt = nullptr, *d_cm_orig = nullptr, *d_cam_start = nullptr;
  int *d_chunk_cam = nullptr, *d_chunk_begin = nullptr, *d_chunk_end = nullptr, *d_cam_chunk_start = nullptr;
  int *d_pt_start = nullptr, *d_pm_orig = nullptr, *d_pm_cam = nullptr, *d_pm_pt = nullptr;
  const int *d_obs_cam = nullptr, *d_obs_pt = nullptr;  // caller-order observation list (owned unless the caller's)
  const double* d_obs_xy = nullptr;
  std::vector<int> h_cam_flags;
  std::vector<double> h_cam_const;
  int *d_tile_of = nullptr, *d_tile_slot_start = nullptr, *d_tile_slots = nullptr;
  cb::SyItem* d_items = nullptr;
  int n_items = 0, n_slots = 0;
  unsigned char* d_active = nullptr;
  double *d_lo = nullptr, *d_hi = nullptr;
  // work buffers (index [2]: current / trial point, selected on the device by LmState::cur)
  double *d_x = nullptr, *d_xc[2] = {nullptr, nullptr}, *d_xp4[2] = {nullptr, nullptr};
  double *d_camtab[2] = {nullptr, nullptr}, *d_Upk[2] = {nullptr, nullptr}, *d_gc[2] = {nullptr, nullptr},
         *d_costsum[2] = {nullptr, nullptr};
  double *d_partial = nullptr, *d_camcost = nullptr, *d_V6 = nullptr, *d_gp = nullptr, *d_Dp2 = nullptr,
         *d_Dc2 = nullptr, *d_Linv6 = nullptr, *d_tvec = nullptr, *d_Zt = nullptr, *d_part = nullptr,
         *d_tpart = nullptr, *d_red = nullptr, *d_Minv = nullptr, *d_dc = nullptr, *d_dp = nullptr,
         *d_bpart = nullptr, *d_sc = nullptr, *d_red2 = nullptr, *d_out2 = nullptr;
  unsigned long long* d_gmax = nullptr;
  unsigned int* d_counter = nullptr;
  cb::LmState* d_state = nullptr;
  cb::LmState* h_state = nullptr;  // pinned, 4 slots
  cb::LmLogRow* d_log = nullptr;
  int log_cap = 4096;
  double* h_x = nullptr;   // pinned staging for x
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev_state[2] = {nullptr, nullptr};
  cudaEvent_t ev_pp[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};  // point-pass / Schur brackets (direct mode)
  cudaStream_t cap_stream = nullptr;
  TrialGraph trial_graph;  // sharded solves: one graph launch per trial
  TrialGraph loop_graph;   // one GPU: ONE graph whose body (a WHILE conditional node) is the LM trial
  // pcg launch configuration
  int pcg_cs = 1, pcg_rows = 0, pcg_mode = 2, pcg_cl = 1, pcg_npa = 0;
  bool direct_solve = false;  // n_camera_params <= DIRECT_MAX_N: prep, dense LDL^T and camera step in one CTA (small_rig_step_kernel)
  size_t direct_smem = 0;
  size_t pcg_smem = 0;
  // rigid-distance constraints (optional)
  int n_c = 0, n_comp = 0, n_dim_max = 0, n_cblk = 0;
  cb::ConstraintTables ct = {};
  double *d_c_rs[2] = {nullptr, nullptr}, *d_c_dirw[2] = {nullptr, nullptr}, *d_compL = nullptr, *d_gpt = nullptr;
  int* d_pt_comp = nullptr;
  size_t comp_build_smem = 0, comp_back_smem = 0;
  std::vector<int> h_ga, h_gb;
  std::vector<double> h_cdist, h_cw;
  int red_slots = 64;
  CbPeerGroup* peer = nullptr;  // set for the duration of a solve that uses the peer transport
  // cb_ba_covariance scratch, allocated on its first call: sweep matrix (cov_n^2), column panel, pivot inverse, S_F^-1,
  // diag of the sweep matrix, pseudo-inverse roots and ranks of V, point covariances, free mask, failure indices
  int cov_n = 0;
  double *d_covA = nullptr, *d_covC = nullptr, *d_covD = nullptr, *d_covS = nullptr, *d_covDiag = nullptr,
         *d_covR = nullptr, *d_covPt = nullptr;
  int *d_covRank = nullptr, *d_covFail = nullptr;
  unsigned char* d_covFree = nullptr;
  float cov_ms[3] = {0.f, 0.f, 0.f};  // last call: linearisation + Schur, dense inverse, point marginals
  size_t red_len() const { return (size_t)nP * nP + 3 * (size_t)nP + 1 + red_slots; }
  cb::CPtr2 c_camtab() const { return {{d_camtab[0], d_camtab[1]}}; }
  cb::Ptr2 m_camtab() const { return {{d_camtab[0], d_camtab[1]}}; }
  cb::CPtr2 c_xp() const { return {{d_xp4[0], d_xp4[1]}}; }
  cb::Ptr2 m_xp() const { return {{d_xp4[0], d_xp4[1]}}; }
  cb::Ptr2 m_xc() const { return {{d_xc[0], d_xc[1]}}; }
  cb::CPtr2 c_Upk() const { return {{d_Upk[0], d_Upk[1]}}; }
  cb::Ptr2 m_Upk() const { return {{d_Upk[0], d_Upk[1]}}; }
  cb::CPtr2 c_gc() const { return {{d_gc[0], d_gc[1]}}; }
  cb::Ptr2 m_gc() const { return {{d_gc[0], d_gc[1]}}; }
  cb::CPtr2 c_costsum() const { return {{d_costsum[0], d_costsum[1]}}; }
  cb::Ptr2 m_costsum() const { return {{d_costsum[0], d_costsum[1]}}; }
  cb::CPtr2 c_crs() const { return {{d_c_rs[0], d_c_rs[1]}}; }
  cb::Ptr2 m_crs() const { return {{d_c_rs[0], d_c_rs[1]}}; }
  cb::CPtr2 c_cdirw() const { return {{d_c_dirw[0], d_c_dirw[1]}}; }
  cb::Ptr2 m_cdirw() const { return {{d_c_dirw[0], d_c_dirw[1]}}; }
};

namespace {

template <typename T>
int palloc(CbBaProblem* p, T** ptr, size_t n) {
  CB_TRY(dalloc(ptr, n));
  p->allocs.push_back((void*)*ptr);
  return CB_OK;
}

int bits_for(unsigned long long v) {
  int b = 1;
  while (b < 64 && (v >> b) != 0ull) ++b;
  return b;
}

void destroy_graph(TrialGraph& g) {
  if (g.exec) cudaGraphExecDestroy(g.exec);
  if (g.graph) cudaGraphDestroy(g.graph);
  g.exec = nullptr; g.graph = nullptr; g.valid = false; g.n_kernels = 0;
}

// ------------------------------------------------------------------------------------------
// index build
// ------------------------------------------------------------------------------------------
// one non-blocking side stream per (thread, device) for copies that overlap the index build
cudaStream_t side_stream() {
  thread_local std::map<int, cudaStream_t> streams;
  int dev = 0;
  cudaGetDevice(&dev);
  auto it = streams.find(dev);
  if (it != streams.end()) return it->second;
  cudaStream_t s = nullptr;
  cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  streams[dev] = s;
  return s;
}

// Internal camera order.  The reduced system and the Schur factor are laid out by camera slot; the Schur product only
// has to visit, per pair of 96-column tiles, the points seen from BOTH tiles.  When visibility is local (ring rigs:
// a point is seen by a few neighbouring cameras) but the caller's numbering is not (e.g. ring by ring), putting cameras
// that share points next to each other empties most tile pairs.  Order = the caller's (`cam_order` = slot -> camera,
// REQUIRED to be the same on every rank of a sharded solve), or chosen here from a sampled co-visibility matrix
// (greedy chain: next = the unplaced camera sharing most points with the last 16 placed), kept only if it lowers the
// number of (point, tile pair) incidences.
int choose_camera_order(CbBaProblem* p, const int* cam_order, cudaStream_t st) {
  const int nc = p->n_cams;
  p->h_perm.resize(nc); p->h_slot.resize(nc);
  for (int i = 0; i < nc; ++i) p->h_perm[i] = i;
  p->order_auto = false;
  if (cam_order) {
    std::vector<char> seen(nc, 0);
    for (int i = 0; i < nc; ++i) {
      const int c = cam_order[i];
      if (c < 0 || c >= nc || seen[c]) { g_last_error = "cam_order is not a permutation of 0..n_cams-1"; return CB_E_INVALID; }
      seen[c] = 1;
      p->h_perm[i] = c;
    }
  } else {
    const int cams_per_tile = std::max(1, cb::SY_TILE / p->P);
    const double avg = (double)p->n_obs / std::max(p->n_pts, 1);
    if (p->n_blk >= 3 && avg <= nc / 3.0) {
      p->order_auto = true;
      const int stride = std::max(1, p->n_pts / 8192), ns = cdiv(p->n_pts, stride);
      unsigned int* d_W;
      CB_TRY(dalloc(&d_W, (size_t)nc * nc));
      ScopedFree sf; sf.dev.push_back(d_W);
      CB_CUDA(cudaMemsetAsync(d_W, 0, sizeof(unsigned int) * nc * nc, st));
      CB_LAUNCH(cb::covis_kernel, cdiv((long long)ns * 32, 256), 256, 0, st, p->d_pt_start, p->d_pm_cam, p->n_pts, stride, nc, d_W);
      std::vector<unsigned int> W((size_t)nc * nc);
      CB_CUDA(cudaMemcpyAsync(W.data(), d_W, sizeof(unsigned int) * nc * nc, cudaMemcpyDeviceToHost, st));
      CB_CUDA(cudaStreamSynchronize(st));
      // greedy chain
      std::vector<char> placed(nc, 0);
      std::vector<int> order;
      int start = 0;
      unsigned long long best = ~0ull;
      for (int c = 0; c < nc; ++c) {
        unsigned long long tot = 0;
        for (int q = 0; q < nc; ++q) if (q != c) tot += W[(size_t)c * nc + q];
        if (tot < best) { best = tot; start = c; }
      }
      order.push_back(start); placed[start] = 1;
      while ((int)order.size() < nc) {
        int pick = -1;
        unsigned long long bw = 0;
        const int lo = std::max(0, (int)order.size() - cams_per_tile);
        for (int c = 0; c < nc; ++c) {
          if (placed[c]) continue;
          unsigned long long w = 0;
          for (int k = lo; k < (int)order.size(); ++k) w += W[(size_t)c * nc + order[k]];
          if (pick < 0 || w > bw) { pick = c; bw = w; }
        }
        order.push_back(pick); placed[pick] = 1;
      }
      // keep it only if it lowers the co-visibility mass that falls OUTSIDE the diagonal tiles (pairs of cameras in
      // different tiles that share points are what forces off-diagonal tile pairs to be visited)
      auto off_mass = [&](const std::vector<int>& ord) {
        std::vector<int> tile(nc);
        for (int i = 0; i < nc; ++i) tile[ord[i]] = (i * p->P) / cb::SY_TILE;
        unsigned long long m = 0;
        for (int a = 0; a < nc; ++a)
          for (int b = 0; b < nc; ++b)
            if (tile[a] != tile[b]) m += W[(size_t)a * nc + b];
        return m;
      };
      std::vector<int> ident(nc);
      for (int i = 0; i < nc; ++i) ident[i] = i;
      if (off_mass(order) < 0.8 * off_mass(ident)) p->h_perm = order;
    }
  }
  p->order_identity = true;
  for (int i = 0; i < nc; ++i) {
    p->h_slot[p->h_perm[i]] = i;
    if (p->h_perm[i] != i) p->order_identity = false;
  }
  CB_CUDA(cudaMemcpyAsync(p->d_cam_slot, p->h_slot.data(), sizeof(int) * nc, cudaMemcpyHostToDevice, st));
  return CB_OK;
}

// The image coordinates (two thirds of an upload from host memory) are only needed by the LAST index-build kernels: a
// background thread stages them through pinned memory on a side stream while the calling thread queues the index sorts.
struct XyUpload {
  bool started = false;
  std::atomic<int> finished{0};
  cudaEvent_t ev = nullptr;
  int rc = CB_OK;
  std::string err;
  ScopedFree pinned;  // the staging block: released after the destructor body has waited for its DMA
  // wait for the staging task, then make `st` wait for the copies it queued
  void join() {
    if (!started) return;
    while (!finished.load(std::memory_order_acquire)) std::this_thread::yield();
    started = false;
  }
  int wait(cudaStream_t st) {
    join();
    if (rc != CB_OK) { g_last_error = err; return rc; }
    if (ev) CB_CUDA(cudaStreamWaitEvent(st, ev, 0));
    return CB_OK;
  }
  ~XyUpload() {
    join();
    if (ev) { cudaEventSynchronize(ev); cudaEventDestroy(ev); }  // the pinned staging block outlives its DMA on every path
  }
};

int build_indices(CbBaProblem* p, const int* d_obs_cam, const int* d_obs_pt, const double* d_obs_xy,
                  const int* cam_order, cudaStream_t st, XyUpload* xy_upload) {
  const int n = p->n_obs;
  const int TB = 256, G = cdiv(std::max(n, 1), TB);
  ScopedFree sf;
  int* d_bad;
  CB_TRY(dalloc(&d_bad, 2)); sf.dev.push_back(d_bad);
  CB_CUDA(cudaMemsetAsync(d_bad, 0, 2 * sizeof(int), st));
  CB_LAUNCH(cb::validate_kernel, G, TB, 0, st, d_obs_cam, d_obs_pt, n, p->n_cams, p->n_pts, d_bad);

  unsigned long long *k_in, *k_out;
  int *v_in, *v_out, *pm_pt, *pm_cam, *cm_cam;
  CB_TRY(dalloc(&k_in, n)); sf.dev.push_back(k_in);
  CB_TRY(dalloc(&k_out, n)); sf.dev.push_back(k_out);
  CB_TRY(dalloc(&v_in, n)); sf.dev.push_back(v_in);
  CB_TRY(dalloc(&v_out, n)); sf.dev.push_back(v_out);
  CB_TRY(dalloc(&cm_cam, n)); sf.dev.push_back(cm_cam);
  pm_pt = p->d_pm_pt; pm_cam = p->d_pm_cam;

  // temp storage for cub
  size_t tb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, k_in, k_out, v_in, v_out, n, 0, 64, st);
  void* d_tmp;
  CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tb, 16))); sf.dev.push_back(d_tmp);

  // (1) point-major order: key = pt * n_cams + cam, stable -> ties keep caller order
  CB_LAUNCH(cb::make_keys_kernel, G, TB, 0, st, d_obs_pt, d_obs_cam, (long long)p->n_cams, n, k_in, v_in);
  const int kb = bits_for((unsigned long long)p->n_pts * (unsigned long long)p->n_cams);
  CB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, k_in, k_out, v_in, p->d_pm_orig, n, 0, kb, st));
  g_launches.fetch_add(4);
  CB_LAUNCH(cb::split_keys_kernel, G, TB, 0, st, k_out, (long long)p->n_cams, n, pm_pt, pm_cam);
  CB_LAUNCH(cb::lower_bound_kernel, cdiv(p->n_pts + 1, TB), TB, 0, st, pm_pt, n, p->n_pts, p->d_pt_start);
  CB_LAUNCH(cb::count_dups_kernel, G, TB, 0, st, pm_pt, pm_cam, n, d_bad + 1);
  // (1b) internal camera order (see choose_camera_order), then pm_cam := internal slots
  CB_TRY(choose_camera_order(p, cam_order, st));
  if (!p->order_identity) CB_LAUNCH(cb::remap_kernel, G, TB, 0, st, pm_cam, (const int*)p->d_cam_slot, n);
  // (2) camera-major order: key = cam * n_pts + pt over the point-major positions (stable)
  CB_LAUNCH(cb::make_keys_kernel, G, TB, 0, st, pm_cam, pm_pt, (long long)p->n_pts, n, k_in, v_in);
  CB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, k_in, k_out, v_in, v_out, n, 0, kb, st));
  g_launches.fetch_add(4);
  CB_LAUNCH(cb::split_keys_kernel, G, TB, 0, st, k_out, (long long)p->n_pts, n, cm_cam, v_in);
  CB_LAUNCH(cb::lower_bound_kernel, cdiv(p->n_cams + 1, TB), TB, 0, st, cm_cam, n, p->n_cams, p->d_cam_start);
  if (xy_upload) CB_TRY(xy_upload->wait(st));
  CB_LAUNCH(cb::cm_gather_kernel, G, TB, 0, st, v_out, p->d_pm_orig, pm_pt,
            reinterpret_cast<const double2*>(d_obs_xy), n, p->d_cm_pt, p->d_cm_orig, p->d_cm_xy);
  CB_LAUNCH(cb::pm_gather_kernel, G, TB, 0, st, p->d_pm_orig, reinterpret_cast<const double2*>(d_obs_xy), n, p->d_pm_xy);
  // (3) chunk table (host, n_cams + 1 integers)
  std::vector<int> cam_start(p->n_cams + 1);
  int bad[2] = {0, 0};
  CB_CUDA(cudaMemcpyAsync(cam_start.data(), p->d_cam_start, sizeof(int) * (p->n_cams + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(bad, d_bad, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  if (bad[0]) {
    g_last_error = "obs_cam / obs_pt index out of range in " + std::to_string(bad[0]) + " observations";
    return CB_E_INVALID;
  }
  p->n_dups = bad[1];
  std::vector<int> cc, cbeg, cend, ccs(p->n_cams + 1);
  const int chunk = cb::RJ_CHUNK;
  for (int c = 0; c < p->n_cams; ++c) {
    ccs[c] = (int)cc.size();
    for (int b = cam_start[c]; b < cam_start[c + 1]; b += chunk) {
      cc.push_back(c);
      cbeg.push_back(b);
      cend.push_back(std::min(b + chunk, cam_start[c + 1]));
    }
  }
  ccs[p->n_cams] = (int)cc.size();
  p->n_chunks = (int)cc.size();
  CB_TRY(palloc(p, &p->d_chunk_cam, cc.size()));
  CB_TRY(palloc(p, &p->d_chunk_begin, cc.size()));
  CB_TRY(palloc(p, &p->d_chunk_end, cc.size()));
  if (!cc.empty()) {
    CB_CUDA(cudaMemcpyAsync(p->d_chunk_cam, cc.data(), sizeof(int) * cc.size(), cudaMemcpyHostToDevice, st));
    CB_CUDA(cudaMemcpyAsync(p->d_chunk_begin, cbeg.data(), sizeof(int) * cc.size(), cudaMemcpyHostToDevice, st));
    CB_CUDA(cudaMemcpyAsync(p->d_chunk_end, cend.data(), sizeof(int) * cc.size(), cudaMemcpyHostToDevice, st));
  }
  CB_CUDA(cudaMemcpyAsync(p->d_cam_chunk_start, ccs.data(), sizeof(int) * ccs.size(), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaStreamSynchronize(st));
  return CB_OK;
}

// ------------------------------------------------------------------------------------------
// the kernels of one evaluation / one LM trial
// ------------------------------------------------------------------------------------------
template <int P>
int run_cam_prep(CbBaProblem* p, const double* xc, double* camtab, cudaStream_t st) {
  CB_LAUNCH(cb::cam_prep_kernel, cdiv(p->n_cams, 64), 64, 0, st, xc, p->d_cam_flags, p->d_cam_const, p->n_cams, P, camtab);
  return CB_OK;
}

// camera-major pass; st_dev == nullptr: stand-alone evaluation at buffer 0
template <int P, int MODE>
void launch_resjac(CbBaProblem* p, const cb::LmState* st_dev, int flip, int loss, double fscale, double* out2,
                   cudaStream_t st) {
  if (p->n_chunks == 0) return;
  CB_LAUNCH((cb::resjac_kernel<P, MODE>), p->n_chunks, cb::RJ_THREADS, 0, st, st_dev, flip, p->d_chunk_cam,
            p->d_chunk_begin, p->d_chunk_end, p->d_cm_xy, p->d_cm_pt, p->d_cm_orig, p->c_camtab(), p->c_xp(), loss,
            fscale, p->d_partial, out2);
}

// COV: the covariance variant (pseudo-inverse root of V into d_covR, rank into d_covRank)
template <int P, bool COV = false>
void launch_pt_pass(CbBaProblem* p, cudaStream_t st) {
#define CB_PT_PASS(LANES, DUPS, SM)                                                                                   \
  CB_LAUNCH((cb::pt_pass_kernel<P, LANES, DUPS, SM, COV>), p->pt_grid, cb::PT_WARPS * 32, p->pt_smem, st, p->d_state, \
            p->d_pt_start, p->d_pm_cam, p->d_pm_xy, p->d_pt_comp, p->n_pts, p->n_cams, p->c_camtab(), p->c_xp(),       \
            p->d_V6, p->d_gp, p->d_Dp2, COV ? p->d_covR : p->d_Linv6, p->d_tvec, p->d_Zt, (size_t)p->LD, p->d_gmax,    \
            COV ? p->d_covRank : nullptr)
#define CB_PT_PASS2(LANES, DUPS) do { if (p->cam_in_smem) CB_PT_PASS(LANES, DUPS, true); else CB_PT_PASS(LANES, DUPS, false); } while (0)
  if (p->pt_lanes == 8) { if (p->n_dups) CB_PT_PASS2(8, true); else CB_PT_PASS2(8, false); }
  else { if (p->n_dups) CB_PT_PASS2(32, true); else CB_PT_PASS2(32, false); }
#undef CB_PT_PASS2
#undef CB_PT_PASS
}

template <int P>
void launch_pt_backsub(CbBaProblem* p, double* dp_out, cudaStream_t st) {
  const int bstride = p->pt_grid + p->n_comp;
#define CB_PT_BACK(LANES, SM)                                                                                         \
  CB_LAUNCH((cb::pt_backsub_kernel<P, LANES, SM>), p->pt_grid, cb::PT_WARPS * 32, p->bs_smem, st, p->d_state,         \
            p->d_pt_start, p->d_pm_cam, p->d_pm_xy, p->d_pt_comp, p->n_pts, p->n_cams, p->nP, p->c_camtab(),           \
            p->m_xp(), p->d_dc, p->d_Linv6, p->d_tvec, p->d_gp, p->d_Dp2, dp_out, p->d_bpart, bstride)
  if (p->pt_lanes == 8) { if (p->cam_in_smem) CB_PT_BACK(8, true); else CB_PT_BACK(8, false); }
  else { if (p->cam_in_smem) CB_PT_BACK(32, true); else CB_PT_BACK(32, false); }
#undef CB_PT_BACK
}

using PcgFn = void (*)(const cb::LmState*, const double*, const double*, const double*, int, int, int, double, int,
                       double*, double*);
// mode 1: slab streamed from L2, 2: slab in registers with cl columns per lane
PcgFn pcg_fn(int mode, int P, int cl) {
  if (mode == 2) {
    if (P == 6)
      return cl == 2 ? cb::pcg_cluster_kernel<2, 6, 2> : cl == 6 ? cb::pcg_cluster_kernel<2, 6, 6>
           : cl == 12 ? cb::pcg_cluster_kernel<2, 6, 12> : cb::pcg_cluster_kernel<2, 6, 18>;
    return cl == 2 ? cb::pcg_cluster_kernel<2, 9, 2> : cl == 6 ? cb::pcg_cluster_kernel<2, 9, 6>
         : cl == 12 ? cb::pcg_cluster_kernel<2, 9, 12> : cb::pcg_cluster_kernel<2, 9, 18>;
  }
  return P == 6 ? cb::pcg_cluster_kernel<1, 6, 1> : cb::pcg_cluster_kernel<1, 9, 1>;
}

int launch_pcg(CbBaProblem* p, const cb::LmState* st_dev, double tol2, int max_iter, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(p->pcg_cs);
  cfg.blockDim = dim3(cb::PCG_THREADS);
  cfg.dynamicSmemBytes = p->pcg_smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = p->pcg_cs;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  const double* S = p->d_red;
  const double* b = p->d_red + (size_t)p->nP * p->nP;
  auto fn = pcg_fn(p->pcg_mode, p->P, p->pcg_cl);
  CB_CUDA(cudaLaunchKernelEx(&cfg, fn, st_dev, S, b, (const double*)p->d_Minv, p->nP, p->pcg_npa, p->pcg_rows, tol2,
                             max_iter, p->d_dc, p->d_sc));
  g_launches.fetch_add(1);
  return CB_OK;
}

// camera-major pass at buffer (cur ^ flip) + reduction of its partials; mode as trial_reduce_kernel
template <int P>
int camera_pass(CbBaProblem* p, int flip, int mode, cudaStream_t st) {
  const int loss = 0;
  const double fscale = 1.0;  // the kernels take both from the device state
  launch_resjac<P, 0>(p, p->d_state, flip, loss, fscale, nullptr, st);
  if (p->n_c)
    CB_LAUNCH((cb::constraint_eval_kernel<false>), p->n_cblk, cb::CC_THREADS, 0, st, (const cb::LmState*)p->d_state, flip,
              p->ct, p->c_xp(), loss, fscale, p->m_crs(), p->m_cdirw(), (double*)nullptr, p->d_camcost + p->n_cams);
  CB_LAUNCH((cb::trial_reduce_kernel<P>), p->n_cams + 1, 64, 0, st, p->d_state, mode, p->n_cams, p->d_cam_chunk_start,
            p->d_partial, p->m_Upk(), p->m_gc(), p->m_costsum(), p->d_camcost, p->n_cblk, p->d_bpart,
            p->pt_grid + p->n_comp, p->pt_grid + p->n_comp, p->d_red2, p->d_counter, p->d_sc, p->d_log);
  return CB_OK;
}

// damped system at the current point: point pass, Schur product, reduced system (+ all-reduce), head-of-iteration tests
// (the last at the head of small_rig_step_kernel on small rigs, see solve_step).  ev: nullptr, or four events that
// bracket the point pass (0, 1) and the Schur product (2, 3).  cov: the undamped covariance linearisation (point pass with
// the pseudo-inverse root of V, no reduced_prep_kernel), single rank only
template <int P>
int build_system(CbBaProblem* p, const CbBaOptions* opt, cudaStream_t st, const cudaEvent_t* ev = nullptr, bool cov = false) {
  if (ev) CB_CUDA(cudaEventRecord(ev[0], st));
  if (cov) launch_pt_pass<P, true>(p, st);
  else launch_pt_pass<P>(p, st);
  if (ev) CB_CUDA(cudaEventRecord(ev[1], st));
  if (p->n_c)
    CB_LAUNCH((cb::comp_build_kernel<P>), p->n_comp, cb::CC_THREADS, p->comp_build_smem, st, (const cb::LmState*)p->d_state,
              p->ct, p->d_pt_start, p->d_pm_cam, p->d_V6, p->d_gp, p->d_Dp2, p->d_gpt, p->c_crs(), p->c_cdirw(), p->n_cams,
              p->d_compL, p->d_tvec, p->d_Zt, (size_t)p->LD, p->d_gmax);
  if (ev) CB_CUDA(cudaEventRecord(ev[2], st));
  CB_LAUNCH(cb::schur_syrk_kernel, p->n_items, cb::SY_THREADS, sizeof(cb::SyrkSmem), st, (const cb::LmState*)p->d_state,
            p->d_Zt, (size_t)p->LD, p->d_tvec, p->d_items, (const int*)p->d_klist, p->d_part, p->d_tpart);
  if (ev) CB_CUDA(cudaEventRecord(ev[3], st));
  const size_t nfin = (size_t)p->nP * p->nP + p->nP + 1;
  // gradient inf-norm over points: one slot per rank so a SUM all-reduce carries the max
  const int rank = sharded(opt) ? std::min(std::max(opt->rank, 0), p->red_slots - 1) : 0;
  if (opt && opt->peer_group) {
    // finalize + all-reduce over NVLink peer memory in one COOPERATIVE launch (cb_peer.cuh)
    CbPeerGroup* g = (CbPeerGroup*)opt->peer_group;
    int nb = 0;
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, cb::schur_finalize_peer_kernel<P>, cb::PEER_THREADS, 0));
    const int grid = std::max(1, std::min(nb, 2)) * p->num_sms;
    const cb::LmState* sd = p->d_state;
    int nP = p->nP, n_blk = p->n_blk, red_slots = p->red_slots, rk = rank;
    cb::CPtr2 upk = p->c_Upk(), gc = p->c_gc(), cs = p->c_costsum();
    const double* gmax = (const double*)p->d_gmax;
    void* args[] = {&sd, &nP, &n_blk, &p->d_tile_of, &p->d_tile_slot_start, &p->d_tile_slots, &p->d_part, &p->d_tpart,
                    &upk, &gc, &cs, &gmax, &red_slots, &rk, &g->tab, &p->d_red};
    CB_CUDA(cudaLaunchCooperativeKernel((const void*)cb::schur_finalize_peer_kernel<P>, dim3(grid), dim3(cb::PEER_THREADS),
                                        args, 0, st));
    g_launches.fetch_add(1);
  } else {
    CB_LAUNCH((cb::schur_finalize_kernel<P>), cdiv((long long)std::max<size_t>(nfin, p->red_slots), 256), 256, 0, st,
              (const cb::LmState*)p->d_state, p->nP, p->n_blk, p->d_tile_of, p->d_tile_slot_start, p->d_tile_slots,
              p->d_part, p->d_tpart, p->c_Upk(), p->c_gc(), p->c_costsum(), (const double*)p->d_gmax, p->red_slots, rank,
              p->d_red);
    if (sharded(opt)) CB_TRY(do_allreduce(opt, p->d_red, (long long)p->red_len(), st));
  }
  if (!p->direct_solve && !cov)
    CB_LAUNCH((cb::reduced_prep_kernel<P>), 1, 256, 0, st, p->d_state, p->nP, p->n_cams, p->red_slots, p->d_red, p->d_Dc2,
              p->d_active, p->d_Minv, p->d_gmax, p->d_sc);
  return CB_OK;
}

template <int P>
int solve_step(CbBaProblem* p, double* dp_out, cudaStream_t st) {
  const size_t nn = (size_t)p->nP * p->nP;
  if (p->direct_solve) {
    CB_LAUNCH((cb::small_rig_step_kernel<P>), 1, cb::DIRECT_THREADS, p->direct_smem, st, p->d_state, p->nP, p->n_cams,
              p->red_slots, p->d_red, p->d_Dc2, p->d_active, p->d_gmax, p->d_sc, p->m_xc(), p->d_dc, p->d_lo, p->d_hi,
              p->d_cam_flags, p->d_cam_const, p->m_camtab());
  } else {
    CB_TRY(launch_pcg(p, p->d_state, 0.0, 0, st));  // tolerance and iteration cap come from the device state
    CB_LAUNCH(cb::cam_step_kernel, 1, 256, 0, st, (const cb::LmState*)p->d_state, p->nP, p->n_cams, p->P, p->m_xc(), p->d_dc,
              p->d_lo, p->d_hi, p->d_red + nn + p->nP, p->d_Dc2, p->d_active, p->d_cam_flags, p->d_cam_const, p->m_camtab(),
              p->d_sc);
  }
  launch_pt_backsub<P>(p, dp_out, st);
  if (p->n_c)
    CB_LAUNCH(cb::comp_backsub_kernel, p->n_comp, cb::CC_THREADS, p->comp_back_smem, st, (const cb::LmState*)p->d_state,
              p->ct, p->nP, p->d_Zt, (size_t)p->LD, p->d_dc, p->d_compL, p->d_tvec, p->d_gpt, p->d_Dp2, p->m_xp(), dp_out,
              p->d_bpart, p->pt_grid + p->n_comp, p->pt_grid);
  return CB_OK;
}

// one whole LM trial: the same launches every time, all decisions on the device
template <int P>
int enqueue_trial(CbBaProblem* p, const CbBaOptions* opt, cudaStream_t st, const cudaEvent_t* ev = nullptr) {
  CB_TRY(build_system<P>(p, opt, st, ev));
  CB_TRY(solve_step<P>(p, nullptr, st));
  const bool multi = sharded(opt);
  CB_TRY(camera_pass<P>(p, 1, multi ? 2 : 1, st));
  if (multi) {
    cb::PeerTable none = {};
    if (opt->peer_group) {
      CB_LAUNCH(cb::lm_decide_kernel, 1, 32, 0, st, p->d_state, (const double*)p->d_sc, p->d_red2, p->d_log,
                ((CbPeerGroup*)opt->peer_group)->tab, 1);
    } else {
      CB_TRY(do_allreduce(opt, p->d_red2, 4, st));
      CB_LAUNCH(cb::lm_decide_kernel, 1, 32, 0, st, p->d_state, (const double*)p->d_sc, p->d_red2, p->d_log, none, 0);
    }
  }
  return CB_OK;
}

int upload_x(CbBaProblem* p, const double* x, cudaStream_t st) {
  stream_copy(p->h_x, x, sizeof(double) * p->n_params);
  CB_CUDA(cudaMemcpyAsync(p->d_x, p->h_x, sizeof(double) * p->n_params, cudaMemcpyHostToDevice, st));
  const int n = std::max(p->n_cams * p->P, p->n_pts);
  CB_LAUNCH(cb::unpack_x_kernel, cdiv(std::max(n, 1), 256), 256, 0, st, p->d_x, p->d_cam_xoff, p->d_cam_flags,
            p->d_cam_const, p->n_cams, p->P, p->n_pts, p->ncp, p->d_xc[0], p->d_xp4[0]);
  return CB_OK;
}

int download_x(CbBaProblem* p, int cur, double* x, cudaStream_t st) {
  const int n = std::max(p->n_cams * p->P, p->n_pts);
  CB_LAUNCH(cb::pack_x_kernel, cdiv(std::max(n, 1), 256), 256, 0, st, p->d_x, p->d_cam_xoff, p->d_cam_flags, p->n_cams,
            p->P, p->n_pts, p->ncp, p->d_xc[cur], p->d_xp4[cur]);
  CB_CUDA(cudaMemcpyAsync(p->h_x, p->d_x, sizeof(double) * p->n_params, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  std::memcpy(x, p->h_x, sizeof(double) * p->n_params);
  return CB_OK;
}

int set_bounds(CbBaProblem* p, bool use_bounds, cudaStream_t st) {
  std::vector<double> lo((size_t)p->nP, -1e300), hi((size_t)p->nP, 1e300);
  if (use_bounds && p->P == 9) {
    for (int c = 0; c < p->n_cams; ++c)
      if (p->h_iflags[c] & CB_CAM_FREE_INTRINSICS) {
        lo[c * 9 + 6] = 0.5; hi[c * 9 + 6] = 2.0;
        lo[c * 9 + 7] = -1.0; hi[c * 9 + 7] = 1.0;
        lo[c * 9 + 8] = -2.0; hi[c * 9 + 8] = 2.0;
      }
  }
  CB_CUDA(cudaMemcpyAsync(p->d_lo, lo.data(), sizeof(double) * p->nP, cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemcpyAsync(p->d_hi, hi.data(), sizeof(double) * p->nP, cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaStreamSynchronize(st));
  return CB_OK;
}

// fresh device state for a solve (or a diagnostic evaluation) starting at buffer 0
int init_state(CbBaProblem* p, const CbBaOptions* opt, double lam, long long max_nfev, cudaStream_t st) {
  cb::LmState& h = p->h_state[3];
  std::memset(&h, 0, sizeof(h));
  h.lam = lam; h.nu = 2.0;
  h.ftol = opt->ftol; h.xtol = opt->xtol; h.gtol = opt->gtol;
  h.nfev = 1; h.njev = 1; h.nit = 0; h.max_nfev = max_nfev;
  h.new_lin = 1;
  h.log_cap = p->log_cap;
  h.loss = opt->loss;
  h.fscale = opt->f_scale > 0 ? opt->f_scale : 1.0;
  const double tol = opt->pcg_tol > 0 ? opt->pcg_tol : 1e-6;
  h.pcg_tol2 = tol * tol;
  h.pcg_max_iter = opt->pcg_max_iter > 0 ? opt->pcg_max_iter : 4 * p->nP;
  if (opt->peer_group) {
    CbPeerGroup* g = (CbPeerGroup*)opt->peer_group;
    h.epoch_big = g->epoch_big; h.epoch_small = g->epoch_small;
  }
  CB_CUDA(cudaMemcpyAsync(p->d_state, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemsetAsync(p->d_gmax, 0, 2 * sizeof(unsigned long long), st));
  CB_CUDA(cudaMemsetAsync(p->d_counter, 0, 4 * sizeof(unsigned int), st));
  CB_CUDA(cudaMemsetAsync(p->d_sc, 0, sizeof(double) * cb::SC_COUNT, st));
  CB_CUDA(cudaMemsetAsync(p->d_Dc2, 0, sizeof(double) * p->nP, st));
  CB_CUDA(cudaMemsetAsync(p->d_Dp2, 0, sizeof(double) * 3 * (size_t)std::max(p->n_pts, 1), st));
  return CB_OK;
}

// Capture one LM trial into g.  loop = false: the trial is the whole graph, launched once per trial.  loop = true: the
// trial is the body of a WHILE conditional node (CUDA 12.4+) whose last kernel sets the loop condition from
// LmState::done, so the whole solve is ONE graph launch and ONE host synchronisation, and no predicated-off trial is
// ever queued.
template <int P>
int ensure_graph(CbBaProblem* p, const CbBaOptions* opt, bool loop) {
  TrialGraph& g = loop ? p->loop_graph : p->trial_graph;
  const TrialGraph::Key key{opt->nccl_comm, opt->peer_group, opt->rank, opt->world_size};
  if (g.key == key && (g.valid || g.failed)) return g.valid ? CB_OK : CB_E_UNSUPPORTED;
  destroy_graph(g);
  g.key = key;
  g.failed = false;
  auto fail = [&](const char* what) {
    g_last_error = std::string(loop ? "device-loop graph: " : "trial graph: ") + what + ": " +
                   cudaGetErrorString(cudaGetLastError());
    destroy_graph(g);
    g.failed = true;
    return CB_E_UNSUPPORTED;
  };
  if (!p->cap_stream && cudaStreamCreateWithFlags(&p->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
    return fail("cudaStreamCreateWithFlags");
  cudaGraphConditionalHandle h = {};
  cudaError_t e;
  if (loop) {
    if (cudaGraphCreate(&g.graph, 0) != cudaSuccess) return fail("cudaGraphCreate");
    if (cudaGraphConditionalHandleCreate(&h, g.graph, 1, cudaGraphCondAssignDefault) != cudaSuccess)
      return fail("cudaGraphConditionalHandleCreate");
    cudaGraphNodeParams np = {};
    np.type = cudaGraphNodeTypeConditional;
    np.conditional.handle = h;
    np.conditional.type = cudaGraphCondTypeWhile;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    if (cudaGraphAddNode(&node, g.graph, nullptr, 0, &np) != cudaSuccess) return fail("cudaGraphAddNode(conditional)");
    e = cudaStreamBeginCaptureToGraph(p->cap_stream, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                      cudaStreamCaptureModeThreadLocal);
  } else {
    e = cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal);
  }
  if (e != cudaSuccess) return fail("begin capture");
  const long long l0 = g_launches.load();
  int rc = enqueue_trial<P>(p, opt, p->cap_stream);
  if (loop && rc == CB_OK) CB_LAUNCH(cb::lm_loop_cond_kernel, 1, 1, 0, p->cap_stream, (const cb::LmState*)p->d_state, h);
  g.n_kernels = (int)(g_launches.load() - l0);
  g_launches.store(l0);  // capture launches nothing
  e = loop ? cudaStreamEndCapture(p->cap_stream, nullptr) : cudaStreamEndCapture(p->cap_stream, &g.graph);
  if (rc != CB_OK || e != cudaSuccess) return fail("capture of the trial");
  if (cudaGraphInstantiate(&g.exec, g.graph, 0) != cudaSuccess) return fail("cudaGraphInstantiate");
  g.valid = true;
  return CB_OK;
}

// ------------------------------------------------------------------------------------------
// Levenberg-Marquardt driver: the loop itself runs on the device (cb_lm.cuh); the host only keeps the GPU fed one
// trial ahead and looks at the state of trial t-1 while trial t executes.
// ------------------------------------------------------------------------------------------
template <int P>
int lm_solve(CbBaProblem* p, const CbBaOptions* opt, double* x_inout, CbBaResult* res, cudaStream_t st) {
  NvtxRange nvtx_solve("cb_ba_solve");
  const long long max_nfev = opt->max_nfev > 0 ? opt->max_nfev : 100ll * p->n_params;
  const bool verbose = opt->verbose >= 2 && opt->rank == 0;
  const long long launches0 = g_launches.load();
  std::memset(res, 0, sizeof(*res));

  // The trials are replayed from CUDA graphs: one GPU -> device loop (ONE graph launch per solve: a WHILE node around the
  // trial); sharded over NCCL or peer memory -> one graph per trial (the host keeps one trial ahead).  Capture +
  // instantiation cost less than the launch gaps and host round trips of even one 3-iteration solve.  Direct launches:
  // a host callback carries the all-reduce (cannot be captured), or opt->time_kernels (CUDA events recorded during a
  // capture cannot be read back).  A graph that cannot be built falls back: device loop -> per-trial graph -> direct.
  const bool direct = opt->allreduce != nullptr || opt->time_kernels;
  bool use_loop = !direct && !sharded(opt);
  if (use_loop && ensure_graph<P>(p, opt, true) != CB_OK) { cudaGetLastError(); use_loop = false; }
  bool use_graph = !direct && !use_loop;
  if (use_graph && ensure_graph<P>(p, opt, false) != CB_OK) { cudaGetLastError(); use_graph = false; }

  CB_TRY(set_bounds(p, opt->use_bounds != 0, st));
  CB_TRY(init_state(p, opt, opt->lambda0 > 0 ? opt->lambda0 : 1e-4, max_nfev, st));
  CB_TRY(upload_x(p, x_inout, st));
  CB_CUDA(cudaEventRecord(p->ev0, st));
  CB_TRY(run_cam_prep<P>(p, p->d_xc[0], p->d_camtab[0], st));
  CB_TRY(camera_pass<P>(p, 0, 0, st));

  double pp_ms_total = 0.0;
  long long pp_launches = 0, trials = 0;
  double sy_ms_total = 0.0;
  long long sy_launches = 0;
  auto read_pp = [&](long long t) {  // direct launches: the event brackets of trial t
    float ms = 0.f;
    const cudaEvent_t* ev = p->ev_pp[t & 1];
    if (cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) { pp_ms_total += ms; ++pp_launches; }
    else cudaGetLastError();
    if (cudaEventElapsedTime(&ms, ev[2], ev[3]) == cudaSuccess) { sy_ms_total += ms; ++sy_launches; }
    else cudaGetLastError();
  };
  bool done = false;
  long long t = 0;
  int rc = CB_OK;
  if (use_loop) {
    // the whole LM loop is one graph launch; the state comes back once
    cudaError_t e = cudaGraphLaunch(p->loop_graph.exec, st);
    if (e != cudaSuccess) {
      // nothing of the loop ran: remember that this configuration cannot be launched and run the trials directly
      cudaGetLastError();
      p->loop_graph.failed = true;
      p->loop_graph.valid = false;
      use_loop = false;
    } else {
      cudaMemcpyAsync(&p->h_state[1], p->d_state, sizeof(cb::LmState), cudaMemcpyDeviceToHost, st);
      t = 2;  // final state in slot (t - 1) & 1
      done = true;
    }
  }
  while (!done) {
    if (use_graph) {
      cudaError_t e = cudaGraphLaunch(p->trial_graph.exec, st);
      if (e != cudaSuccess) { g_last_error = std::string("cudaGraphLaunch: ") + cudaGetErrorString(e); rc = CB_E_CUDA; break; }
      g_launches.fetch_add(p->trial_graph.n_kernels);
    } else {
      NvtxRange nvtx_trial("lm_trial (direct launches)");
      rc = enqueue_trial<P>(p, opt, st, p->ev_pp[t & 1]);
      if (rc != CB_OK) break;
    }
    cudaMemcpyAsync(&p->h_state[t & 1], p->d_state, sizeof(cb::LmState), cudaMemcpyDeviceToHost, st);
    cudaEventRecord(p->ev_state[t & 1], st);
    ++trials;
    if (t >= 1) {
      // trial t is queued; now look at the outcome of trial t-1
      cudaError_t e = cudaEventSynchronize(p->ev_state[(t - 1) & 1]);
      if (e != cudaSuccess) { g_last_error = std::string("LM trial: ") + cudaGetErrorString(e); rc = CB_E_CUDA; break; }
      if (!use_graph) read_pp(t - 1);
      if (p->h_state[(t - 1) & 1].done) done = true;
    }
    ++t;
  }
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == CB_OK && e != cudaSuccess) { g_last_error = std::string("LM solve: ") + cudaGetErrorString(e); rc = CB_E_CUDA; }
  if (rc != CB_OK) { if (p->peer) p->peer->poisoned = true; return rc; }
  const cb::LmState fin = p->h_state[(t - 1) & 1];   // trial t-1 ran predicated-off or finished: final either way
  if (p->peer) {
    int peer_err = 0;
    CB_CUDA(cudaMemcpy(&peer_err, p->peer->tab.err, sizeof(int), cudaMemcpyDeviceToHost));
    p->peer->epoch_big = fin.epoch_big;
    p->peer->epoch_small = fin.epoch_small;
    if (peer_err) {
      p->peer->poisoned = true;
      g_last_error = "peer all-reduce timed out waiting for another rank";
      return CB_E_CALLBACK;
    }
  }
  if (fin.err == cb::LM_ERR_NONFINITE_X0) {  // scipy: ValueError("Residuals are not finite in the initial point.")
    g_last_error = "Residuals are not finite in the initial point.";
    return CB_E_INVALID;
  }
  if (verbose) {
    const int nl = std::min(fin.n_log, p->log_cap);
    std::vector<cb::LmLogRow> rows((size_t)std::max(nl, 1));
    if (nl) CB_CUDA(cudaMemcpy(rows.data(), p->d_log, sizeof(cb::LmLogRow) * nl, cudaMemcpyDeviceToHost));
    std::fprintf(stderr, "%5s %5s %22s %22s %9s %10s %10s %10s %5s\n", "nit", "nfev", "cost", "cost_new", "ratio", "lambda",
                 "|step|", "|g|inf", "pcg");
    for (int i = 0; i < nl; ++i)
      std::fprintf(stderr, "%5lld %5lld %22.15e %22.15e %+9.3f %10.2e %10.2e %10.2e %5d\n", (long long)rows[i].nit,
                   (long long)rows[i].nfev, rows[i].cost, rows[i].cost_new, rows[i].ratio, rows[i].lam, rows[i].step,
                   rows[i].gnorm, (int)rows[i].pcg);
  }
  CB_CUDA(cudaEventRecord(p->ev1, st));
  CB_TRY(download_x(p, fin.cur, x_inout, st));
  float ms = 0.f;
  CB_CUDA(cudaEventElapsedTime(&ms, p->ev0, p->ev1));
  res->status = fin.status;
  res->nfev = fin.nfev;
  res->njev = fin.njev;
  res->nit = fin.nit;
  res->cost = fin.cost;
  res->initial_cost = fin.initial_cost;
  res->optimality = fin.gnorm;
  res->lambda_final = fin.lam;
  res->pcg_iterations = fin.pcg_total;
  res->kernel_launches = g_launches.load() - launches0;
  res->solve_ms = ms;
  res->rj_ms = pp_ms_total;
  res->rj_launches = pp_launches;
  res->syrk_ms = sy_ms_total;
  res->syrk_launches = sy_launches;
  if (use_loop) {
    trials = fin.nfev - 1 + ((fin.status == 1 || fin.err) ? 1 : 0);
    g_launches.fetch_add((long long)p->loop_graph.n_kernels * trials);
    res->kernel_launches = g_launches.load() - launches0;
  }
  res->trials_queued = trials;
  res->used_graph = use_loop ? 2 : use_graph ? 1 : 0;
  if (fin.err == cb::LM_ERR_STUCK_NONFINITE)
    g_last_error = "every trial step is non-finite with the damping at its cap; stopped with status 0";
  if (opt->verbose >= 1 && opt->rank == 0)
    std::fprintf(stderr,
                 "[caliscope_b200] status %d nfev %lld njev %lld nit %lld cost %.15e -> %.15e |g| %.2e  %.3f ms (%lld trials queued, %s)\n",
                 fin.status, (long long)fin.nfev, (long long)fin.njev, (long long)fin.nit, fin.initial_cost, fin.cost,
                 fin.gnorm, ms, trials, use_loop ? "device loop" : use_graph ? "graph" : "direct");
  return CB_OK;
}

int choose_pcg_config(CbBaProblem* p) {
  const int nP = p->nP, P = p->P;
  int max_optin = 0;
  cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device);
  const size_t budget = (size_t)std::max(max_optin, 48 * 1024);
  const size_t minv = (((size_t)(nP / P) * P * P + 7) & ~(size_t)7);
  const int nw = cb::PCG_THREADS / 32;
  auto try_config = [&](int mode, int cs, int cl) -> bool {
    const int rows = (nP + cs - 1) / cs;
    const int npa = std::max((nP + 7) & ~7, mode == 2 ? cl * 32 : 0);
    const size_t smem = (9 * (size_t)npa + 2 * nw + 2 * 16 * nw + minv) * sizeof(double);
    if (smem > budget) return false;
    if (mode == 2 && rows > 3 * nw) return false;
    const void* fn = (const void*)pcg_fn(mode, P, cl);
    cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs);
    cfg.blockDim = dim3(cb::PCG_THREADS);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int ncl = 0;
    if (cudaOccupancyMaxActiveClusters(&ncl, fn, &cfg) != cudaSuccess || ncl < 1) {
      cudaGetLastError();
      return false;
    }
    p->pcg_cs = cs; p->pcg_rows = rows; p->pcg_mode = mode; p->pcg_cl = cl; p->pcg_npa = npa; p->pcg_smem = smem;
    return true;
  };
  // (0) small rigs: prep, direct LDL^T and camera step in one CTA (small_rig_step_kernel) when it fits
  p->direct_solve = false;
  if (nP <= cb::DIRECT_MAX_N) {
    const size_t smem = ((size_t)(nP + 1) * (nP | 1) + nP) * sizeof(double);
    const void* fn = P == 6 ? (const void*)cb::small_rig_step_kernel<6> : (const void*)cb::small_rig_step_kernel<9>;
    if (smem <= budget && cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess) {
      p->direct_solve = true;
      p->direct_smem = smem;
    } else {
      cudaGetLastError();
    }
  }
  // (1) slab in registers: 3 rows x (32 cl) columns per warp; up to 384 reduced parameters in one portable cluster (<= 8
  //     CTAs), up to 576 (64 cameras with free intrinsics) in a 12-CTA cluster (non-portable size, allowed up to 16)
  if (nP <= 576) {
    const int cl = nP <= 64 ? 2 : nP <= 192 ? 6 : nP <= 384 ? 12 : 18;
    const int cs = (nP + 3 * nw - 1) / (3 * nw);
    if (cs <= 16 && try_config(2, cs, cl)) return CB_OK;
  }
  // (2) larger systems, or a register-mode cluster the device refuses: slab streamed from L2
  if (try_config(1, 8, 1)) return CB_OK;
  g_last_error = "no feasible PCG cluster configuration for n_camera_params = " + std::to_string(nP);
  return CB_E_UNSUPPORTED;
}

}  // namespace

// ==========================================================================================
// C ABI
// ==========================================================================================
extern "C" {

int cb_ba_abi_version(void) { return CB_BA_ABI_VERSION; }

const char* cb_ba_error_string(int code) {
  switch (code) {
    case CB_OK: return "ok";
    case CB_E_INVALID: return "invalid argument";
    case CB_E_CUDA: return "CUDA runtime error";
    case CB_E_NO_DEVICE: return "no CUDA device";
    case CB_E_UNSUPPORTED: return "unsupported configuration";
    case CB_E_CALLBACK: return "all-reduce callback failed";
    case CB_E_NOMEM: return "out of device memory";
    default: return "unknown error";
  }
}

const char* cb_ba_last_error(void) { return g_last_error.c_str(); }

void cb_ba_default_options(CbBaOptions* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->ftol = 1e-8; o->xtol = 1e-8; o->gtol = 1e-8;
  o->max_nfev = 0;
  o->loss = CB_LOSS_LINEAR;
  o->f_scale = 1.0;
  o->verbose = 0;
  o->use_bounds = 1;
  o->lambda0 = 1e-4;
  o->pcg_tol = 1e-6;
  o->pcg_max_iter = 0;
  o->allreduce = nullptr;
  o->allreduce_user = nullptr;
  o->nccl_comm = nullptr;
  o->peer_group = nullptr;
  o->rank = 0;
  o->world_size = 1;
  o->time_kernels = 0;
}

int64_t cb_ba_launch_count(void) { return (int64_t)g_launches.load(); }

int cb_peer_create(int rank, int world_size, int device, int64_t capacity_doubles, CbPeerGroup** out,
                   char handle_out[64]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  if (!out || !handle_out || rank < 0 || rank >= world_size || world_size > cb::PEER_MAXW || capacity_doubles <= 0) {
    g_last_error = "cb_peer_create: bad argument (world_size <= 16)";
    return CB_E_INVALID;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); g_last_error = "no CUDA device"; return CB_E_NO_DEVICE; }
  CB_CUDA(cudaSetDevice(device));
  auto* g = new CbPeerGroup();
  g->rank = rank; g->world = world_size; g->device = device;
  g->cap = ((size_t)capacity_doubles + 31) / 32 * 32;
  g->bytes = cb::PEER_OFF_DATA + 2 * g->cap * sizeof(double);
  cudaError_t e = cudaMalloc(&g->base, g->bytes);  // a whole allocation of its own: IPC handles name allocations
  if (e != cudaSuccess) { g_last_error = std::string("cudaMalloc: ") + cudaGetErrorString(e); delete g; return CB_E_NOMEM; }
  e = cudaMemset(g->base, 0, g->bytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, g->base);
  if (e != cudaSuccess) {
    g_last_error = std::string("cb_peer_create: ") + cudaGetErrorString(e);
    cudaFree(g->base);
    delete g;
    return CB_E_CUDA;
  }
  std::memcpy(handle_out, &h, 64);
  *out = g;
  return CB_OK;
}

int cb_peer_connect(CbPeerGroup* g, const char* handles) {
  if (!g || !handles) { g_last_error = "cb_peer_connect: null argument"; return CB_E_INVALID; }
  if (g->connected) return CB_OK;
  CB_CUDA(cudaSetDevice(g->device));
  for (int r = 0; r < g->world; ++r) {
    if (r == g->rank) { g->peer_base[r] = g->base; continue; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handles + 64 * (size_t)r, 64);
    cudaError_t e = cudaIpcOpenMemHandle(&g->peer_base[r], h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      g_last_error = "cudaIpcOpenMemHandle(rank " + std::to_string(r) + "): " + cudaGetErrorString(e);
      cudaGetLastError();
      for (int q = 0; q < r; ++q)
        if (q != g->rank && g->peer_base[q]) { cudaIpcCloseMemHandle(g->peer_base[q]); g->peer_base[q] = nullptr; }
      return CB_E_UNSUPPORTED;
    }
  }
  cb::PeerTable& t = g->tab;
  t.rank = g->rank; t.world = g->world;
  for (int r = 0; r < g->world; ++r) {
    char* b = (char*)g->peer_base[r];
    t.data[r][0] = (const double*)(b + cb::PEER_OFF_DATA);
    t.data[r][1] = (const double*)(b + cb::PEER_OFF_DATA) + g->cap;
    t.flags_big_of[r] = (unsigned long long*)(b + cb::PEER_OFF_FLAGS_BIG);
    t.flags_small_of[r] = (unsigned long long*)(b + cb::PEER_OFF_FLAGS_SMALL);
    t.small_of[r] = (double*)(b + cb::PEER_OFF_SMALL);
  }
  char* mine = (char*)g->base;
  t.my_data[0] = (double*)(mine + cb::PEER_OFF_DATA);
  t.my_data[1] = (double*)(mine + cb::PEER_OFF_DATA) + g->cap;
  t.my_flags_big = (unsigned long long*)(mine + cb::PEER_OFF_FLAGS_BIG);
  t.my_flags_small = (unsigned long long*)(mine + cb::PEER_OFF_FLAGS_SMALL);
  t.my_small = (double*)(mine + cb::PEER_OFF_SMALL);
  t.done = (unsigned int*)(mine + cb::PEER_OFF_DONE);
  t.err = (int*)(mine + cb::PEER_OFF_ERR);
  g->connected = true;
  return CB_OK;
}

int cb_peer_destroy(CbPeerGroup* g) {
  if (!g) return CB_OK;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  if (g->connected)
    for (int r = 0; r < g->world; ++r)
      if (r != g->rank && g->peer_base[r]) cudaIpcCloseMemHandle(g->peer_base[r]);
  if (g->base) cudaFree(g->base);
  cudaGetLastError();
  delete g;
  return CB_OK;
}

int cb_nccl_unique_id(char id_out[128]) {
  NcclApi& a = nccl();
  if (!a.ok) { g_last_error = a.err; return CB_E_UNSUPPORTED; }
  UidBlob u;
  const int rc = a.GetUniqueId(&u);
  if (rc != 0) { g_last_error = "ncclGetUniqueId failed"; return CB_E_CALLBACK; }
  std::memcpy(id_out, u.internal, 128);
  return CB_OK;
}

int cb_nccl_comm_create(const char id[128], int rank, int world_size, int device, void** comm_out) {
  if (!id || !comm_out || rank < 0 || rank >= world_size) { g_last_error = "cb_nccl_comm_create: bad argument"; return CB_E_INVALID; }
  NcclApi& a = nccl();
  if (!a.ok) { g_last_error = a.err; return CB_E_UNSUPPORTED; }
  CB_CUDA(cudaSetDevice(device));
  UidBlob u;
  std::memcpy(u.internal, id, 128);
  void* comm = nullptr;
  const int rc = a.CommInitRank(&comm, world_size, u, rank);
  if (rc != 0) {
    g_last_error = std::string("ncclCommInitRank: ") + (a.GetErrorString ? a.GetErrorString(rc) : "error");
    return CB_E_CALLBACK;
  }
  *comm_out = comm;
  return CB_OK;
}

int cb_nccl_comm_destroy(void* comm) {
  if (!comm) return CB_OK;
  NcclApi& a = nccl();
  if (!a.ok) return CB_E_UNSUPPORTED;
  return a.CommDestroy(comm) == 0 ? CB_OK : CB_E_CALLBACK;
}

int cb_ba_problem_destroy(CbBaProblem* p) {
  if (!p) return CB_OK;
  cudaSetDevice(p->device);
  destroy_graph(p->trial_graph);
  destroy_graph(p->loop_graph);
  if (p->cap_stream) cudaStreamDestroy(p->cap_stream);
  for (void* a : p->allocs) cached_free(a);
  cached_free_host(p->h_state);
  cached_free_host(p->h_x);
  for (cudaEvent_t e : {p->ev0, p->ev1, p->ev2, p->ev3, p->ev_state[0], p->ev_state[1], p->ev_pp[0][0], p->ev_pp[0][1],
                        p->ev_pp[0][2], p->ev_pp[0][3], p->ev_pp[1][0], p->ev_pp[1][1], p->ev_pp[1][2], p->ev_pp[1][3]})
    if (e) cudaEventDestroy(e);
  delete p;
  return CB_OK;
}

int64_t cb_ba_problem_n_params(const CbBaProblem* p) { return p ? p->n_params : -1; }
int cb_ba_cam_stride(const CbBaProblem* p) { return p ? p->P : -1; }
double cb_ba_problem_stat(const CbBaProblem* p, int what) {
  if (!p) return -1.0;
  switch (what) {
    case 0: return p->schur_sparse ? 1.0 : 0.0;
    case 1: return p->schur_flop_issued;
    case 2: return p->direct_solve ? 1.0 : 0.0;
    case 3: return (double)p->n_items;
    case 4: case 5: case 6: return (double)p->cov_ms[what - 4];
    case 7: return (double)p->pt_lanes;
    case 8: return p->n_dups ? 1.0 : 0.0;
    case 9: return (double)p->cam_in_smem;
    case 10: return p->direct_solve ? 0.0 : (double)p->pcg_mode;
    case 11: return (double)p->pcg_cs;
    case 12: return p->pcg_mode == 2 ? (double)p->pcg_cl : 0.0;
    case 13: return p->order_identity ? 0.0 : 1.0;
    default: return -1.0;
  }
}

// Schur work items.  Dense visibility: off-diagonal tiles and pairs of diagonal tiles, each split over k so that the
// grid is one CTA per SM with equal DMMA work (a diagonal pair costs 45/36 of a full tile per chunk).  Sparse
// visibility (fewer than 70 % of the (point, tile pair) incidences exist): every tile pair gets the compacted list of
// the k rows of the points BOTH its column tiles see, and CTAs are dealt in proportion to list length.
static int build_schur_items(CbBaProblem* p, cudaStream_t st) {
  const int nb = p->n_blk;
  std::vector<int> tof((size_t)nb * nb, -1);
  int nt = 0;
  for (int I = 0; I < nb; ++I)
    for (int J = I; J < nb; ++J) tof[(size_t)I * nb + J] = nt++;
  const double w_pair = 1.55;  // measured cost of a diagonal-pair CTA per k chunk relative to an off-diagonal one
  const double w_single = 0.75;

  // per-pair row lists, if sparse: offset of each tile pair's list in d_klist (-1: no common point) and its point count
  std::vector<long long> pair_koff, pair_cnt;
  bool sparse = false;
  int want_sparse = -1;
  if (const char* ev = std::getenv("CB_SY_SPARSE")) want_sparse = std::atoi(ev);
  if (nb >= 2 && nb <= 64 && p->n_pts > 0 && want_sparse != 0) {
    unsigned long long* d_mask;
    CB_TRY(dalloc(&d_mask, (size_t)p->n_pts));
    ScopedFree sf; sf.dev.push_back(d_mask);
    CB_LAUNCH(cb::pt_tile_mask_kernel, cdiv(p->n_pts, 256), 256, 0, st, p->d_pt_start, p->d_pm_cam, p->n_pts, p->P, d_mask);
    if (p->n_comp)  // rebuilt by cb_ba_problem_set_constraints: the lists must see the components' fill-in
      CB_LAUNCH(cb::comp_tile_mask_kernel, cdiv(p->n_comp, 256), 256, 0, st, p->ct.comp_pt_start, p->ct.comp_pts, p->n_comp,
                d_mask);
    // incidence counts per tile pair (dense rigs stop here: no mask download, no host pass over the points)
    unsigned long long* d_cnt;
    CB_TRY(dalloc(&d_cnt, (size_t)nt));
    sf.dev.push_back(d_cnt);
    CB_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long) * nt, st));
    CB_LAUNCH(cb::tile_pair_count_kernel, cdiv(p->n_pts, 256), 256, sizeof(unsigned) * nt, st, d_mask, p->n_pts, nb, d_cnt);
    std::vector<unsigned long long> cnt_u((size_t)nt);
    CB_CUDA(cudaMemcpyAsync(cnt_u.data(), d_cnt, sizeof(unsigned long long) * nt, cudaMemcpyDeviceToHost, st));
    CB_CUDA(cudaStreamSynchronize(st));
    std::vector<long long> cnt(cnt_u.begin(), cnt_u.end());
    double listed = 0.0, dense = 0.0;
    for (int I = 0; I < nb; ++I)
      for (int J = I; J < nb; ++J) {
        const double w = (I == J) ? w_single : 1.0;
        listed += w * (double)cnt[tof[(size_t)I * nb + J]];
        dense += w * (double)p->n_pts;
      }
    p->schur_rows_dense = 3.0 * dense; p->schur_rows_listed = 3.0 * listed;
    sparse = want_sparse == 1 || listed < 0.7 * dense;
    if (sparse) {
      // the row lists are built on the device (inc_count .. klist_expand in cb_kernels.cuh); the host only lays out where each
      // tile pair's list starts
      const int zero_row = p->K_pad;  // rows K_pad .. K_pad + SY_KC - 1 of Zt / tvec are never written
      std::vector<long long> pair_start((size_t)nt + 1, 0), koff_h((size_t)nt, -1);
      long long klen = 0;
      for (int t = 0; t < nt; ++t) {
        pair_start[(size_t)t + 1] = pair_start[(size_t)t] + cnt[(size_t)t];
        if (cnt[(size_t)t] == 0) continue;
        koff_h[(size_t)t] = klen;
        klen += cdiv(3 * cnt[(size_t)t], (long long)cb::SY_KC) * cb::SY_KC;
      }
      const long long n_inc = pair_start[(size_t)nt];
      if (klen > 0x7fffffffLL || n_inc > 0x7fffffffLL) { g_last_error = "Schur row lists exceed 2^31 entries"; return CB_E_UNSUPPORTED; }
      pair_koff.assign(koff_h.begin(), koff_h.end());
      pair_cnt.assign(cnt.begin(), cnt.end());
      int *d_ninc = nullptr, *d_incoff = nullptr;
      unsigned long long *d_keys = nullptr, *d_keys_s = nullptr;
      long long *d_pair_start = nullptr, *d_koff = nullptr;
      CB_TRY(dalloc(&d_ninc, (size_t)p->n_pts + 1)); sf.dev.push_back(d_ninc);
      CB_TRY(dalloc(&d_incoff, (size_t)p->n_pts + 1)); sf.dev.push_back(d_incoff);
      CB_TRY(dalloc(&d_keys, (size_t)n_inc)); sf.dev.push_back(d_keys);
      CB_TRY(dalloc(&d_keys_s, (size_t)n_inc)); sf.dev.push_back(d_keys_s);
      CB_TRY(dalloc(&d_pair_start, (size_t)nt + 1)); sf.dev.push_back(d_pair_start);
      CB_TRY(dalloc(&d_koff, (size_t)nt)); sf.dev.push_back(d_koff);
      CB_TRY(palloc(p, &p->d_klist, (size_t)klen));
      CB_CUDA(cudaMemsetAsync(d_ninc + p->n_pts, 0, sizeof(int), st));
      CB_LAUNCH(cb::inc_count_kernel, cdiv(p->n_pts, 256), 256, 0, st, (const unsigned long long*)d_mask, p->n_pts, d_ninc);
      size_t tb_a = 0, tb_b = 0;
      const int key_bits = bits_for((unsigned long long)nt * (unsigned long long)p->n_pts);
      cub::DeviceScan::ExclusiveSum(nullptr, tb_a, d_ninc, d_incoff, p->n_pts + 1, st);
      cub::DeviceRadixSort::SortKeys(nullptr, tb_b, d_keys, d_keys_s, (int)n_inc, 0, key_bits, st);
      void* d_tmp = nullptr;
      size_t tbm = std::max(tb_a, tb_b);
      CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tbm, 16))); sf.dev.push_back(d_tmp);
      CB_CUDA(cub::DeviceScan::ExclusiveSum(d_tmp, tbm, d_ninc, d_incoff, p->n_pts + 1, st));
      CB_LAUNCH(cb::inc_emit_kernel, cdiv(p->n_pts, 256), 256, 0, st, (const unsigned long long*)d_mask, (const int*)d_incoff,
                p->n_pts, nb, d_keys);
      tbm = std::max(tb_a, tb_b);
      CB_CUDA(cub::DeviceRadixSort::SortKeys(d_tmp, tbm, d_keys, d_keys_s, (int)n_inc, 0, key_bits, st));
      g_launches.fetch_add(5);
      CB_CUDA(cudaMemcpyAsync(d_pair_start, pair_start.data(), sizeof(long long) * pair_start.size(), cudaMemcpyHostToDevice, st));
      CB_CUDA(cudaMemcpyAsync(d_koff, koff_h.data(), sizeof(long long) * koff_h.size(), cudaMemcpyHostToDevice, st));
      CB_LAUNCH(cb::fill_int_kernel, cdiv(klen, 256), 256, 0, st, p->d_klist, klen, zero_row);
      CB_LAUNCH(cb::klist_expand_kernel, cdiv(n_inc, 256), 256, 0, st, (const unsigned long long*)d_keys_s, n_inc, p->n_pts,
                (const long long*)d_pair_start, (const long long*)d_koff, p->d_klist);
      CB_CUDA(cudaStreamSynchronize(st));  // pair_start / koff_h are host temporaries of this scope
    }
  }
  p->schur_sparse = sparse;

  struct Group { int kind, I, J; double w; int chunks; int koff; };
  std::vector<Group> groups;
  if (!sparse) {
    for (int I = 0; I < nb; ++I)
      for (int J = I + 1; J < nb; ++J) groups.push_back({0, I, J, 1.0, p->k_chunks, -1});
    for (int I = 0; I < nb; I += 2) {
      if (I + 1 < nb) groups.push_back({1, I, I + 1, w_pair, p->k_chunks, -1});
      else groups.push_back({1, I, -1, w_single, p->k_chunks, -1});
    }
  } else {
    for (int I = 0; I < nb; ++I)
      for (int J = I; J < nb; ++J) {
        const int t = tof[(size_t)I * nb + J];
        if (pair_cnt[(size_t)t] == 0) continue;
        const int koff = (int)pair_koff[(size_t)t];
        const int chunks = (int)cdiv(3 * pair_cnt[(size_t)t], (long long)cb::SY_KC);
        if (I == J) groups.push_back({1, I, -1, w_single, chunks, koff});
        else groups.push_back({0, I, J, 1.0, chunks, koff});
      }
  }
  double W = 0.0;
  for (auto& g : groups) W += g.w * g.chunks;
  // flops the product issues per launch: an off-diagonal tile is 96 x 96 outputs per k row, a diagonal tile its 10
  // upper-triangular 24 x 24 blocks
  p->schur_flop_issued = 0.0;
  for (auto& g : groups) {
    const double cols2 = g.kind == 0 ? 96.0 * 96.0 : (g.J >= 0 ? 2.0 : 1.0) * 10.0 * 24.0 * 24.0;
    p->schur_flop_issued += 2.0 * cols2 * (double)g.chunks * cb::SY_KC;
  }
  std::vector<cb::SyItem> items;
  std::vector<std::vector<int>> slots_of(nt);
  int slot = 0;
  // CTAs per group: proportional share rounded down, then the SMs left over go one by one to the group whose CTAs carry
  // the most work (6 tiles at P = 9: 18 groups, floor alone leaves up to 17 SMs idle)
  // A CTA gets at least SY_MIN_CHUNKS k-chunks: every split-K slot is a 96x96 partial tile the finalize kernel reads back
  // serially, and on a small rig (8 cameras x 2000 points: 188 chunks in ONE tile) one slot per SM, 1-2 chunks each made the
  // finalize kernel cost several times the product it reduces.
  constexpr int SY_MIN_CHUNKS = 8;
  auto cap_of = [&](const Group& g) { return std::max(1, g.chunks / SY_MIN_CHUNKS); };
  std::vector<int> n_of(groups.size(), 1);
  {
    int used = 0;
    for (size_t gi = 0; gi < groups.size(); ++gi) {
      const Group& g = groups[gi];
      int n = (int)std::floor(p->num_sms * (g.w * g.chunks) / std::max(W, 1.0));
      n_of[gi] = std::max(1, std::min(n, cap_of(g)));
      used += n_of[gi];
    }
    while (used < p->num_sms) {
      int best = -1;
      double load = 0.0;
      for (size_t gi = 0; gi < groups.size(); ++gi) {
        if (n_of[gi] >= cap_of(groups[gi])) continue;
        const double l = groups[gi].w * groups[gi].chunks / n_of[gi];
        if (l > load) { load = l; best = (int)gi; }
      }
      if (best < 0) break;
      ++n_of[(size_t)best];
      ++used;
    }
  }
  for (size_t gi = 0; gi < groups.size(); ++gi) {
    const Group& g = groups[gi];
    const int n = n_of[gi];
    for (int s2 = 0; s2 < n; ++s2) {
      cb::SyItem it;
      it.kind = g.kind; it.I = g.I; it.J = g.J; it.koff = g.koff;
      it.c0 = (int)(((long long)g.chunks * s2) / n);
      it.c1 = (int)(((long long)g.chunks * (s2 + 1)) / n);
      it.slotA = slot++;
      it.slotB = -1;
      if (g.kind == 0) {
        slots_of[tof[(size_t)g.I * nb + g.J]].push_back(it.slotA);
      } else {
        slots_of[tof[(size_t)g.I * nb + g.I]].push_back(it.slotA);
        if (g.J >= 0) {
          it.slotB = slot++;
          slots_of[tof[(size_t)g.J * nb + g.J]].push_back(it.slotB);
        }
      }
      items.push_back(it);
    }
  }
  p->n_items = (int)items.size();
  p->n_slots = std::max(slot, 1);
  std::vector<int> sstart(nt + 1, 0), sflat;
  for (int t = 0; t < nt; ++t) {
    sstart[t] = (int)sflat.size();
    sflat.insert(sflat.end(), slots_of[t].begin(), slots_of[t].end());
  }
  sstart[nt] = (int)sflat.size();
  CB_TRY(palloc(p, &p->d_items, std::max<size_t>(items.size(), 1)));
  CB_TRY(palloc(p, &p->d_tile_of, tof.size()));
  CB_TRY(palloc(p, &p->d_tile_slot_start, sstart.size()));
  CB_TRY(palloc(p, &p->d_tile_slots, std::max<size_t>(sflat.size(), 1)));
  if (!items.empty())
    CB_CUDA(cudaMemcpyAsync(p->d_items, items.data(), sizeof(cb::SyItem) * items.size(), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemcpyAsync(p->d_tile_of, tof.data(), sizeof(int) * tof.size(), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemcpyAsync(p->d_tile_slot_start, sstart.data(), sizeof(int) * sstart.size(), cudaMemcpyHostToDevice, st));
  if (!sflat.empty())
    CB_CUDA(cudaMemcpyAsync(p->d_tile_slots, sflat.data(), sizeof(int) * sflat.size(), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaStreamSynchronize(st));  // the host vectors above go out of scope
  return CB_OK;
}

// Constraint components arrive after problem creation and fill in the Zt rows of their points (comp_tile_mask_kernel).
// Row lists built without them would leave those rows out of the tile pairs they reach, so the work items are built
// again: the dense / list decision, the lists and the CTA split.  The partial-tile buffers follow the new slot count.
static int rebuild_schur_items(CbBaProblem* p, cudaStream_t st) {
  CB_CUDA(cudaStreamSynchronize(st));
  for (void** a : {(void**)&p->d_klist, (void**)&p->d_items, (void**)&p->d_tile_of, (void**)&p->d_tile_slot_start,
                   (void**)&p->d_tile_slots, (void**)&p->d_part, (void**)&p->d_tpart}) {
    if (!*a) continue;
    p->allocs.erase(std::remove(p->allocs.begin(), p->allocs.end(), *a), p->allocs.end());
    cached_free(*a);
    *a = nullptr;
  }
  CB_TRY(build_schur_items(p, st));
  CB_TRY(palloc(p, &p->d_part, (size_t)p->n_slots * cb::SY_TILE * cb::SY_TILE));
  CB_TRY(palloc(p, &p->d_tpart, (size_t)p->n_slots * cb::SY_TILE));
  CB_CUDA(cudaMemsetAsync(p->d_tpart, 0, sizeof(double) * (size_t)p->n_slots * cb::SY_TILE, st));
  CB_CUDA(cudaMemsetAsync(p->d_part, 0, sizeof(double) * (size_t)p->n_slots * cb::SY_TILE * cb::SY_TILE, st));
  CB_CUDA(cudaStreamSynchronize(st));
  return CB_OK;
}

static int problem_create_impl(const CbBaProblemDesc* d, int device, cudaStream_t st, CbBaProblem* p) {
  NvtxRange nvtx_create("cb_ba_problem_create (upload + index build)");
  // CB_PROFILE_CREATE=1: host wall-clock of the stages of problem creation on stderr (diagnostic)
  const bool prof = std::getenv("CB_PROFILE_CREATE") != nullptr;
  auto t_prev = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!prof) return;
    cudaStreamSynchronize(st);
    const auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[create] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
    t_prev = now;
  };
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    g_last_error = "no CUDA device visible";
    return CB_E_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { g_last_error = "device index out of range"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(device));
  p->device = device;
  cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, device);
  p->n_cams = d->n_cams; p->n_pts = d->n_pts; p->n_obs = (int)d->n_obs;
  p->h_cam_off.assign(p->n_cams + 1, 0);
  bool any_free = false;
  for (int c = 0; c < p->n_cams; ++c) {
    const int f = d->cam_flags[c];
    if ((f & CB_CAM_FREE_INTRINSICS) && (f & CB_CAM_FISHEYE)) {
      g_last_error = "fisheye cameras cannot have free intrinsics (bundle_parameterization.py:76-94)";
      return CB_E_INVALID;
    }
    any_free = any_free || (f & CB_CAM_FREE_INTRINSICS);
    p->h_cam_off[c + 1] = p->h_cam_off[c] + ((f & CB_CAM_FREE_INTRINSICS) ? 9 : 6);
    if (!(d->cam_const[c * 9] != 0.0)) { g_last_error = "fx_initial must be non-zero"; return CB_E_INVALID; }
  }
  p->P = any_free ? 9 : 6;
  p->nP = p->n_cams * p->P;
  p->ncp = p->h_cam_off[p->n_cams];
  p->n_params = p->ncp + 3 * p->n_pts;
  p->n_blk = cdiv(p->nP, cb::SY_TILE);
  p->LD = p->n_blk * cb::SY_TILE;
  p->n_tiles = p->n_blk * (p->n_blk + 1) / 2;
  p->K_pad = cdiv(3ll * std::max(p->n_pts, 1), cb::SY_KC) * cb::SY_KC;
  p->k_chunks = p->K_pad / cb::SY_KC;
  p->n_split = std::max(1, std::min(p->k_chunks, p->num_sms / std::max(p->n_tiles, 1)));
  // point kernels: 8 lanes per point when points have few observations (typical rigs: 2-6 cameras per point), a whole
  // warp otherwise; persistent grid (2 CTAs per SM) so the camera table is staged into shared memory once per CTA
  // (8 lanes keep every lane busy for any group size that is not tiny against 8; a whole warp per point only pays when
  // points carry hundreds of rows -- static objects seen in every frame)
  p->pt_lanes = ((double)p->n_obs / std::max(p->n_pts, 1) <= 96.0) ? 8 : 32;
  {
    const int per_block = cb::PT_WARPS * (32 / p->pt_lanes);
    p->pt_grid = std::max(1, std::min(cdiv(std::max(p->n_pts, 1), per_block), 2 * p->num_sms));
    const size_t tab_bytes = sizeof(double) * cb::CT_SMEM * (size_t)p->n_cams;
    p->cam_in_smem = tab_bytes <= 64 * 1024 ? 1 : 0;
    p->pt_smem = p->cam_in_smem ? tab_bytes : 0;
    p->bs_smem = sizeof(double) * (((size_t)p->nP + 3) & ~(size_t)3) + (p->cam_in_smem ? tab_bytes : 0);
  }

  const int n = p->n_obs;
  // tables
  CB_TRY(palloc(p, &p->d_cam_xoff, p->n_cams)); CB_TRY(palloc(p, &p->d_cam_slot, p->n_cams));
  CB_TRY(palloc(p, &p->d_cam_flags, p->n_cams));
  CB_TRY(palloc(p, &p->d_cam_const, (size_t)p->n_cams * 9));
  CB_TRY(palloc(p, &p->d_cm_xy, n)); CB_TRY(palloc(p, &p->d_cm_pt, n)); CB_TRY(palloc(p, &p->d_pm_xy, n));
  CB_TRY(palloc(p, &p->d_cm_orig, n)); CB_TRY(palloc(p, &p->d_cam_start, p->n_cams + 1));
  CB_TRY(palloc(p, &p->d_cam_chunk_start, p->n_cams + 1));
  CB_TRY(palloc(p, &p->d_pt_start, p->n_pts + 1)); CB_TRY(palloc(p, &p->d_pm_orig, n));
  CB_TRY(palloc(p, &p->d_pm_cam, n));
  CB_TRY(palloc(p, &p->d_pm_pt, n));
  // observation list: host -> device if needed
  const int *d_cam = d->obs_cam, *d_pt = d->obs_pt;
  const double* d_xy = d->obs_xy;
  int *t_cam = nullptr, *t_pt = nullptr;
  double* t_xy = nullptr;
  ScopedFree stage;  // pinned staging blocks: released when this function returns (it synchronises before)
  XyUpload xy_up;    // declared after `stage`: its destructor joins the staging thread before the pinned blocks go
  if (!d->obs_on_device) {
    CB_TRY(dalloc(&t_cam, n)); CB_TRY(dalloc(&t_pt, n)); CB_TRY(dalloc(&t_xy, 2 * (size_t)n));
    p->allocs.push_back(t_cam); p->allocs.push_back(t_pt); p->allocs.push_back(t_xy);  // kept: the cull path compacts them
    // the pixel upload (two thirds of the bytes) starts first and runs beside everything up to the last index kernels
    CB_CUDA(cudaEventCreateWithFlags(&xy_up.ev, cudaEventDisableTiming));
    {
      cudaStream_t side = side_stream();
      const double* src = d->obs_xy;
      const size_t bytes = sizeof(double) * 2 * (size_t)n;
      const int dev = p->device;
      xy_up.started = true;
      WorkerPool::get().submit([&xy_up, t_xy, src, bytes, side, dev] {
        cudaSetDevice(dev);
        xy_up.rc = staged_h2d(t_xy, src, bytes, side, xy_up.pinned, 8);
        if (xy_up.rc == CB_OK && cudaEventRecord(xy_up.ev, side) != cudaSuccess) xy_up.rc = CB_E_CUDA;
        if (xy_up.rc != CB_OK) xy_up.err = "staged upload of obs_xy failed";
        xy_up.finished.store(1, std::memory_order_release);
      });
    }
    if (d->obs_cam_bits == 16) {
      short* t16 = nullptr;
      CB_TRY(dalloc(&t16, n));
      stage.dev.push_back(t16);
      CB_TRY(staged_h2d(t16, d->obs_cam, sizeof(short) * (size_t)n, st, stage));
      CB_LAUNCH(cb::widen_i16_kernel, cdiv(n, 256), 256, 0, st, (const short*)t16, n, t_cam);
    } else {
      CB_TRY(staged_h2d(t_cam, d->obs_cam, sizeof(int) * (size_t)n, st, stage));
    }
    CB_TRY(staged_h2d(t_pt, d->obs_pt, sizeof(int) * (size_t)n, st, stage));
    d_cam = t_cam; d_pt = t_pt; d_xy = t_xy;
  } else if (d->obs_cam_bits == 16) {
    CB_TRY(dalloc(&t_cam, n));
    p->allocs.push_back(t_cam);
    CB_LAUNCH(cb::widen_i16_kernel, cdiv(n, 256), 256, 0, st, (const short*)d->obs_cam, n, t_cam);
    d_cam = t_cam;
  }
  p->d_obs_cam = d_cam; p->d_obs_pt = d_pt; p->d_obs_xy = d_xy;
  p->h_cam_flags.assign(d->cam_flags, d->cam_flags + p->n_cams);
  p->h_cam_const.assign(d->cam_const, d->cam_const + 9 * (size_t)p->n_cams);
  lap("alloc + staged upload");
  CB_TRY(build_indices(p, d_cam, d_pt, d_xy, d->cam_order, st, xy_up.started ? &xy_up : nullptr));
  // camera tables by internal slot
  {
    std::vector<int> xoff(p->n_cams);
    std::vector<double> iconst((size_t)p->n_cams * 9);
    p->h_iflags.resize(p->n_cams);
    for (int i = 0; i < p->n_cams; ++i) {
      const int c = p->h_perm[i];
      xoff[i] = p->h_cam_off[c];
      p->h_iflags[i] = d->cam_flags[c];
      std::memcpy(&iconst[(size_t)i * 9], d->cam_const + (size_t)c * 9, 9 * sizeof(double));
    }
    CB_CUDA(cudaMemcpyAsync(p->d_cam_xoff, xoff.data(), sizeof(int) * p->n_cams, cudaMemcpyHostToDevice, st));
    CB_CUDA(cudaMemcpyAsync(p->d_cam_flags, p->h_iflags.data(), sizeof(int) * p->n_cams, cudaMemcpyHostToDevice, st));
    CB_CUDA(cudaMemcpyAsync(p->d_cam_const, iconst.data(), sizeof(double) * 9 * p->n_cams, cudaMemcpyHostToDevice, st));
    CB_CUDA(cudaStreamSynchronize(st));
  }

  lap("index build + camera tables");
  CB_TRY(build_schur_items(p, st));
  lap("schur work items");
  std::vector<unsigned char> act((size_t)p->nP, 0);
  for (int c = 0; c < p->n_cams; ++c)
    for (int a = 0; a < ((p->h_iflags[c] & CB_CAM_FREE_INTRINSICS) ? 9 : 6); ++a) act[(size_t)c * p->P + a] = 1;
  CB_TRY(palloc(p, &p->d_active, p->nP));
  CB_CUDA(cudaMemcpyAsync(p->d_active, act.data(), p->nP, cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaStreamSynchronize(st));
  CB_TRY(palloc(p, &p->d_lo, p->nP)); CB_TRY(palloc(p, &p->d_hi, p->nP));

  // work buffers
  const int NACC = (p->P == 6) ? 28 : 55, NU = (p->P == 6) ? 21 : 45;
  const size_t npts = (size_t)std::max(p->n_pts, 1);
  CB_TRY(palloc(p, &p->d_x, (size_t)p->n_params + 1));
  for (int k = 0; k < 2; ++k) {
    CB_TRY(palloc(p, &p->d_xc[k], p->nP)); CB_TRY(palloc(p, &p->d_xp4[k], 4 * npts));
    CB_TRY(palloc(p, &p->d_camtab[k], (size_t)p->n_cams * cb::CT_SIZE));
    CB_TRY(palloc(p, &p->d_Upk[k], (size_t)p->n_cams * NU)); CB_TRY(palloc(p, &p->d_gc[k], p->nP));
    CB_TRY(palloc(p, &p->d_costsum[k], 4));
  }
  CB_TRY(palloc(p, &p->d_partial, (size_t)std::max(p->n_chunks, 1) * NACC));
  CB_TRY(palloc(p, &p->d_camcost, p->n_cams));
  CB_TRY(palloc(p, &p->d_gpt, 3 * npts));
  CB_TRY(palloc(p, &p->d_V6, 6 * npts)); CB_TRY(palloc(p, &p->d_gp, 3 * npts)); CB_TRY(palloc(p, &p->d_Dp2, 3 * npts));
  CB_TRY(palloc(p, &p->d_Dc2, p->nP)); CB_TRY(palloc(p, &p->d_Linv6, 6 * npts));
  // + one chunk of rows that stay zero for good: the padding target of the compacted k-lists
  CB_TRY(palloc(p, &p->d_tvec, (size_t)p->K_pad + cb::SY_KC));
  CB_TRY(palloc(p, &p->d_Zt, ((size_t)p->K_pad + cb::SY_KC) * p->LD));
  CB_TRY(palloc(p, &p->d_part, (size_t)p->n_slots * cb::SY_TILE * cb::SY_TILE));
  CB_TRY(palloc(p, &p->d_tpart, (size_t)p->n_slots * cb::SY_TILE));
  CB_TRY(palloc(p, &p->d_red, p->red_len()));
  CB_TRY(palloc(p, &p->d_Minv, (size_t)p->n_cams * p->P * p->P));
  CB_TRY(palloc(p, &p->d_dc, p->nP)); CB_TRY(palloc(p, &p->d_dp, 3 * npts));
  CB_TRY(palloc(p, &p->d_bpart, 3 * (size_t)p->pt_grid));
  CB_TRY(palloc(p, &p->d_sc, cb::SC_COUNT)); CB_TRY(palloc(p, &p->d_red2, 8));
  CB_TRY(palloc(p, &p->d_gmax, 2));
  CB_TRY(palloc(p, &p->d_counter, 4));
  CB_TRY(palloc(p, &p->d_state, 1));
  CB_TRY(palloc(p, &p->d_log, (size_t)p->log_cap));
  CB_TRY(palloc(p, &p->d_out2, 2 * (size_t)std::max(n, 1)));
  CB_CUDA(cudaMemsetAsync(p->d_Zt, 0, sizeof(double) * ((size_t)p->K_pad + cb::SY_KC) * p->LD, st));
  CB_CUDA(cudaMemsetAsync(p->d_tvec, 0, sizeof(double) * ((size_t)p->K_pad + cb::SY_KC), st));
  CB_CUDA(cudaMemsetAsync(p->d_tpart, 0, sizeof(double) * (size_t)p->n_slots * cb::SY_TILE, st));
  CB_CUDA(cudaMemsetAsync(p->d_part, 0, sizeof(double) * (size_t)p->n_slots * cb::SY_TILE * cb::SY_TILE, st));
  CB_CUDA(cudaMemsetAsync(p->d_red2, 0, sizeof(double) * 8, st));
  CB_CUDA(cudaMemsetAsync(p->d_Linv6, 0, sizeof(double) * 6 * npts, st));
  CB_TRY(cached_malloc_host((void**)&p->h_state, sizeof(cb::LmState) * 4));
  CB_TRY(cached_malloc_host((void**)&p->h_x, sizeof(double) * ((size_t)p->n_params + 1)));
  for (cudaEvent_t* e : {&p->ev0, &p->ev1, &p->ev2, &p->ev3, &p->ev_pp[0][0], &p->ev_pp[0][1], &p->ev_pp[0][2], &p->ev_pp[0][3],
                         &p->ev_pp[1][0], &p->ev_pp[1][1], &p->ev_pp[1][2], &p->ev_pp[1][3]})
    CB_CUDA(cudaEventCreate(e));
  for (cudaEvent_t* e : {&p->ev_state[0], &p->ev_state[1]}) CB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  CB_CUDA(cudaFuncSetAttribute(cb::schur_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)sizeof(cb::SyrkSmem)));
  if (p->pt_smem > 48 * 1024 || p->bs_smem > 48 * 1024) {
    const int a = (int)p->pt_smem, b2 = (int)p->bs_smem;
#define CB_SMEM_ATTR(PP)                                                                                           \
    do {                                                                                                             \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 8, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a);  \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 8, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a);   \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 32, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a); \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 32, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a);  \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 8, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a); \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 8, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a); \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 32, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a); \
      cudaFuncSetAttribute(cb::pt_pass_kernel<PP, 32, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, a); \
      cudaFuncSetAttribute(cb::pt_backsub_kernel<PP, 8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, b2);     \
      cudaFuncSetAttribute(cb::pt_backsub_kernel<PP, 32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, b2);    \
      cudaFuncSetAttribute(cb::pt_backsub_kernel<PP, 8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, b2);    \
      cudaFuncSetAttribute(cb::pt_backsub_kernel<PP, 32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, b2);   \
    } while (0)
    if (p->P == 6) CB_SMEM_ATTR(6); else CB_SMEM_ATTR(9);
#undef CB_SMEM_ATTR
    CB_CUDA(cudaGetLastError());
  }
  lap("work buffers + memsets");
  CB_TRY(choose_pcg_config(p));
  CB_CUDA(cudaStreamSynchronize(st));
  lap("pcg config");
  return CB_OK;
}

int cb_ba_problem_create(const CbBaProblemDesc* d, int device, void* stream, CbBaProblem** out) {
  if (d && d->n_obs == 0) {
    // CaptureVolume._validate_geometry (capture_volume.py:97-98) rejects this before optimize() can run
    g_last_error = "No image observations provided";
    return CB_E_INVALID;
  }
  if (d && d->obs_cam_bits != 0 && d->obs_cam_bits != 16 && d->obs_cam_bits != 32) {
    g_last_error = "obs_cam_bits must be 0, 16 or 32";
    return CB_E_INVALID;
  }
  if (!d || !out || d->n_cams <= 0 || d->n_pts <= 0 || d->n_obs < 0 || d->n_obs > (1ll << 30) || !d->cam_flags ||
      !d->cam_const || (d->n_obs > 0 && (!d->obs_cam || !d->obs_pt || !d->obs_xy))) {
    g_last_error = "cb_ba_problem_create: bad descriptor";
    return CB_E_INVALID;
  }
  *out = nullptr;
  CbBaProblem* p = new CbBaProblem();
  int rc = problem_create_impl(d, device, (cudaStream_t)stream, p);
  if (rc != CB_OK) {
    std::string keep = g_last_error;
    cb_ba_problem_destroy(p);
    g_last_error = keep;
    return rc;
  }
  *out = p;
  return CB_OK;
}

int cb_ba_solve(CbBaProblem* p, const CbBaOptions* opt, double* x_inout, CbBaResult* result, void* stream) {
  if (!p || !opt || !x_inout || !result) { g_last_error = "cb_ba_solve: null argument"; return CB_E_INVALID; }
  if (opt->loss < 0 || opt->loss > CB_LOSS_ARCTAN) { g_last_error = "unknown loss id"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  // with an all-reduce hook the caller shards by constraint component (distributed.shard_points), so every
  // constraint row and every point it touches are local to this rank
  p->peer = nullptr;
  if (opt->peer_group) {
    CbPeerGroup* g = (CbPeerGroup*)opt->peer_group;
    if (!g->connected || g->device != p->device) { g_last_error = "peer group is not connected on this device"; return CB_E_INVALID; }
    if (g->cap < p->red_len()) {
      g_last_error = "peer group capacity " + std::to_string(g->cap) + " doubles < " + std::to_string(p->red_len());
      return CB_E_INVALID;
    }
    if (opt->rank != g->rank || opt->world_size != g->world) { g_last_error = "rank / world_size differ from the peer group's"; return CB_E_INVALID; }
    if (g->poisoned) {
      g_last_error = "peer group is unusable after a failed solve (the ranks' sequence numbers may differ): re-create it";
      return CB_E_INVALID;
    }
    p->peer = g;
  }
  if (sharded(opt) && p->order_auto && !p->order_identity) {
    g_last_error = "sharded solve on a problem whose camera order was chosen from this rank's observations only: pass "
                   "CbBaProblemDesc.cam_order (the same on every rank)";
    return CB_E_INVALID;
  }
  const int rc = p->P == 6 ? lm_solve<6>(p, opt, x_inout, result, st) : lm_solve<9>(p, opt, x_inout, result, st);
  p->peer = nullptr;
  return rc;
}

}  // extern "C"
namespace {
template <int P, int MODE>
int eval_mode(CbBaProblem* p, const double* x, cudaStream_t st) {
  CB_TRY(upload_x(p, x, st));
  CB_TRY(run_cam_prep<P>(p, p->d_xc[0], p->d_camtab[0], st));
  launch_resjac<P, MODE>(p, nullptr, 0, 0, 1.0, p->d_out2, st);
  return CB_OK;
}
}  // namespace
extern "C" {

int cb_ba_residuals(CbBaProblem* p, const double* x, double* r_out, void* stream) {
  if (!p || !x || !r_out) { g_last_error = "cb_ba_residuals: null argument"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  CB_TRY(p->P == 6 ? (eval_mode<6, 2>(p, x, st)) : (eval_mode<9, 2>(p, x, st)));
  CB_CUDA(cudaMemcpyAsync(r_out, p->d_out2, sizeof(double) * 2 * (size_t)p->n_obs, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  return CB_OK;
}

int cb_ba_reproj_errors_px(CbBaProblem* p, const double* x, double* err_xy, void* stream) {
  if (!p || !x || !err_xy) { g_last_error = "cb_ba_reproj_errors_px: null argument"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  CB_TRY(p->P == 6 ? (eval_mode<6, 3>(p, x, st)) : (eval_mode<9, 3>(p, x, st)));
  CB_CUDA(cudaMemcpyAsync(err_xy, p->d_out2, sizeof(double) * 2 * (size_t)p->n_obs, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  return CB_OK;
}

int cb_ba_jacobian_blocks(CbBaProblem* p, const double* x, double* Jc, double* Jp, void* stream) {
  if (!p || !x || !Jc || !Jp) { g_last_error = "cb_ba_jacobian_blocks: null argument"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int n = p->n_obs;
  CB_TRY(upload_x(p, x, st));
  double *dJc, *dJp;
  CB_TRY(dalloc(&dJc, 18 * (size_t)std::max(n, 1)));
  CB_TRY(dalloc(&dJp, 6 * (size_t)std::max(n, 1)));
  if (p->P == 6) {
    CB_TRY(run_cam_prep<6>(p, p->d_xc[0], p->d_camtab[0], st));
    if (n) CB_LAUNCH((cb::jac_blocks_kernel<6>), cdiv(n, 128), 128, 0, st, p->d_obs_cam, (const int*)p->d_cam_slot, p->d_obs_pt,
                     reinterpret_cast<const double2*>(p->d_obs_xy), n, (const double*)p->d_camtab[0], (const double*)p->d_xp4[0], dJc, dJp);
  } else {
    CB_TRY(run_cam_prep<9>(p, p->d_xc[0], p->d_camtab[0], st));
    if (n) CB_LAUNCH((cb::jac_blocks_kernel<9>), cdiv(n, 128), 128, 0, st, p->d_obs_cam, (const int*)p->d_cam_slot, p->d_obs_pt,
                     reinterpret_cast<const double2*>(p->d_obs_xy), n, (const double*)p->d_camtab[0], (const double*)p->d_xp4[0], dJc, dJp);
  }
  cudaError_t e1 = cudaMemcpyAsync(Jc, dJc, sizeof(double) * 18 * (size_t)n, cudaMemcpyDeviceToHost, st);
  cudaError_t e2 = cudaMemcpyAsync(Jp, dJp, sizeof(double) * 6 * (size_t)n, cudaMemcpyDeviceToHost, st);
  cudaError_t e3 = cudaStreamSynchronize(st);
  cached_free(dJc); cached_free(dJp);
  CB_CUDA(e1); CB_CUDA(e2); CB_CUDA(e3);
  return CB_OK;
}

}  // extern "C"
namespace {
template <int P>
int normal_eq_impl(CbBaProblem* p, const double* x, double lam, int loss, double fs, double* cost, double* U,
                          double* gc, double* V, double* gp, double* S, double* b, double* dc, double* dp,
                          cudaStream_t st) {
  using RT = cb::RowT<P>;
  CbBaOptions opt;
  cb_ba_default_options(&opt);
  opt.loss = loss; opt.f_scale = fs;
  opt.ftol = opt.xtol = opt.gtol = 0.0;
  CB_TRY(set_bounds(p, false, st));
  CB_TRY(init_state(p, &opt, lam, 1ll << 40, st));
  CB_TRY(upload_x(p, x, st));
  CB_TRY(run_cam_prep<P>(p, p->d_xc[0], p->d_camtab[0], st));
  CB_TRY(camera_pass<P>(p, 0, 0, st));
  CB_TRY(build_system<P>(p, &opt, st));
  CB_TRY(solve_step<P>(p, p->d_dp, st));
  // after solve_step: small rigs apply the damping in small_rig_step_kernel; nothing in solve_step writes d_red otherwise
  const size_t nn = (size_t)p->nP * p->nP;
  std::vector<double> hS(nn + 3 * (size_t)p->nP + 1);
  CB_CUDA(cudaMemcpyAsync(hS.data(), p->d_red, sizeof(double) * hS.size(), cudaMemcpyDeviceToHost, st));
  std::vector<double> hU((size_t)p->n_cams * RT::NU), hV(6 * (size_t)std::max(p->n_pts, 1));
  CB_CUDA(cudaMemcpyAsync(hU.data(), p->d_Upk[0], sizeof(double) * hU.size(), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(hV.data(), p->d_V6, sizeof(double) * hV.size(), cudaMemcpyDeviceToHost, st));
  if (gc) CB_CUDA(cudaMemcpyAsync(gc, p->d_gc[0], sizeof(double) * p->nP, cudaMemcpyDeviceToHost, st));
  if (gp) CB_CUDA(cudaMemcpyAsync(gp, p->d_gp, sizeof(double) * 3 * (size_t)p->n_pts, cudaMemcpyDeviceToHost, st));
  if (dc) CB_CUDA(cudaMemcpyAsync(dc, p->d_dc, sizeof(double) * p->nP, cudaMemcpyDeviceToHost, st));
  if (dp) CB_CUDA(cudaMemcpyAsync(dp, p->d_dp, sizeof(double) * 3 * (size_t)p->n_pts, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  if (cost) *cost = hS[nn + 3 * (size_t)p->nP];
  // reduced system back in the caller's camera order
  const int nP = p->nP;
  if (S)
    for (int i = 0; i < nP; ++i)
      for (int j = 0; j < nP; ++j)
        S[((size_t)p->h_perm[i / P] * P + i % P) * nP + (size_t)p->h_perm[j / P] * P + j % P] = hS[(size_t)i * nP + j];
  if (b)
    for (int i = 0; i < nP; ++i) b[(size_t)p->h_perm[i / P] * P + i % P] = hS[nn + i];
  if (!p->order_identity) {
    std::vector<double> tmp(nP);
    for (double* v : {gc, dc})
      if (v) {
        std::memcpy(tmp.data(), v, sizeof(double) * nP);
        for (int i = 0; i < nP; ++i) v[(size_t)p->h_perm[i / P] * P + i % P] = tmp[i];
      }
  }
  if (U)
    for (int i = 0; i < p->n_cams; ++i) {
      const int c = p->h_perm[i];
      int u = 0;
      for (int a = 0; a < P; ++a)
        for (int bb = a; bb < P; ++bb, ++u) {
          U[((size_t)c * P + a) * P + bb] = hU[(size_t)i * RT::NU + u];
          U[((size_t)c * P + bb) * P + a] = hU[(size_t)i * RT::NU + u];
        }
    }
  if (V)
    for (int j = 0; j < p->n_pts; ++j) {
      const double* v = &hV[6 * (size_t)j];
      double* o = V + 9 * (size_t)j;
      o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[1]; o[4] = v[3]; o[5] = v[4]; o[6] = v[2]; o[7] = v[4]; o[8] = v[5];
    }
  return CB_OK;
}
}  // namespace
extern "C" {

int cb_ba_normal_equations(CbBaProblem* p, const double* x, double lambda, int32_t loss, double f_scale, double* cost,
                           double* U, double* gc, double* V, double* gp, double* S, double* b, double* dc, double* dp,
                           void* stream) {
  if (!p || !x) { g_last_error = "cb_ba_normal_equations: null argument"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  return p->P == 6 ? normal_eq_impl<6>(p, x, lambda, loss, f_scale, cost, U, gc, V, gp, S, b, dc, dp, st)
                   : normal_eq_impl<9>(p, x, lambda, loss, f_scale, cost, U, gc, V, gp, S, b, dc, dp, st);
}

}  // extern "C"
namespace {
template <int P>
int covariance_impl(CbBaProblem* p, const double* x, int loss, double fs, int n_fixed, const int32_t* fixed, double vf,
                    double* cam_cov, double* pt_cov, double* s2_out, int64_t* dof_out, int32_t* pt_rank, cudaStream_t st) {
  const int nP = p->nP, nc = p->n_cams, npts = std::max(p->n_pts, 1);
  const size_t nn = (size_t)nP * nP;
  // free mask (internal slot order): the camera's own slots, camera observed, not fixed
  std::vector<int> cs(nc + 1);
  CB_CUDA(cudaMemcpyAsync(cs.data(), p->d_cam_start, sizeof(int) * (nc + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  std::vector<char> is_fixed((size_t)p->ncp, 0);
  for (int i = 0; i < n_fixed; ++i) is_fixed[fixed[i]] = 1;
  std::vector<unsigned char> fr((size_t)nP, 0);
  std::vector<int> xidx((size_t)nP, -1);  // caller x index of each internal slot (-1: padding)
  long long n_masked = 0, n_fix = 0;
  for (int i = 0; i < nc; ++i) {
    const int c = p->h_perm[i], w = p->h_cam_off[c + 1] - p->h_cam_off[c];
    const bool observed = cs[i + 1] > cs[i];
    for (int a = 0; a < w; ++a) {
      const int xi = p->h_cam_off[c] + a;
      xidx[(size_t)i * P + a] = xi;
      if (!observed) ++n_masked;
      else if (is_fixed[xi]) ++n_fix;
      else fr[(size_t)i * P + a] = 1;
    }
  }
  if (!p->d_covA) {
    const int n = (int)cdiv(nP, cb::CV_B) * cb::CV_B;
    CB_TRY(palloc(p, &p->d_covA, (size_t)n * n));
    CB_TRY(palloc(p, &p->d_covC, (size_t)n * cb::CV_B));
    CB_TRY(palloc(p, &p->d_covD, (size_t)cb::CV_B * cb::CV_B));
    CB_TRY(palloc(p, &p->d_covDiag, (size_t)n));
    CB_TRY(palloc(p, &p->d_covS, nn));
    CB_TRY(palloc(p, &p->d_covR, 9 * (size_t)npts));
    CB_TRY(palloc(p, &p->d_covPt, 9 * (size_t)npts));
    CB_TRY(palloc(p, &p->d_covRank, (size_t)npts));
    CB_TRY(palloc(p, &p->d_covFail, 2));
    CB_TRY(palloc(p, &p->d_covFree, (size_t)nP));
    p->cov_n = n;
  }
  const int n = p->cov_n;
  CbBaOptions opt;
  cb_ba_default_options(&opt);
  opt.loss = loss; opt.f_scale = fs;
  opt.ftol = opt.xtol = opt.gtol = 0.0;
  CB_CUDA(cudaEventRecord(p->ev0, st));
  CB_TRY(init_state(p, &opt, 0.0, 1ll << 40, st));
  CB_CUDA(cudaMemsetAsync(p->d_covRank, 0, sizeof(int) * npts, st));
  const int big[2] = {INT32_MAX, INT32_MAX};
  CB_CUDA(cudaMemcpyAsync(p->d_covFail, big, sizeof(big), cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemcpyAsync(p->d_covFree, fr.data(), nP, cudaMemcpyHostToDevice, st));
  CB_TRY(upload_x(p, x, st));
  CB_TRY(run_cam_prep<P>(p, p->d_xc[0], p->d_camtab[0], st));
  CB_TRY(camera_pass<P>(p, 0, 0, st));
  CB_TRY(build_system<P>(p, &opt, st, nullptr, true));
  if (p->n_c) CB_LAUNCH(cb::comp_failed_kernel, cdiv(p->n_comp, 128), 128, 0, st, p->ct, (const double*)p->d_compL, p->d_covFail + 1);
  CB_CUDA(cudaEventRecord(p->ev1, st));
  // dense inverse of the gauge-fixed reduced system
  CB_LAUNCH(cb::cov_prep_kernel, cdiv((long long)n * n, 256), 256, 0, st, (const double*)p->d_red, nP,
            (const unsigned char*)p->d_covFree, n, p->d_covA, p->d_covDiag);
  for (int kb = 0; kb < n; kb += cb::CV_B) {
    CB_LAUNCH(cb::cov_sweep_pivot_kernel, 1, cb::CV_B * cb::CV_B, 0, st, (const double*)p->d_covA, n, kb,
              (const double*)p->d_covDiag, CB_COV_PIVOT_RTOL, p->d_covD, p->d_covC, p->d_covFail);
    CB_LAUNCH(cb::cov_sweep_update_kernel, dim3(n / cb::CV_B, n / cb::CV_B), cb::CV_B * cb::CV_B, 0, st, p->d_covA, n, kb,
              (const double*)p->d_covD, (const double*)p->d_covC);
  }
  CB_LAUNCH(cb::cov_finish_kernel, cdiv((long long)nn, 256), 256, 0, st, (const double*)p->d_covA, n, nP,
            (const unsigned char*)p->d_covFree, p->d_covS);
  CB_CUDA(cudaEventRecord(p->ev2, st));
  double cost = 0.0;
  int fail[2];
  std::vector<int> rank((size_t)npts);
  CB_CUDA(cudaMemcpyAsync(&cost, p->d_red + nn + 3 * (size_t)nP, sizeof(double), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(fail, p->d_covFail, sizeof(fail), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(rank.data(), p->d_covRank, sizeof(int) * npts, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  char msg[256];
  if (fail[1] != INT32_MAX) {
    std::snprintf(msg, sizeof msg, "cb_ba_covariance: constraint component %d is not positive definite at lambda = 0", fail[1]);
    g_last_error = msg;
    return CB_E_INVALID;
  }
  if (fail[0] != INT32_MAX) {
    const int slot = fail[0] / P, a = fail[0] % P;
    std::snprintf(msg, sizeof msg,
                  "cb_ba_covariance: the gauge-fixed reduced camera system is singular: the pivot of camera %d parameter %d "
                  "(x index %d) collapsed below %.0e of its diagonal; fix more parameters (see default_gauge)",
                  p->h_perm[slot], a, xidx[fail[0]], CB_COV_PIVOT_RTOL);
    g_last_error = msg;
    return CB_E_INVALID;
  }
  long long null_pts = 0;
  for (int j = 0; j < p->n_pts; ++j)
    if (rank[j] >= 0) null_pts += 3 - rank[j];
  const long long m = 2ll * p->n_obs + p->n_c;
  const long long rk = (long long)p->n_params - n_fix - n_masked - null_pts;
  const long long dof = m - rk;
  const double s2 = vf > 0.0 ? vf : (dof > 0 ? 2.0 * cost / (double)dof : std::nan(""));
  if (s2_out) *s2_out = s2;
  if (dof_out) *dof_out = dof;
  if (pt_rank) std::memcpy(pt_rank, rank.data(), sizeof(int) * p->n_pts);
  if (pt_cov && p->n_pts > 0) {
    CB_LAUNCH((cb::cov_point_kernel<P>), 4 * p->num_sms, 256, 0, st, (const int*)p->d_pt_start, (const int*)p->d_pm_cam,
              p->n_pts, (const double*)p->d_Zt, (size_t)p->LD, (const double*)p->d_covS, nP, (const double*)p->d_covR,
              (const int*)p->d_covRank, s2, p->d_covPt);
  }
  CB_CUDA(cudaEventRecord(p->ev3, st));
  if (pt_cov && p->n_pts > 0)
    CB_CUDA(cudaMemcpyAsync(pt_cov, p->d_covPt, sizeof(double) * 9 * p->n_pts, cudaMemcpyDeviceToHost, st));
  std::vector<double> hS;
  if (cam_cov) {
    hS.resize(nn);
    CB_CUDA(cudaMemcpyAsync(hS.data(), p->d_covS, sizeof(double) * nn, cudaMemcpyDeviceToHost, st));
  }
  CB_CUDA(cudaStreamSynchronize(st));
  CB_CUDA(cudaEventElapsedTime(&p->cov_ms[0], p->ev0, p->ev1));
  CB_CUDA(cudaEventElapsedTime(&p->cov_ms[1], p->ev1, p->ev2));
  CB_CUDA(cudaEventElapsedTime(&p->cov_ms[2], p->ev2, p->ev3));
  if (cam_cov) {
    // caller layout: NaN rows / columns for the cameras without observations, zero for the fixed parameters
    const size_t ncp = (size_t)p->ncp;
    std::vector<double> rowv(ncp);
    for (int i = 0; i < nc; ++i) {
      const bool observed = cs[i + 1] > cs[i];
      const int c = p->h_perm[i];
      for (int a = p->h_cam_off[c]; a < p->h_cam_off[c + 1]; ++a) rowv[a] = observed ? 0.0 : std::nan("");
    }
    for (size_t i = 0; i < ncp; ++i)
      for (size_t j = 0; j < ncp; ++j) cam_cov[i * ncp + j] = std::isnan(rowv[i]) ? rowv[i] : rowv[j];
    for (int i = 0; i < nP; ++i) {
      if (!fr[i]) continue;
      for (int j = 0; j < nP; ++j)
        if (fr[j]) cam_cov[(size_t)xidx[i] * ncp + xidx[j]] = s2 * hS[(size_t)i * nP + j];
    }
  }
  return CB_OK;
}
}  // namespace
extern "C" {

int cb_ba_covariance(CbBaProblem* p, const double* x, int32_t loss, double f_scale, int32_t n_fixed, const int32_t* fixed,
                     double variance_factor, double* cam_cov, double* pt_cov, double* s2_out, int64_t* dof_out,
                     int32_t* pt_rank, void* stream) {
  if (!p || !x || (n_fixed > 0 && !fixed) || n_fixed < 0) { g_last_error = "cb_ba_covariance: null argument"; return CB_E_INVALID; }
  if (loss < CB_LOSS_LINEAR || loss > CB_LOSS_ARCTAN) { g_last_error = "cb_ba_covariance: unknown loss"; return CB_E_INVALID; }
  for (int i = 0; i < n_fixed; ++i)
    if (fixed[i] < 0 || fixed[i] >= p->ncp) {
      g_last_error = "cb_ba_covariance: fixed index " + std::to_string(fixed[i]) + " is outside the camera section of x";
      return CB_E_INVALID;
    }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  return p->P == 6 ? covariance_impl<6>(p, x, loss, f_scale, n_fixed, fixed, variance_factor, cam_cov, pt_cov, s2_out, dof_out, pt_rank, st)
                   : covariance_impl<9>(p, x, loss, f_scale, n_fixed, fixed, variance_factor, cam_cov, pt_cov, s2_out, dof_out, pt_rank, st);
}

// Diagnostic: time `reps` launches of the PCG kernel on the system left by the last
// cb_ba_normal_equations call, forcing exactly max_iter iterations (tolerance 0).
int cb_ba_debug_pcg_time(CbBaProblem* p, int max_iter, int reps, double* ms_per_launch, void* stream) {
  if (!p || !ms_per_launch || reps <= 0) { g_last_error = "cb_ba_debug_pcg_time: bad argument"; return CB_E_INVALID; }
  if (p->direct_solve) { g_last_error = "cb_ba_debug_pcg_time: this problem is solved directly, not by PCG"; return CB_E_UNSUPPORTED; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  CB_TRY(launch_pcg(p, nullptr, 0.0, max_iter, st));
  CB_CUDA(cudaEventRecord(p->ev2, st));
  for (int r = 0; r < reps; ++r) CB_TRY(launch_pcg(p, nullptr, 0.0, max_iter, st));
  CB_CUDA(cudaEventRecord(p->ev3, st));
  CB_CUDA(cudaEventSynchronize(p->ev3));
  float ms = 0.f;
  CB_CUDA(cudaEventElapsedTime(&ms, p->ev2, p->ev3));
  *ms_per_launch = ms / reps;
  double t[cb::SC_COUNT];
  CB_CUDA(cudaMemcpy(t, p->d_sc, sizeof(t), cudaMemcpyDeviceToHost));
  std::fprintf(stderr, "[pcg profile] cycles/iteration on CTA 0 thread 0: A(update+precond) %.0f block-barrier %.0f B(matvec) %.0f cluster-barrier %.0f C(dots) %.0f\n",
               t[cb::SC_PCG_T0] / max_iter, t[cb::SC_PCG_T0 + 1] / max_iter, t[cb::SC_PCG_T0 + 2] / max_iter,
               t[cb::SC_PCG_T0 + 3] / max_iter, t[cb::SC_PCG_T0 + 4] / max_iter);
  return CB_OK;
}

}  // extern "C"
namespace {
template <int NT>
__global__ void fp64_dmma_peak_kernel(double* out, int iters, double a0, double b0) {
  double c[NT][2];
#pragma unroll
  for (int i = 0; i < NT; ++i) { c[i][0] = threadIdx.x; c[i][1] = i; }
  double a = a0 + threadIdx.x * 1e-9, b = b0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NT; ++i) cb::dmma884(c[i][0], c[i][1], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NT; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int NT>
__global__ void fp64_dmma16816_peak_kernel(double* out, int iters, double a0, double b0) {
  double c[NT][4], a[8], b[4];
#pragma unroll
  for (int i = 0; i < NT; ++i) { c[i][0] = threadIdx.x; c[i][1] = i; c[i][2] = 0.0; c[i][3] = 1.0; }
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = a0 + threadIdx.x * 1e-9 + i * 1e-12;
#pragma unroll
  for (int j = 0; j < 4; ++j) b[j] = b0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NT; ++i) cb::dmma16816(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NT; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int NACC>
__global__ void fp64_dfma_peak_kernel(double* out, int iters, double a, double b) {
  double acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = fma(acc[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NACC; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
}  // namespace
extern "C" {

int cb_debug_fp64_peak(int device, double* dmma_tflops, double* dfma_tflops) {
  if (!dmma_tflops || !dfma_tflops) { g_last_error = "cb_debug_fp64_peak: null argument"; return CB_E_INVALID; }
  CB_TRY(select_device(device));
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int warps = 8, threads = warps * 32, iters = 20000;
  double* out = nullptr;
  CB_TRY(dalloc(&out, (size_t)sms * threads));
  ScopedFree sf; sf.dev.push_back(out);
  cudaEvent_t e0, e1;
  CB_CUDA(cudaEventCreate(&e0)); CB_CUDA(cudaEventCreate(&e1));
  float ms = 0.f;
  double best_mma = 0.0, best_fma = 0.0;
  for (int rep = 0; rep < 3; ++rep) {
    fp64_dmma_peak_kernel<16><<<sms, threads>>>(out, rep == 0 ? 200 : iters, 1.0000001, 1e-9);
    if (rep == 0) { cudaDeviceSynchronize(); continue; }
    cudaEventRecord(e0);
    fp64_dmma_peak_kernel<16><<<sms, threads>>>(out, iters, 1.0000001, 1e-9);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    best_mma = std::max(best_mma, 2.0 * 256 * 16 * iters * (double)warps * sms / ms * 1e-9);
    // the m16n8k16 shape the off-diagonal Schur tiles issue
    if (rep == 1) fp64_dmma16816_peak_kernel<8><<<sms, threads>>>(out, 200, 1.0000001, 1e-9);
    cudaEventRecord(e0);
    fp64_dmma16816_peak_kernel<8><<<sms, threads>>>(out, iters / 4, 1.0000001, 1e-9);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    best_mma = std::max(best_mma, 2.0 * 2048 * 8 * (iters / 4) * (double)warps * sms / ms * 1e-9);
    cudaEventRecord(e0);
    fp64_dfma_peak_kernel<16><<<sms, threads>>>(out, iters, 1.0000001, 1e-9);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    best_fma = std::max(best_fma, 2.0 * 16 * iters * (double)threads * sms / ms * 1e-9);
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  CB_CUDA(cudaGetLastError());
  *dmma_tflops = best_mma;
  *dfma_tflops = best_fma;
  return CB_OK;
}

int cb_ba_error_order_stats(CbBaProblem* p, const double* x, double q_percent, double* err, double* lo, double* hi,
                            int64_t* count, void* stream) {
  if (!p || !x || !lo || !hi || !count) { g_last_error = "cb_ba_error_order_stats: null argument"; return CB_E_INVALID; }
  if (!(q_percent >= 0.0 && q_percent <= 100.0)) { g_last_error = "q_percent outside [0, 100]"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int n = p->n_obs;
  CB_TRY(p->P == 6 ? (eval_mode<6, 4>(p, x, st)) : (eval_mode<9, 4>(p, x, st)));
  double *d_lo, *d_hi;
  long long* d_cnt;
  CB_TRY(dalloc(&d_lo, p->n_cams)); CB_TRY(dalloc(&d_hi, p->n_cams)); CB_TRY(dalloc(&d_cnt, p->n_cams));
  CB_LAUNCH(cb::order_stats_kernel, p->n_cams, 256, 0, st, p->d_out2, p->d_cam_start, q_percent / 100.0, d_lo, d_hi,
            d_cnt);
  if (err && n) {
    CB_LAUNCH(cb::cm_to_orig_kernel, cdiv(n, 256), 256, 0, st, p->d_out2, p->d_cm_orig, n, p->d_out2 + n);
    cudaMemcpyAsync(err, p->d_out2 + n, sizeof(double) * n, cudaMemcpyDeviceToHost, st);
  }
  std::vector<long long> hc(p->n_cams);
  std::vector<double> hlo(p->n_cams), hhi(p->n_cams);
  cudaMemcpyAsync(hlo.data(), d_lo, sizeof(double) * p->n_cams, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(hhi.data(), d_hi, sizeof(double) * p->n_cams, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(hc.data(), d_cnt, sizeof(long long) * p->n_cams, cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  cached_free(d_lo); cached_free(d_hi); cached_free(d_cnt);
  CB_CUDA(e);
  for (int i = 0; i < p->n_cams; ++i) {  // internal slot -> caller's camera index
    const int c = p->h_perm[i];
    count[c] = hc[i]; lo[c] = hlo[i]; hi[c] = hhi[i];
  }
  return CB_OK;
}

// Rigid-distance constraint rows (reprojection.py:112-117, 207-226; arrays as built by
// CaptureVolume._build_constraint_arrays, capture_volume.py:446-516, with
// weights = (pixel_sigma / f_median) / sigma, :377-381).  Host arrays; call once after problem_create.
int cb_ba_problem_set_constraints(CbBaProblem* p, int64_t n_c, const int32_t* groups_a, const int32_t* groups_b,
                                  const double* distances, const double* weights, void* stream) {
  if (!p || n_c < 0 || (n_c > 0 && (!groups_a || !groups_b || !distances || !weights))) {
    g_last_error = "cb_ba_problem_set_constraints: bad argument";
    return CB_E_INVALID;
  }
  if (p->n_c) { g_last_error = "constraints already set on this problem"; return CB_E_INVALID; }
  if (n_c == 0) return CB_OK;
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int nc = (int)n_c, npts = p->n_pts;
  for (long long i = 0; i < 4ll * nc; ++i)
    if (groups_a[i] < 0 || groups_a[i] >= npts || groups_b[i] < 0 || groups_b[i] >= npts) {
      g_last_error = "constraint group index out of range";
      return CB_E_INVALID;
    }
  // connected components of the constraint graph (union-find over points)
  std::vector<int> parent(npts);
  for (int i = 0; i < npts; ++i) parent[i] = i;
  auto find = [&](int a) { while (parent[a] != a) { parent[a] = parent[parent[a]]; a = parent[a]; } return a; };
  std::vector<char> used(npts, 0);
  for (int k = 0; k < nc; ++k) {
    const int r0 = find(groups_a[4 * k]);
    used[groups_a[4 * k]] = 1;
    for (int q = 0; q < 4; ++q) {
      used[groups_a[4 * k + q]] = 1; used[groups_b[4 * k + q]] = 1;
      parent[find(groups_a[4 * k + q])] = r0;
      parent[find(groups_b[4 * k + q])] = r0;
    }
  }
  std::vector<int> comp_of_root(npts, -1), pt_comp(npts, -1), pt_lidx(npts, -1);
  std::vector<std::vector<int>> comp_pts;
  for (int j = 0; j < npts; ++j) {
    if (!used[j]) continue;
    const int r = find(j);
    if (comp_of_root[r] < 0) { comp_of_root[r] = (int)comp_pts.size(); comp_pts.emplace_back(); }
    const int c = comp_of_root[r];
    pt_comp[j] = c;
    pt_lidx[j] = (int)comp_pts[c].size();
    comp_pts[c].push_back(j);
  }
  const int ncomp = (int)comp_pts.size();
  std::vector<int> cps(ncomp + 1, 0), cpts, ccs(ncomp + 1, 0), ccons(nc);
  std::vector<long long> loff(ncomp);
  long long ltot = 0;
  int ndmax = 0;
  for (int c = 0; c < ncomp; ++c) {
    cps[c] = (int)cpts.size();
    cpts.insert(cpts.end(), comp_pts[c].begin(), comp_pts[c].end());
    const long long n = 3ll * comp_pts[c].size();
    loff[c] = ltot;
    ltot += n * n;
    ndmax = std::max(ndmax, (int)n);
  }
  cps[ncomp] = (int)cpts.size();
  if (ndmax > 1200) {
    g_last_error = "a rigid component couples more than 400 points; not supported by this build";
    return CB_E_UNSUPPORTED;
  }
  std::vector<int> cnu(nc), cg((size_t)nc * 8, -1), cl((size_t)nc * 8, 0), ccomp(nc);
  std::vector<double> ccoef((size_t)nc * 8, 0.0);
  for (int k = 0; k < nc; ++k) {
    int nu = 0;
    for (int side = 0; side < 2; ++side)
      for (int q = 0; q < 4; ++q) {
        const int pt = side == 0 ? groups_a[4 * k + q] : groups_b[4 * k + q];
        int u = 0;
        for (; u < nu; ++u)
          if (cg[(size_t)k * 8 + u] == pt) break;
        if (u == nu) { cg[(size_t)k * 8 + u] = pt; cl[(size_t)k * 8 + u] = pt_lidx[pt]; ++nu; }
        ccoef[(size_t)k * 8 + u] += side == 0 ? 0.25 : -0.25;
      }
    cnu[k] = nu;
    ccomp[k] = pt_comp[groups_a[4 * k]];
    ccs[ccomp[k] + 1]++;
  }
  for (int c = 0; c < ncomp; ++c) ccs[c + 1] += ccs[c];
  {
    std::vector<int> cur(ccs.begin(), ccs.end() - 1);
    for (int k = 0; k < nc; ++k) ccons[cur[ccomp[k]]++] = k;  // ascending constraint id within a component
  }
  // upload
  int *d_nu, *d_g, *d_l, *d_cps, *d_cpts, *d_ccs, *d_ccons;
  double *d_coef, *d_dist, *d_w;
  long long* d_loff;
  CB_TRY(palloc(p, &d_nu, nc)); CB_TRY(palloc(p, &d_g, (size_t)nc * 8)); CB_TRY(palloc(p, &d_l, (size_t)nc * 8));
  CB_TRY(palloc(p, &d_coef, (size_t)nc * 8)); CB_TRY(palloc(p, &d_dist, nc)); CB_TRY(palloc(p, &d_w, nc));
  CB_TRY(palloc(p, &d_cps, ncomp + 1)); CB_TRY(palloc(p, &d_cpts, cpts.size())); CB_TRY(palloc(p, &d_ccs, ncomp + 1));
  CB_TRY(palloc(p, &d_ccons, nc)); CB_TRY(palloc(p, &d_loff, ncomp)); CB_TRY(palloc(p, &p->d_pt_comp, npts));
  for (int k = 0; k < 2; ++k) { CB_TRY(palloc(p, &p->d_c_rs[k], nc)); CB_TRY(palloc(p, &p->d_c_dirw[k], 3 * (size_t)nc)); }
  CB_TRY(palloc(p, &p->d_compL, (size_t)ltot));
#define CB_UP(dst, vec) CB_CUDA(cudaMemcpyAsync(dst, (vec).data(), sizeof((vec)[0]) * (vec).size(), cudaMemcpyHostToDevice, st))
  CB_UP(d_nu, cnu); CB_UP(d_g, cg); CB_UP(d_l, cl); CB_UP(d_coef, ccoef); CB_UP(d_cps, cps); CB_UP(d_cpts, cpts);
  CB_UP(d_ccs, ccs); CB_UP(d_ccons, ccons); CB_UP(d_loff, loff); CB_UP(p->d_pt_comp, pt_comp);
#undef CB_UP
  CB_CUDA(cudaMemcpyAsync(d_dist, distances, sizeof(double) * nc, cudaMemcpyHostToDevice, st));
  CB_CUDA(cudaMemcpyAsync(d_w, weights, sizeof(double) * nc, cudaMemcpyHostToDevice, st));
  p->n_cblk = cdiv(nc, cb::CC_THREADS);
  // the cost / step partial-sum arrays grow by the constraint blocks / components
  const int NACC = (p->P == 6) ? 28 : 55;
  CB_TRY(palloc(p, &p->d_camcost, (size_t)p->n_cams + p->n_cblk));
  CB_TRY(palloc(p, &p->d_partial, (size_t)std::max(p->n_chunks, 1) * NACC + p->n_cblk));
  CB_TRY(palloc(p, &p->d_bpart, 3 * ((size_t)p->pt_grid + ncomp)));
  // captured launches hold the old buffer addresses
  destroy_graph(p->trial_graph);
  destroy_graph(p->loop_graph);
  CB_CUDA(cudaStreamSynchronize(st));
  p->ct.n_c = nc; p->ct.n_comp = ncomp; p->ct.n_dim_max = ndmax;
  p->ct.c_nu = d_nu; p->ct.c_gidx = d_g; p->ct.c_lidx = d_l; p->ct.c_coef = d_coef; p->ct.c_dist = d_dist; p->ct.c_w = d_w;
  p->ct.comp_pt_start = d_cps; p->ct.comp_pts = d_cpts; p->ct.comp_c_start = d_ccs; p->ct.comp_cons = d_ccons;
  p->ct.comp_L_off = d_loff; p->ct.pt_comp = p->d_pt_comp;
  p->n_c = nc; p->n_comp = ncomp; p->n_dim_max = ndmax;
  const int esm = std::min(ndmax, cb::CC_SMEM_DIM);
  p->comp_build_smem = sizeof(double) * ((size_t)ndmax * (1 + p->P) + (size_t)esm * esm) + 4 * ((size_t)(p->n_cams + 31) / 32 + 4);
  p->comp_back_smem = sizeof(double) * ((size_t)p->nP + ndmax);
  if (p->P == 6)
    CB_CUDA(cudaFuncSetAttribute(cb::comp_build_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->comp_build_smem));
  else
    CB_CUDA(cudaFuncSetAttribute(cb::comp_build_kernel<9>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->comp_build_smem));
  CB_CUDA(cudaFuncSetAttribute(cb::comp_backsub_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->comp_back_smem));
  // merging the components' tile masks only adds incidences, so problems on the dense product stay on it unchanged
  if (p->schur_sparse) CB_TRY(rebuild_schur_items(p, st));
  p->h_ga.assign(groups_a, groups_a + 4 * (size_t)nc); p->h_gb.assign(groups_b, groups_b + 4 * (size_t)nc);
  p->h_cdist.assign(distances, distances + nc); p->h_cw.assign(weights, weights + nc);
  return CB_OK;
}

int64_t cb_ba_problem_n_constraints(const CbBaProblem* p) { return p ? p->n_c : -1; }

// Constraint rows at x: r (n_c, == the tail of joint_residuals) and dir (n_c x 3) = w * unit(mean(P[ga]) - mean(P[gb]));
// the Jacobian entry of member point q of group a (b) is +(-) dir / 4, summed over repeats (reprojection.py:207-226).
int cb_ba_constraint_rows(CbBaProblem* p, const double* x, double* r_out, double* dir_out, void* stream) {
  if (!p || !x || !r_out) { g_last_error = "cb_ba_constraint_rows: null argument"; return CB_E_INVALID; }
  if (!p->n_c) return CB_OK;
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  CB_TRY(upload_x(p, x, st));
  double *d_r, *d_rs, *d_dir;
  CB_TRY(dalloc(&d_r, p->n_c)); CB_TRY(dalloc(&d_rs, p->n_c)); CB_TRY(dalloc(&d_dir, 3 * (size_t)p->n_c));
  CB_LAUNCH((cb::constraint_eval_kernel<false>), p->n_cblk, cb::CC_THREADS, 0, st, (const cb::LmState*)nullptr, 0, p->ct,
            p->c_xp(), 0, 1.0, (cb::Ptr2{{d_rs, d_rs}}), (cb::Ptr2{{d_dir, d_dir}}), d_r, (double*)nullptr);
  cudaMemcpyAsync(r_out, d_r, sizeof(double) * p->n_c, cudaMemcpyDeviceToHost, st);
  if (dir_out) cudaMemcpyAsync(dir_out, d_dir, sizeof(double) * 3 * (size_t)p->n_c, cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  cached_free(d_r); cached_free(d_rs); cached_free(d_dir);
  CB_CUDA(e);
  return CB_OK;
}

// Overall and per-camera RMS pixel error (reprojection_report's overall_rmse / by_camera,
// capture_volume.py:197-202), reduced on the device.
int cb_ba_rmse_px(CbBaProblem* p, const double* x, double* overall, double* per_camera, void* stream) {
  if (!p || !x || !overall) { g_last_error = "cb_ba_rmse_px: null argument"; return CB_E_INVALID; }
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  CB_TRY(p->P == 6 ? (eval_mode<6, 4>(p, x, st)) : (eval_mode<9, 4>(p, x, st)));
  double* d_ss;
  CB_TRY(dalloc(&d_ss, p->n_cams));
  CB_LAUNCH(cb::cam_err_stats_kernel, p->n_cams, 256, 0, st, p->d_out2, p->d_cam_start, (const double*)nullptr,
            (long long*)nullptr, d_ss);
  std::vector<double> ss(p->n_cams);
  std::vector<int> cs(p->n_cams + 1);
  cudaMemcpyAsync(ss.data(), d_ss, sizeof(double) * p->n_cams, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(cs.data(), p->d_cam_start, sizeof(int) * (p->n_cams + 1), cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  cached_free(d_ss);
  CB_CUDA(e);
  double tot = 0.0;
  for (int c = 0; c < p->n_cams; ++c) {
    tot += ss[c];
    const int nc = cs[c + 1] - cs[c];
    if (per_camera) per_camera[p->h_perm[c]] = nc > 0 ? std::sqrt(ss[c] / nc) : 0.0;
  }
  *overall = p->n_obs > 0 ? std::sqrt(tot / p->n_obs) : 0.0;
  return CB_OK;
}

// Observation cull on the device (capture_volume.py:607-646): keep error <= thresholds[camera], restore the
// lowest-error observations of a camera that would fall below min_per_camera, compact the caller-order list
// and build the filtered problem from it without a host round trip.  keep_mask (host, n_obs bytes, caller
// order) may be NULL.
int cb_ba_cull(CbBaProblem* p, const double* x, const double* thresholds, int32_t min_per_camera, CbBaProblem** out,
               int64_t* n_kept, uint8_t* keep_mask, void* stream) {
  if (!p || !x || !thresholds || !out || min_per_camera < 0) { g_last_error = "cb_ba_cull: bad argument"; return CB_E_INVALID; }
  *out = nullptr;
  CB_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int n = p->n_obs, nc = p->n_cams;
  CB_TRY(p->P == 6 ? (eval_mode<6, 4>(p, x, st)) : (eval_mode<9, 4>(p, x, st)));
  double *d_thr, *d_ss;
  long long* d_kept;
  unsigned char* d_flag;
  int *d_iota, *d_sel, *d_nsel;
  ScopedFree sf;  // every early return below releases the temporaries
  CB_TRY(dalloc(&d_thr, nc)); sf.dev.push_back(d_thr);
  CB_TRY(dalloc(&d_ss, nc)); sf.dev.push_back(d_ss);
  CB_TRY(dalloc(&d_kept, nc)); sf.dev.push_back(d_kept);
  CB_TRY(dalloc(&d_flag, n)); sf.dev.push_back(d_flag);
  CB_TRY(dalloc(&d_iota, n)); sf.dev.push_back(d_iota);
  CB_TRY(dalloc(&d_sel, n)); sf.dev.push_back(d_sel);
  CB_TRY(dalloc(&d_nsel, 1)); sf.dev.push_back(d_nsel);
  std::vector<double> thr(nc);
  for (int i = 0; i < nc; ++i) thr[i] = thresholds[p->h_perm[i]];  // by internal camera slot
  std::vector<long long> kept(nc);
  std::vector<int> cs(nc + 1);
  CB_CUDA(cudaMemcpyAsync(d_thr, thr.data(), sizeof(double) * nc, cudaMemcpyHostToDevice, st));
  CB_LAUNCH(cb::cam_err_stats_kernel, nc, 256, 0, st, p->d_out2, p->d_cam_start, (const double*)d_thr, d_kept, d_ss);
  CB_CUDA(cudaMemcpyAsync(kept.data(), d_kept, sizeof(long long) * nc, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(cs.data(), p->d_cam_start, sizeof(int) * (nc + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  bool changed = false;
  for (int c = 0; c < nc; ++c) {  // safety floor (rare): threshold := n_needed-th smallest of the dropped errors
    const long long total = cs[c + 1] - cs[c];
    if (kept[c] < min_per_camera && kept[c] < total) {
      const long long need = std::min<long long>(min_per_camera, total) - kept[c];
      std::vector<double> ec((size_t)total);
      CB_CUDA(cudaMemcpy(ec.data(), p->d_out2 + cs[c], sizeof(double) * total, cudaMemcpyDeviceToHost));
      std::vector<double> dropped;
      for (double v : ec)
        if (!(v <= thr[c])) dropped.push_back(v);
      if ((long long)dropped.size() >= need) {
        std::nth_element(dropped.begin(), dropped.begin() + (need - 1), dropped.end());
        thr[c] = dropped[need - 1];
        changed = true;
      }
    }
  }
  if (changed) CB_CUDA(cudaMemcpyAsync(d_thr, thr.data(), sizeof(double) * nc, cudaMemcpyHostToDevice, st));
  CB_LAUNCH(cb::keep_flag_kernel, cdiv(n, 256), 256, 0, st, p->d_out2, p->d_cm_orig, p->d_cam_start, nc,
            (const double*)d_thr, n, d_flag);
  CB_LAUNCH(cb::iota_kernel, cdiv(n, 256), 256, 0, st, d_iota, n);
  size_t tb = 0;
  cub::DeviceSelect::Flagged(nullptr, tb, d_iota, d_flag, d_sel, d_nsel, n, st);
  void* d_tmp;
  CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tb, 16)));
  sf.dev.push_back(d_tmp);
  CB_CUDA(cub::DeviceSelect::Flagged(d_tmp, tb, d_iota, d_flag, d_sel, d_nsel, n, st));
  g_launches.fetch_add(2);
  int nsel = 0;
  CB_CUDA(cudaMemcpyAsync(&nsel, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (keep_mask) CB_CUDA(cudaMemcpyAsync(keep_mask, d_flag, n, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  int rc = CB_OK;
  if (nsel <= 0) {
    g_last_error = "No image observations provided";  // every observation was culled
    rc = CB_E_INVALID;
  } else {
    int *c_cam = nullptr, *c_pt = nullptr;
    double* c_xy = nullptr;
    if (dalloc(&c_cam, nsel) != CB_OK || dalloc(&c_pt, nsel) != CB_OK || dalloc(&c_xy, 2 * (size_t)nsel) != CB_OK) {
      cached_free(c_cam); cached_free(c_pt); cached_free(c_xy);
      return CB_E_NOMEM;
    }
    CB_LAUNCH(cb::gather_obs_kernel, cdiv(nsel, 256), 256, 0, st, d_sel, nsel, p->d_obs_cam, p->d_obs_pt,
              reinterpret_cast<const double2*>(p->d_obs_xy), c_cam, c_pt, reinterpret_cast<double2*>(c_xy));
    CbBaProblemDesc d2;
    d2.n_cams = nc; d2.n_pts = p->n_pts; d2.n_obs = nsel;
    d2.cam_flags = p->h_cam_flags.data(); d2.cam_const = p->h_cam_const.data();
    d2.obs_cam = c_cam; d2.obs_pt = c_pt; d2.obs_xy = c_xy; d2.obs_on_device = 1;
    d2.obs_cam_bits = 32;
    d2.cam_order = p->h_perm.data();  // the filtered problem keeps this problem's camera order
    CbBaProblem* q = new CbBaProblem();
    q->allocs.push_back(c_cam); q->allocs.push_back(c_pt); q->allocs.push_back(c_xy);  // owned by the new problem
    rc = problem_create_impl(&d2, p->device, st, q);
    if (rc != CB_OK) {
      std::string keep = g_last_error;
      cb_ba_problem_destroy(q);
      g_last_error = keep;
    } else {
      if (p->n_c)
        rc = cb_ba_problem_set_constraints(q, p->n_c, p->h_ga.data(), p->h_gb.data(), p->h_cdist.data(), p->h_cw.data(),
                                           stream);
      if (rc != CB_OK) {
        std::string keep = g_last_error;
        cb_ba_problem_destroy(q);
        g_last_error = keep;
      } else {
        q->order_auto = p->order_auto;
        *out = q;
      }
    }
  }
  if (n_kept) *n_kept = nsel;
  return rc;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// the step in front of bundle adjustment: undistortion + DLT triangulation (SURVEY.md §8(f) rank 3)
// ------------------------------------------------------------------------------------------
namespace {



int build_undist_table(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                       std::vector<cb::UndistCam>& tab) {
  tab.resize(n_cams);
  for (int c = 0; c < n_cams; ++c) {
    cb::UndistCam& u = tab[c];
    u.fx = cam_k[5 * c]; u.fy = cam_k[5 * c + 1]; u.cx = cam_k[5 * c + 2]; u.cy = cam_k[5 * c + 3]; u.skew = cam_k[5 * c + 4];
    for (int k = 0; k < 12; ++k) u.d[k] = cam_dist[12 * c + k];
    u.fisheye = cam_fisheye[c] ? 1 : 0;
    u.pad = 0;
    if (!(u.fx != 0.0) || !(u.fy != 0.0)) { g_last_error = "zero focal length in the camera table"; return CB_E_INVALID; }
  }
  return CB_OK;
}

// host array -> device through a pinned bounce buffer (or pass through when already on the device)
template <typename T>
int to_device(const T* src, size_t n, int on_device, const T** out, ScopedFree& sf, cudaStream_t st) {
  if (on_device) { *out = src; return CB_OK; }
  T* d = nullptr;
  CB_TRY(dalloc(&d, n));
  sf.dev.push_back(d);
  if (sizeof(T) * n >= ((size_t)2 << 20)) {  // large arrays: pool threads stage, the DMA is queued block by block
    CB_TRY(staged_h2d(d, src, sizeof(T) * n, st, sf, 8));
    *out = d;
    return CB_OK;
  }
  T* h = nullptr;
  CB_TRY(cached_malloc_host((void**)&h, sizeof(T) * std::max<size_t>(n, 1)));
  sf.host.push_back(h);
  stream_copy(h, src, sizeof(T) * n);  // non-temporal: the DMA reads it next (see stream_copy)
  CB_CUDA(cudaMemcpyAsync(d, h, sizeof(T) * n, cudaMemcpyHostToDevice, st));
  *out = d;
  return CB_OK;
}

// host doubles -> device floats, converted while staging into the pinned bounce buffer
int to_device_f32(const double* src, size_t n, const float** out, ScopedFree& sf, cudaStream_t st) {
  float* d = nullptr;
  CB_TRY(dalloc(&d, n));
  sf.dev.push_back(d);
  float* h = nullptr;
  CB_TRY(cached_malloc_host((void**)&h, sizeof(float) * std::max<size_t>(n, 1)));
  sf.host.push_back(h);
  const size_t chunk = (size_t)1 << 20;  // elements
  for (size_t off = 0; off < n; off += chunk) {
    const size_t m = std::min(chunk, n - off);
    for (size_t i = 0; i < m; ++i) h[off + i] = (float)src[off + i];
    CB_CUDA(cudaMemcpyAsync(d + off, h + off, sizeof(float) * m, cudaMemcpyHostToDevice, st));
  }
  *out = d;
  return CB_OK;
}

int validate_rows(const int* d_cam, const long long* d_key, long long n, int n_cams, cudaStream_t st, const char* who) {
  int* d_bad = nullptr;
  CB_TRY(dalloc(&d_bad, 1));
  CB_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
  CB_LAUNCH(cb::tri_validate_kernel, cdiv(n, 256), 256, 0, st, d_cam, d_key, n, n_cams, d_bad);
  int bad = 0;
  CB_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  cached_free(d_bad);
  if (bad) {
    g_last_error = std::string(who) + ": camera index out of range or negative group key in " + std::to_string(bad) + " rows";
    return CB_E_INVALID;
  }
  return CB_OK;
}

}  // namespace

extern "C" {

int cb_undistort_points(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                        int64_t n, const int32_t* obs_cam, const double* xy_in, int on_device, int to_pixels,
                        double* xy_out, int device, void* stream) {
  if (n_cams <= 0 || !cam_fisheye || !cam_k || !cam_dist || n < 0 || (n > 0 && (!xy_in || !xy_out))) {
    g_last_error = "cb_undistort_points: bad argument";
    return CB_E_INVALID;
  }
  if (n_cams > 1 && !obs_cam) { g_last_error = "cb_undistort_points: obs_cam is required with more than one camera"; return CB_E_INVALID; }
  CB_TRY(select_device(device));
  if (n == 0) return CB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ScopedFree sf;
  std::vector<cb::UndistCam> tab;
  CB_TRY(build_undist_table(n_cams, cam_fisheye, cam_k, cam_dist, tab));
  cb::UndistCam* d_tab = nullptr;
  CB_TRY(dalloc(&d_tab, (size_t)n_cams));
  sf.dev.push_back(d_tab);
  CB_CUDA(cudaMemcpyAsync(d_tab, tab.data(), sizeof(cb::UndistCam) * n_cams, cudaMemcpyHostToDevice, st));
  const int* d_cam = nullptr;
  const double* d_in = nullptr;
  if (obs_cam) CB_TRY(to_device(obs_cam, (size_t)n, on_device, &d_cam, sf, st));
  CB_TRY(to_device(xy_in, 2 * (size_t)n, on_device, &d_in, sf, st));
  double* d_out = xy_out;
  double* h_out = nullptr;
  if (!on_device) {
    CB_TRY(dalloc(&d_out, 2 * (size_t)n));
    sf.dev.push_back(d_out);
    CB_TRY(cached_malloc_host((void**)&h_out, sizeof(double) * 2 * (size_t)n));
    sf.host.push_back(h_out);
  }
  if (d_cam) CB_TRY(validate_rows(d_cam, nullptr, n, n_cams, st, "cb_undistort_points"));
  CB_LAUNCH(cb::undistort_kernel<double>, cdiv(n, 256), 256, 0, st, d_tab, d_cam, d_in, d_out, (long long)n,
            to_pixels ? 1 : 0);
  CB_CUDA(cudaGetLastError());
  if (!on_device) {
    CB_CUDA(cudaMemcpyAsync(h_out, d_out, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost, st));
    CB_CUDA(cudaStreamSynchronize(st));
    std::memcpy(xy_out, h_out, sizeof(double) * 2 * (size_t)n);
  } else {
    CB_CUDA(cudaStreamSynchronize(st));  // the camera table is a stack-lifetime upload
  }
  return CB_OK;
}

}  // extern "C"

namespace {

int group_by_key(const long long* d_key, int n, cudaStream_t st, ScopedFree& sf, int** d_rows, int** d_start, int* n_groups);

// shared body of cb_triangulate_dlt / cb_undistort_triangulate: `undist` non-null = obs_xy are raw pixels,
// undistorted on the device (normalised output) before the DLT, never leaving HBM in between.
int triangulate_impl(int32_t n_cams, const std::vector<cb::UndistCam>* undist, const double* proj, int64_t n_obs,
                     const int32_t* obs_cam, const int64_t* obs_key, const double* obs_xy, int obs_on_device,
                     int32_t max_groups, int32_t* n_groups_out, double* xyz_out, int32_t* count_out,
                     int32_t* rep_row_out, uint64_t* camset_sig_out, CbTriStats* stats, int device, void* stream) {
  if (n_cams <= 0 || !proj || n_obs < 0 || n_obs > 0x7fffffffLL || !n_groups_out || max_groups < 0 ||
      (n_obs > 0 && (!obs_cam || !obs_key || !obs_xy)) ||
      (max_groups > 0 && (!xyz_out || !count_out || !rep_row_out || !camset_sig_out))) {
    g_last_error = "cb_triangulate_dlt: bad argument";
    return CB_E_INVALID;
  }
  CB_TRY(select_device(device));
  *n_groups_out = 0;
  if (stats) std::memset(stats, 0, sizeof(*stats));
  if (n_obs == 0) return CB_OK;
  const long long launches0 = g_launches.load();
  cudaStream_t st = (cudaStream_t)stream;
  ScopedFree sf;
  const int n = (int)n_obs;
  const int TB = 256, G = cdiv(n, TB);
  cudaEvent_t ev[4];
  for (auto& e : ev) CB_CUDA(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 4; ++i) cudaEventDestroy(e[i]); } } evg{ev};
  CB_CUDA(cudaEventRecord(ev[0], st));

  const int* d_cam = nullptr;
  const long long* d_key = nullptr;
  const double* d_xy = nullptr;
  CB_TRY(to_device(obs_cam, (size_t)n, obs_on_device, &d_cam, sf, st));
  CB_TRY(to_device((const long long*)obs_key, (size_t)n, obs_on_device, &d_key, sf, st));
  CB_TRY(validate_rows(d_cam, d_key, n, n_cams, st, "cb_triangulate_dlt"));
  if (undist) {
    cb::UndistCam* d_tab = nullptr;
    CB_TRY(dalloc(&d_tab, (size_t)n_cams));
    sf.dev.push_back(d_tab);
    CB_CUDA(cudaMemcpyAsync(d_tab, undist->data(), sizeof(cb::UndistCam) * n_cams, cudaMemcpyHostToDevice, st));
    double* d_und = nullptr;
    CB_TRY(dalloc(&d_und, 2 * (size_t)n));
    sf.dev.push_back(d_und);
    if (obs_on_device) {
      CB_LAUNCH(cb::undistort_kernel<double>, G, TB, 0, st, d_tab, d_cam, obs_xy, d_und, (long long)n, 0);
    } else {
      // host pixels: round to float32 while staging (the reference does the same cast, camera_array.py:156),
      // which halves the upload
      const float* d_px = nullptr;
      CB_TRY(to_device_f32(obs_xy, 2 * (size_t)n, &d_px, sf, st));
      CB_LAUNCH(cb::undistort_kernel<float>, G, TB, 0, st, d_tab, d_cam, d_px, d_und, (long long)n, 0);
    }
    d_xy = d_und;
  } else {
    CB_TRY(to_device(obs_xy, 2 * (size_t)n, obs_on_device, &d_xy, sf, st));
  }
  double* d_proj = nullptr;
  CB_TRY(dalloc(&d_proj, 12 * (size_t)n_cams));
  sf.dev.push_back(d_proj);
  CB_CUDA(cudaMemcpyAsync(d_proj, proj, sizeof(double) * 12 * (size_t)n_cams, cudaMemcpyHostToDevice, st));

  // (1) stable radix sort of (key, row) -> rows of one group adjacent, in caller order inside the group; (2) boundaries
  int *v_out = nullptr, *d_start = nullptr, n_groups = 0;
  CB_TRY(group_by_key(d_key, n, st, sf, &v_out, &d_start, &n_groups));
  CB_CUDA(cudaEventRecord(ev[1], st));
  *n_groups_out = n_groups;
  if (n_groups > max_groups) {
    g_last_error = "cb_triangulate_dlt: " + std::to_string(n_groups) + " groups but room for " + std::to_string(max_groups);
    return CB_E_INVALID;
  }
  // (3) DLT per group
  double* d_xyz = nullptr;
  int *d_count = nullptr, *d_rep = nullptr;
  unsigned long long* d_sig = nullptr;
  CB_TRY(dalloc(&d_xyz, 3 * (size_t)n_groups)); sf.dev.push_back(d_xyz);
  CB_TRY(dalloc(&d_count, (size_t)n_groups)); sf.dev.push_back(d_count);
  CB_TRY(dalloc(&d_rep, (size_t)n_groups)); sf.dev.push_back(d_rep);
  CB_TRY(dalloc(&d_sig, 2 * (size_t)n_groups)); sf.dev.push_back(d_sig);
  const size_t proj_bytes = sizeof(double) * 13 * (size_t)n_cams;  // padded stride, see tri_dlt_kernel
  const int in_smem = proj_bytes <= 40 * 1024 ? 1 : 0;
  // 8 lanes per group: the serial 4x4 eigen-solve of one lane per group, not the gather, bounds this kernel, so
  // more groups per warp wins until groups get very long
  const int lanes = (n / std::max(n_groups, 1) > 96) ? 32 : 8;
  const long long threads = (long long)n_groups * lanes;
  CB_CUDA(cudaEventRecord(ev[2], st));
  if (lanes == 32)
    CB_LAUNCH(cb::tri_dlt_kernel<32>, cdiv(threads, cb::TRI_THREADS), cb::TRI_THREADS, in_smem ? proj_bytes : 0, st,
              d_proj, n_cams, in_smem, d_start, v_out, d_cam, d_xy, n_groups, d_xyz, d_count, d_rep, d_sig);
  else
    CB_LAUNCH(cb::tri_dlt_kernel<8>, cdiv(threads, cb::TRI_THREADS), cb::TRI_THREADS, in_smem ? proj_bytes : 0, st,
              d_proj, n_cams, in_smem, d_start, v_out, d_cam, d_xy, n_groups, d_xyz, d_count, d_rep, d_sig);
  CB_CUDA(cudaGetLastError());
  CB_CUDA(cudaEventRecord(ev[3], st));
  CB_CUDA(cudaMemcpyAsync(xyz_out, d_xyz, sizeof(double) * 3 * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(count_out, d_count, sizeof(int) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(rep_row_out, d_rep, sizeof(int) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(camset_sig_out, d_sig, sizeof(unsigned long long) * 2 * (size_t)n_groups,
                          cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[0], ev[1]); stats->group_ms = ms;
    cudaEventElapsedTime(&ms, ev[2], ev[3]); stats->dlt_ms = ms;
    cudaEventElapsedTime(&ms, ev[0], ev[3]); stats->total_ms = ms;
    stats->kernel_launches = (int)(g_launches.load() - launches0);
  }
  return CB_OK;
}

}  // namespace

extern "C" {

int cb_triangulate_dlt(int32_t n_cams, const double* proj, int64_t n_obs, const int32_t* obs_cam,
                       const int64_t* obs_key, const double* obs_xy, int obs_on_device, int32_t max_groups,
                       int32_t* n_groups_out, double* xyz_out, int32_t* count_out, int32_t* rep_row_out,
                       uint64_t* camset_sig_out, CbTriStats* stats, int device, void* stream) {
  return triangulate_impl(n_cams, nullptr, proj, n_obs, obs_cam, obs_key, obs_xy, obs_on_device, max_groups,
                          n_groups_out, xyz_out, count_out, rep_row_out, camset_sig_out, stats, device, stream);
}

int cb_undistort_triangulate(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                             const double* proj, int64_t n_obs, const int32_t* obs_cam, const int64_t* obs_key,
                             const double* obs_px, int obs_on_device, int32_t max_groups, int32_t* n_groups_out,
                             double* xyz_out, int32_t* count_out, int32_t* rep_row_out, uint64_t* camset_sig_out,
                             CbTriStats* stats, int device, void* stream) {
  if (n_cams <= 0 || !cam_fisheye || !cam_k || !cam_dist) {
    g_last_error = "cb_undistort_triangulate: bad argument";
    return CB_E_INVALID;
  }
  std::vector<cb::UndistCam> tab;
  CB_TRY(build_undist_table(n_cams, cam_fisheye, cam_k, cam_dist, tab));
  return triangulate_impl(n_cams, &tab, proj, n_obs, obs_cam, obs_key, obs_px, obs_on_device, max_groups, n_groups_out,
                          xyz_out, count_out, rep_row_out, camset_sig_out, stats, device, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// extrinsic bootstrap: batched planar PnP and stereo RMSE (SURVEY.md §8(f) rank 1)
// ------------------------------------------------------------------------------------------
namespace {

// stable sort of the rows by key, group boundaries: d_rows (n), d_start (n_groups + 1)
int group_by_key(const long long* d_key, int n, cudaStream_t st, ScopedFree& sf, int** d_rows, int** d_start, int* n_groups) {
  const int TB = 256, G = cdiv(n, TB);
  unsigned long long* k_out = nullptr;
  int *v_in = nullptr, *v_out = nullptr, *d_head = nullptr, *d_gid = nullptr, *dstart = nullptr;
  CB_TRY(dalloc(&k_out, (size_t)n)); sf.dev.push_back(k_out);
  CB_TRY(dalloc(&v_in, (size_t)n)); sf.dev.push_back(v_in);
  CB_TRY(dalloc(&v_out, (size_t)n)); sf.dev.push_back(v_out);
  CB_TRY(dalloc(&d_head, (size_t)n)); sf.dev.push_back(d_head);
  CB_TRY(dalloc(&d_gid, (size_t)n)); sf.dev.push_back(d_gid);
  CB_TRY(dalloc(&dstart, (size_t)n + 1)); sf.dev.push_back(dstart);
  size_t tb_sort = 0, tb_scan = 0, tb_red = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, (const unsigned long long*)d_key, k_out, v_in, v_out, n, 0, 64, st);
  cub::DeviceScan::InclusiveSum(nullptr, tb_scan, d_head, d_gid, n, st);
  cub::DeviceReduce::Max(nullptr, tb_red, (const unsigned long long*)d_key, (unsigned long long*)nullptr, n, st);
  void* d_tmp = nullptr;
  size_t tb = std::max(std::max(tb_sort, tb_scan), tb_red);
  CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tb, 16)));
  sf.dev.push_back(d_tmp);
  CB_LAUNCH(cb::tri_iota_kernel, G, TB, 0, st, v_in, (long long)n);
  // radix passes only over the key's significant bits (a packed (sync, object, keypoint) key of a 50k-point rig has 16)
  unsigned long long* d_max = nullptr;
  CB_TRY(dalloc(&d_max, 1)); sf.dev.push_back(d_max);
  size_t tb_max = tb;
  CB_CUDA(cub::DeviceReduce::Max(d_tmp, tb_max, (const unsigned long long*)d_key, d_max, n, st));
  unsigned long long h_max = 0;
  CB_CUDA(cudaMemcpyAsync(&h_max, d_max, sizeof(h_max), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  const int key_bits = std::min(63, bits_for(h_max));
  CB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const unsigned long long*)d_key, k_out, v_in, v_out, n, 0, key_bits, st));
  g_launches.fetch_add(2 + 2 * ((key_bits + 7) / 8));
  CB_LAUNCH(cb::tri_heads_kernel, G, TB, 0, st, k_out, (long long)n, d_head);
  CB_CUDA(cub::DeviceScan::InclusiveSum(d_tmp, tb, d_head, d_gid, n, st));
  g_launches.fetch_add(2);
  CB_LAUNCH(cb::tri_starts_kernel, G, TB, 0, st, d_head, d_gid, (long long)n, dstart);
  CB_CUDA(cudaMemcpyAsync(n_groups, d_gid + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  *d_rows = v_out;
  *d_start = dstart;
  return CB_OK;
}

// pixels (host, double) -> device, undistorted to the normalised plane with the reference's float32 rounding
int upload_undistorted(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist, int n,
                       const int* d_cam, const double* obs_px, ScopedFree& sf, cudaStream_t st, double** d_norm) {
  std::vector<cb::UndistCam> tab;
  CB_TRY(build_undist_table(n_cams, cam_fisheye, cam_k, cam_dist, tab));
  cb::UndistCam* d_tab = nullptr;
  CB_TRY(dalloc(&d_tab, (size_t)n_cams));
  sf.dev.push_back(d_tab);
  CB_CUDA(cudaMemcpy(d_tab, tab.data(), sizeof(cb::UndistCam) * n_cams, cudaMemcpyHostToDevice));
  double* d_und = nullptr;
  CB_TRY(dalloc(&d_und, 2 * (size_t)n));
  sf.dev.push_back(d_und);
  const float* d_px = nullptr;
  CB_TRY(to_device_f32(obs_px, 2 * (size_t)n, &d_px, sf, st));
  CB_LAUNCH(cb::undistort_kernel<float>, cdiv(n, 256), 256, 0, st, d_tab, d_cam, d_px, d_und, (long long)n, 0);
  *d_norm = d_und;
  return CB_OK;
}

}  // namespace

extern "C" {

int cb_pnp_ippe(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist, int64_t n_obs,
                const int32_t* obs_cam, const int64_t* obs_key, const double* obs_px, const double* obs_obj,
                int32_t min_points, int32_t max_groups, int32_t* n_groups_out, double* R_out, double* t_out,
                double* rmse_out, int32_t* status_out, int32_t* count_out, int32_t* rep_row_out, CbTriStats* stats,
                int device, void* stream) {
  if (n_cams <= 0 || !cam_fisheye || !cam_k || !cam_dist || n_obs < 0 || n_obs > 0x7fffffffLL || !n_groups_out ||
      max_groups < 0 || (n_obs > 0 && (!obs_cam || !obs_key || !obs_px || !obs_obj)) ||
      (max_groups > 0 && (!R_out || !t_out || !rmse_out || !status_out || !count_out || !rep_row_out))) {
    g_last_error = "cb_pnp_ippe: bad argument";
    return CB_E_INVALID;
  }
  CB_TRY(select_device(device));
  *n_groups_out = 0;
  if (stats) std::memset(stats, 0, sizeof(*stats));
  if (n_obs == 0) return CB_OK;
  const long long launches0 = g_launches.load();
  cudaStream_t st = (cudaStream_t)stream;
  ScopedFree sf;
  const int n = (int)n_obs;
  cudaEvent_t ev[4];
  for (auto& e : ev) CB_CUDA(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 4; ++i) cudaEventDestroy(e[i]); } } evg{ev};
  CB_CUDA(cudaEventRecord(ev[0], st));
  const int* d_cam = nullptr;
  const long long* d_key = nullptr;
  const double* d_obj = nullptr;
  CB_TRY(to_device(obs_cam, (size_t)n, 0, &d_cam, sf, st));
  CB_TRY(to_device((const long long*)obs_key, (size_t)n, 0, &d_key, sf, st));
  CB_TRY(to_device(obs_obj, 3 * (size_t)n, 0, &d_obj, sf, st));
  CB_TRY(validate_rows(d_cam, d_key, n, n_cams, st, "cb_pnp_ippe"));
  double* d_norm = nullptr;
  CB_TRY(upload_undistorted(n_cams, cam_fisheye, cam_k, cam_dist, n, d_cam, obs_px, sf, st, &d_norm));
  int *d_rows = nullptr, *d_start = nullptr, n_groups = 0;
  CB_TRY(group_by_key(d_key, n, st, sf, &d_rows, &d_start, &n_groups));
  CB_CUDA(cudaEventRecord(ev[1], st));
  *n_groups_out = n_groups;
  if (n_groups > max_groups) {
    g_last_error = "cb_pnp_ippe: " + std::to_string(n_groups) + " groups but room for " + std::to_string(max_groups);
    return CB_E_INVALID;
  }
  double *d_R, *d_t, *d_rmse;
  int *d_status, *d_count, *d_rep;
  CB_TRY(dalloc(&d_R, 9 * (size_t)n_groups)); sf.dev.push_back(d_R);
  CB_TRY(dalloc(&d_t, 3 * (size_t)n_groups)); sf.dev.push_back(d_t);
  CB_TRY(dalloc(&d_rmse, (size_t)n_groups)); sf.dev.push_back(d_rmse);
  CB_TRY(dalloc(&d_status, (size_t)n_groups)); sf.dev.push_back(d_status);
  CB_TRY(dalloc(&d_count, (size_t)n_groups)); sf.dev.push_back(d_count);
  CB_TRY(dalloc(&d_rep, (size_t)n_groups)); sf.dev.push_back(d_rep);
  CB_CUDA(cudaEventRecord(ev[2], st));
  CB_LAUNCH(cb::pnp_ippe_kernel, cdiv((long long)n_groups * 32, cb::BS_THREADS), cb::BS_THREADS, 0, st, d_start, d_rows, d_obj,
            (const double*)d_norm, n_groups, (int)min_points, d_R, d_t, d_rmse, d_status, d_count, d_rep);
  CB_CUDA(cudaGetLastError());
  CB_CUDA(cudaEventRecord(ev[3], st));
  CB_CUDA(cudaMemcpyAsync(R_out, d_R, sizeof(double) * 9 * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(t_out, d_t, sizeof(double) * 3 * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(rmse_out, d_rmse, sizeof(double) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(status_out, d_status, sizeof(int) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(count_out, d_count, sizeof(int) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(rep_row_out, d_rep, sizeof(int) * (size_t)n_groups, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[0], ev[1]); stats->group_ms = ms;
    cudaEventElapsedTime(&ms, ev[2], ev[3]); stats->dlt_ms = ms;
    cudaEventElapsedTime(&ms, ev[0], ev[3]); stats->total_ms = ms;
    stats->kernel_launches = (int)(g_launches.load() - launches0);
  }
  return CB_OK;
}

int cb_stereo_rmse(int32_t n_cams, const int32_t* cam_fisheye, const double* cam_k, const double* cam_dist,
                   int32_t n_pairs, const int32_t* pair_a, const int32_t* pair_b, const double* pair_Rt, int64_t n_obs,
                   const int32_t* obs_cam, const int64_t* obs_key, const double* obs_px, int32_t min_common,
                   double* rmse_out, int64_t* count_out, CbTriStats* stats, int device, void* stream) {
  if (n_cams <= 0 || !cam_fisheye || !cam_k || !cam_dist || n_pairs < 0 || n_obs < 0 || n_obs > 0x7fffffffLL ||
      (n_pairs > 0 && (!pair_a || !pair_b || !pair_Rt || !rmse_out || !count_out)) ||
      (n_obs > 0 && (!obs_cam || !obs_key || !obs_px))) {
    g_last_error = "cb_stereo_rmse: bad argument";
    return CB_E_INVALID;
  }
  CB_TRY(select_device(device));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  const double nan = std::nan("");
  for (int p = 0; p < n_pairs; ++p) { rmse_out[p] = nan; count_out[p] = 0; }
  if (n_pairs == 0 || n_obs == 0) return CB_OK;
  const long long launches0 = g_launches.load();
  cudaStream_t st = (cudaStream_t)stream;
  ScopedFree sf;
  const int n = (int)n_obs;
  std::vector<int> pair_of((size_t)n_cams * n_cams, -1);
  for (int p = 0; p < n_pairs; ++p) {
    const int a = pair_a[p], b = pair_b[p];
    if (a < 0 || b < 0 || a >= n_cams || b >= n_cams || a >= b) {
      g_last_error = "cb_stereo_rmse: pairs must satisfy 0 <= a < b < n_cams";
      return CB_E_INVALID;
    }
    pair_of[(size_t)a * n_cams + b] = p;
  }
  cudaEvent_t ev[4];
  for (auto& e : ev) CB_CUDA(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 4; ++i) cudaEventDestroy(e[i]); } } evg{ev};
  CB_CUDA(cudaEventRecord(ev[0], st));
  const int* d_cam = nullptr;
  const long long* d_key = nullptr;
  const int* d_pair_of = nullptr;
  const double* d_Rt = nullptr;
  CB_TRY(to_device(obs_cam, (size_t)n, 0, &d_cam, sf, st));
  CB_TRY(to_device((const long long*)obs_key, (size_t)n, 0, &d_key, sf, st));
  CB_TRY(to_device(pair_of.data(), pair_of.size(), 0, &d_pair_of, sf, st));
  CB_TRY(to_device(pair_Rt, 12 * (size_t)n_pairs, 0, &d_Rt, sf, st));
  CB_TRY(validate_rows(d_cam, d_key, n, n_cams, st, "cb_stereo_rmse"));
  double* d_norm = nullptr;
  CB_TRY(upload_undistorted(n_cams, cam_fisheye, cam_k, cam_dist, n, d_cam, obs_px, sf, st, &d_norm));
  int *d_rows = nullptr, *d_start = nullptr, n_groups = 0;
  CB_TRY(group_by_key(d_key, n, st, sf, &d_rows, &d_start, &n_groups));
  CB_CUDA(cudaEventRecord(ev[1], st));
  // slots per group, exclusive scan
  long long *d_nslots = nullptr, *d_slot_start = nullptr;
  CB_TRY(dalloc(&d_nslots, (size_t)n_groups + 1)); sf.dev.push_back(d_nslots);
  CB_TRY(dalloc(&d_slot_start, (size_t)n_groups + 1)); sf.dev.push_back(d_slot_start);
  CB_CUDA(cudaMemsetAsync(d_nslots, 0, sizeof(long long) * ((size_t)n_groups + 1), st));
  CB_LAUNCH(cb::stereo_slots_kernel, cdiv(n_groups, 256), 256, 0, st, d_start, n_groups, d_nslots);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, d_nslots, d_slot_start, n_groups + 1, st);
  void* d_tmp = nullptr;
  CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tb, 16))); sf.dev.push_back(d_tmp);
  CB_CUDA(cub::DeviceScan::ExclusiveSum(d_tmp, tb, d_nslots, d_slot_start, n_groups + 1, st));
  g_launches.fetch_add(2);
  long long total = 0;
  CB_CUDA(cudaMemcpyAsync(&total, d_slot_start + n_groups, sizeof(long long), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  if (total > 0x7fffffffLL) { g_last_error = "cb_stereo_rmse: more than 2^31 observation pairs"; return CB_E_UNSUPPORTED; }
  if (total == 0) return CB_OK;
  const int m = (int)total;
  int *d_k = nullptr, *d_ks = nullptr;
  double *d_v = nullptr, *d_vs = nullptr;
  CB_TRY(dalloc(&d_k, (size_t)m)); sf.dev.push_back(d_k);
  CB_TRY(dalloc(&d_ks, (size_t)m)); sf.dev.push_back(d_ks);
  CB_TRY(dalloc(&d_v, (size_t)m)); sf.dev.push_back(d_v);
  CB_TRY(dalloc(&d_vs, (size_t)m)); sf.dev.push_back(d_vs);
  CB_CUDA(cudaEventRecord(ev[2], st));
  const int lanes = (n / std::max(n_groups, 1) > 12) ? 32 : 8;
  if (lanes == 32)
    CB_LAUNCH(cb::stereo_pairs_kernel<32>, cdiv((long long)n_groups * 32, cb::BS_THREADS), cb::BS_THREADS, 0, st, d_start, d_rows,
              d_cam, (const double*)d_norm, n_groups, (const long long*)d_slot_start, (int)n_cams, d_pair_of, d_Rt, (int)n_pairs, d_k, d_v);
  else
    CB_LAUNCH(cb::stereo_pairs_kernel<8>, cdiv((long long)n_groups * 8, cb::BS_THREADS), cb::BS_THREADS, 0, st, d_start, d_rows,
              d_cam, (const double*)d_norm, n_groups, (const long long*)d_slot_start, (int)n_cams, d_pair_of, d_Rt, (int)n_pairs, d_k, d_v);
  CB_CUDA(cudaGetLastError());
  CB_CUDA(cudaEventRecord(ev[3], st));
  // stable sort by pair id, then one segmented sum per pair (fixed order => reproducible sums)
  size_t tb2 = 0, tb3 = 0;
  const int kbits = bits_for((unsigned long long)n_pairs);
  cub::DeviceRadixSort::SortPairs(nullptr, tb2, d_k, d_ks, d_v, d_vs, m, 0, kbits, st);
  int *d_uk = nullptr, *d_nruns = nullptr;
  double* d_sum = nullptr;
  CB_TRY(dalloc(&d_uk, (size_t)n_pairs + 2)); sf.dev.push_back(d_uk);
  CB_TRY(dalloc(&d_sum, (size_t)n_pairs + 2)); sf.dev.push_back(d_sum);
  CB_TRY(dalloc(&d_nruns, 1)); sf.dev.push_back(d_nruns);
  cub::DeviceReduce::ReduceByKey(nullptr, tb3, d_ks, d_uk, d_vs, d_sum, d_nruns, cub::Sum(), m, st);
  void* d_tmp2 = nullptr;
  CB_TRY(cached_malloc(&d_tmp2, std::max<size_t>(std::max(tb2, tb3), 16))); sf.dev.push_back(d_tmp2);
  size_t tbs = std::max(tb2, tb3);
  CB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp2, tbs, d_k, d_ks, d_v, d_vs, m, 0, kbits, st));
  CB_CUDA(cub::DeviceReduce::ReduceByKey(d_tmp2, tbs, d_ks, d_uk, d_vs, d_sum, d_nruns, cub::Sum(), m, st));
  g_launches.fetch_add(6);
  // counts per pair: run lengths of the sorted keys (same run order as the segmented sums)
  int *d_uk2 = nullptr, *d_len = nullptr;
  CB_TRY(dalloc(&d_uk2, (size_t)n_pairs + 2)); sf.dev.push_back(d_uk2);
  CB_TRY(dalloc(&d_len, (size_t)n_pairs + 2)); sf.dev.push_back(d_len);
  size_t tb4 = 0;
  cub::DeviceRunLengthEncode::Encode(nullptr, tb4, d_ks, d_uk2, d_len, d_nruns, m, st);
  void* d_tmp3 = nullptr;
  CB_TRY(cached_malloc(&d_tmp3, std::max<size_t>(tb4, 16))); sf.dev.push_back(d_tmp3);
  std::vector<int> uk((size_t)n_pairs + 2), len((size_t)n_pairs + 2);
  std::vector<double> sums((size_t)n_pairs + 2);
  int nruns = 0;
  CB_CUDA(cudaMemcpyAsync(&nruns, d_nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(uk.data(), d_uk, sizeof(int) * ((size_t)n_pairs + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(sums.data(), d_sum, sizeof(double) * ((size_t)n_pairs + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cub::DeviceRunLengthEncode::Encode(d_tmp3, tb4, d_ks, d_uk2, d_len, d_nruns, m, st));
  g_launches.fetch_add(2);
  CB_CUDA(cudaMemcpyAsync(len.data(), d_len, sizeof(int) * ((size_t)n_pairs + 1), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  for (int r = 0; r < nruns; ++r) {
    const int pid = uk[r];
    if (pid < 0 || pid >= n_pairs) continue;
    const long long cnt = len[r];
    count_out[pid] = cnt;
    if (cnt >= min_common) rmse_out[pid] = std::sqrt(sums[r] / (2.0 * (double)cnt));  // mean over the 2N stacked rows
  }
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[0], ev[1]); stats->group_ms = ms;
    cudaEventElapsedTime(&ms, ev[2], ev[3]); stats->dlt_ms = ms;
    cudaEventElapsedTime(&ms, ev[0], ev[3]); stats->total_ms = ms;
    stats->kernel_launches = (int)(g_launches.load() - launches0);
  }
  return CB_OK;
}

int cb_relative_pose_network(int32_t n_groups, int32_t n_frames, const int32_t* frame_start, const int32_t* cam_id,
                             const int32_t* cam_pos, const double* R, const double* t, double rot_mult, double tr_mult,
                             int32_t max_pairs, int32_t* n_pairs_out, int32_t* pair_a, int32_t* pair_b, double* R_out,
                             double* t_out, int64_t* count_out, int64_t n_rel, uint8_t* rel_valid, uint8_t* rel_keep,
                             CbTriStats* stats, int device, void* stream) {
  if (n_groups < 0 || n_frames < 0 || !n_pairs_out || max_pairs < 0 ||
      (n_groups > 0 && (!frame_start || !cam_id || !cam_pos || !R || !t)) ||
      (max_pairs > 0 && (!pair_a || !pair_b || !R_out || !t_out || !count_out))) {
    g_last_error = "cb_relative_pose_network: bad argument";
    return CB_E_INVALID;
  }
  *n_pairs_out = 0;
  if (stats) std::memset(stats, 0, sizeof(*stats));
  // combinations per frame group (host: n_frames + 1 integers)
  std::vector<long long> pair_off((size_t)n_frames + 1, 0);
  int max_id = 0;
  for (int f = 0; f < n_frames; ++f) {
    const long long sz = (long long)frame_start[f + 1] - frame_start[f];
    if (sz < 0 || frame_start[f] < 0 || frame_start[f + 1] > n_groups) {
      g_last_error = "cb_relative_pose_network: frame_start must be non-decreasing within [0, n_groups]";
      return CB_E_INVALID;
    }
    pair_off[(size_t)f + 1] = pair_off[(size_t)f] + sz * (sz - 1) / 2;
  }
  for (int g = 0; g < n_groups; ++g) {
    if (cam_id[g] < 0) { g_last_error = "cb_relative_pose_network: negative camera id"; return CB_E_INVALID; }
    max_id = std::max(max_id, cam_id[g]);
  }
  const long long M = pair_off[(size_t)n_frames];
  if ((rel_valid || rel_keep) && n_rel != M) {
    g_last_error = "cb_relative_pose_network: n_rel must equal the number of combinations, " + std::to_string(M);
    return CB_E_INVALID;
  }
  if (M == 0) return CB_OK;
  if (M > 0x7fffffffLL) { g_last_error = "cb_relative_pose_network: more than 2^31 relative poses"; return CB_E_UNSUPPORTED; }
  const unsigned span = (unsigned)max_id + 1u;
  if ((unsigned long long)span * span >= 0xffffffffull) { g_last_error = "cb_relative_pose_network: camera ids too large"; return CB_E_UNSUPPORTED; }
  CB_TRY(select_device(device));
  const long long launches0 = g_launches.load();
  cudaStream_t st = (cudaStream_t)stream;
  ScopedFree sf;
  cudaEvent_t ev[3];
  for (auto& e : ev) CB_CUDA(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 3; ++i) cudaEventDestroy(e[i]); } } evg{ev};
  CB_CUDA(cudaEventRecord(ev[0], st));
  const long long* d_pair_off = nullptr;
  const int *d_fs = nullptr, *d_id = nullptr, *d_pos = nullptr;
  const double *d_R = nullptr, *d_t = nullptr;
  CB_TRY(to_device(pair_off.data(), pair_off.size(), 0, &d_pair_off, sf, st));
  CB_TRY(to_device(frame_start, (size_t)n_frames + 1, 0, &d_fs, sf, st));
  CB_TRY(to_device(cam_id, (size_t)n_groups, 0, &d_id, sf, st));
  CB_TRY(to_device(cam_pos, (size_t)n_groups, 0, &d_pos, sf, st));
  CB_TRY(to_device(R, 9 * (size_t)n_groups, 0, &d_R, sf, st));
  CB_TRY(to_device(t, 3 * (size_t)n_groups, 0, &d_t, sf, st));
  const size_t m = (size_t)M;
  unsigned *d_key = nullptr, *d_idx = nullptr, *d_key_s = nullptr, *d_perm = nullptr;
  double *d_Rr = nullptr, *d_tr = nullptr, *d_q = nullptr, *d_tm = nullptr;
  unsigned char *d_valid = nullptr, *d_keep = nullptr;
  CB_TRY(dalloc(&d_key, m)); sf.dev.push_back(d_key);
  CB_TRY(dalloc(&d_idx, m)); sf.dev.push_back(d_idx);
  CB_TRY(dalloc(&d_key_s, m)); sf.dev.push_back(d_key_s);
  CB_TRY(dalloc(&d_perm, m)); sf.dev.push_back(d_perm);
  CB_TRY(dalloc(&d_Rr, 9 * m)); sf.dev.push_back(d_Rr);
  CB_TRY(dalloc(&d_tr, 3 * m)); sf.dev.push_back(d_tr);
  CB_TRY(dalloc(&d_q, 4 * m)); sf.dev.push_back(d_q);
  CB_TRY(dalloc(&d_tm, m)); sf.dev.push_back(d_tm);
  if (rel_valid) { CB_TRY(dalloc(&d_valid, m)); sf.dev.push_back(d_valid); }
  if (rel_keep) {
    CB_TRY(dalloc(&d_keep, m)); sf.dev.push_back(d_keep);
    CB_CUDA(cudaMemsetAsync(d_keep, 0, m, st));
  }
  CB_LAUNCH(cb::rel_pose_kernel, cdiv(M, 256), 256, 0, st, d_pair_off, d_fs, (int)n_frames, M, d_id, d_pos, d_R, d_t, span,
            d_key, d_idx, d_Rr, d_tr, d_q, d_tm, d_valid);
  // stable sort by pair key; rows that were not formed / are not finite carry key span^2 and end up last
  const int kbits = bits_for((unsigned long long)span * span + 1ull);
  const int max_runs = (int)std::min<long long>(M, (long long)span * (span - 1) / 2 + 1) + 1;
  unsigned* d_uk = nullptr;
  int *d_len = nullptr, *d_nruns = nullptr;
  CB_TRY(dalloc(&d_uk, (size_t)max_runs)); sf.dev.push_back(d_uk);
  CB_TRY(dalloc(&d_len, (size_t)max_runs)); sf.dev.push_back(d_len);
  CB_TRY(dalloc(&d_nruns, 1)); sf.dev.push_back(d_nruns);
  size_t tb1 = 0, tb2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb1, d_key, d_key_s, d_idx, d_perm, (int)M, 0, kbits, st);
  cub::DeviceRunLengthEncode::Encode(nullptr, tb2, d_key_s, d_uk, d_len, d_nruns, (int)M, st);
  void* d_tmp = nullptr;
  size_t tb = std::max(tb1, tb2);
  CB_TRY(cached_malloc(&d_tmp, std::max<size_t>(tb, 16))); sf.dev.push_back(d_tmp);
  CB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_key, d_key_s, d_idx, d_perm, (int)M, 0, kbits, st));
  tb = std::max(tb1, tb2);
  CB_CUDA(cub::DeviceRunLengthEncode::Encode(d_tmp, tb, d_key_s, d_uk, d_len, d_nruns, (int)M, st));
  g_launches.fetch_add(6);
  int nruns = 0;
  CB_CUDA(cudaMemcpyAsync(&nruns, d_nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  std::vector<unsigned> uk((size_t)std::max(nruns, 1));
  std::vector<int> len((size_t)std::max(nruns, 1));
  CB_CUDA(cudaMemcpyAsync(uk.data(), d_uk, sizeof(unsigned) * (size_t)nruns, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(len.data(), d_len, sizeof(int) * (size_t)nruns, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  int n_seg = nruns;
  if (n_seg > 0 && uk[(size_t)n_seg - 1] == span * span) --n_seg;  // the run of unformed / non-finite rows
  if (rel_valid) CB_CUDA(cudaMemcpyAsync(rel_valid, d_valid, m, cudaMemcpyDeviceToHost, st));
  if (n_seg == 0) {
    if (rel_keep) std::memset(rel_keep, 0, m);
    CB_CUDA(cudaStreamSynchronize(st));
    return CB_OK;
  }
  if (n_seg > max_pairs) {
    g_last_error = "cb_relative_pose_network: " + std::to_string(n_seg) + " camera pairs, max_pairs is " + std::to_string(max_pairs);
    return CB_E_INVALID;
  }
  std::vector<int> seg_off((size_t)n_seg + 1, 0);
  for (int s2 = 0; s2 < n_seg; ++s2) seg_off[(size_t)s2 + 1] = seg_off[(size_t)s2] + len[(size_t)s2];
  const long long Mv = seg_off[(size_t)n_seg];
  const int* d_off = nullptr;
  CB_TRY(to_device(seg_off.data(), seg_off.size(), 0, &d_off, sf, st));
  const size_t mv = (size_t)Mv;
  double *d_Rs = nullptr, *d_ts = nullptr, *d_qs = nullptr, *d_tms = nullptr, *d_sorted = nullptr, *d_ang = nullptr;
  int* d_seg = nullptr;
  unsigned char* d_ok = nullptr;
  CB_TRY(dalloc(&d_Rs, 9 * mv)); sf.dev.push_back(d_Rs);
  CB_TRY(dalloc(&d_ts, 3 * mv)); sf.dev.push_back(d_ts);
  CB_TRY(dalloc(&d_qs, 4 * mv)); sf.dev.push_back(d_qs);
  CB_TRY(dalloc(&d_tms, mv)); sf.dev.push_back(d_tms);
  CB_TRY(dalloc(&d_sorted, mv)); sf.dev.push_back(d_sorted);
  CB_TRY(dalloc(&d_ang, mv)); sf.dev.push_back(d_ang);
  CB_TRY(dalloc(&d_seg, mv)); sf.dev.push_back(d_seg);
  CB_TRY(dalloc(&d_ok, mv)); sf.dev.push_back(d_ok);
  double *d_Rm = nullptr, *d_tmn = nullptr, *d_q13 = nullptr;
  long long* d_cnt = nullptr;
  CB_TRY(dalloc(&d_Rm, 9 * (size_t)n_seg)); sf.dev.push_back(d_Rm);
  CB_TRY(dalloc(&d_tmn, 3 * (size_t)n_seg)); sf.dev.push_back(d_tmn);
  CB_TRY(dalloc(&d_q13, 4 * (size_t)n_seg)); sf.dev.push_back(d_q13);
  CB_TRY(dalloc(&d_cnt, (size_t)n_seg)); sf.dev.push_back(d_cnt);
  CB_LAUNCH(cb::rel_gather_kernel, cdiv(Mv, 256), 256, 0, st, (const unsigned*)d_perm, Mv, (const double*)d_Rr,
            (const double*)d_tr, (const double*)d_q, (const double*)d_tm, d_Rs, d_ts, d_qs, d_tms);
  CB_LAUNCH(cb::seg_fill_kernel, n_seg, 128, 0, st, d_off, n_seg, d_seg);
  CB_CUDA(cudaEventRecord(ev[1], st));
  // quartiles of |t| per pair
  size_t tb3 = 0;
  cub::DeviceSegmentedSort::SortKeys(nullptr, tb3, (const double*)d_tms, d_sorted, (int)Mv, n_seg, d_off, d_off + 1, st);
  void* d_tmp2 = nullptr;
  CB_TRY(cached_malloc(&d_tmp2, std::max<size_t>(tb3, 16))); sf.dev.push_back(d_tmp2);
  CB_CUDA(cub::DeviceSegmentedSort::SortKeys(d_tmp2, tb3, (const double*)d_tms, d_sorted, (int)Mv, n_seg, d_off, d_off + 1, st));
  CB_LAUNCH(cb::seg_quartile_kernel, cdiv(n_seg, 128), 128, 0, st, (const double*)d_sorted, d_off, n_seg, d_q13, d_q13 + n_seg);
  // mean rotation per pair, angle of every sample to it, quartiles of the angle
  CB_LAUNCH(cb::quat_average_kernel, n_seg, cb::REL_THREADS, 0, st, d_off, n_seg, (const double*)d_qs, (const double*)d_ts,
            (const double*)d_Rs, (const unsigned char*)nullptr, d_Rm, d_tmn, d_cnt);
  CB_LAUNCH(cb::rel_angle_kernel, cdiv(Mv, 256), 256, 0, st, (const double*)d_Rs, (const int*)d_seg, (const double*)d_Rm, Mv, d_ang);
  CB_CUDA(cub::DeviceSegmentedSort::SortKeys(d_tmp2, tb3, (const double*)d_ang, d_sorted, (int)Mv, n_seg, d_off, d_off + 1, st));
  CB_LAUNCH(cb::seg_quartile_kernel, cdiv(n_seg, 128), 128, 0, st, (const double*)d_sorted, d_off, n_seg, d_q13 + 2 * (size_t)n_seg,
            d_q13 + 3 * (size_t)n_seg);
  g_launches.fetch_add(4);
  CB_LAUNCH(cb::rel_flag_kernel, cdiv(Mv, 256), 256, 0, st, (const int*)d_seg, d_off, Mv, (const double*)d_tms,
            (const double*)d_ang, (const double*)d_q13, (const double*)(d_q13 + n_seg), (const double*)(d_q13 + 2 * (size_t)n_seg),
            (const double*)(d_q13 + 3 * (size_t)n_seg), rot_mult, tr_mult, (const unsigned*)d_perm, d_ok, d_keep);
  // aggregate the survivors
  CB_LAUNCH(cb::quat_average_kernel, n_seg, cb::REL_THREADS, 0, st, d_off, n_seg, (const double*)d_qs, (const double*)d_ts,
            (const double*)d_Rs, (const unsigned char*)d_ok, d_Rm, d_tmn, d_cnt);
  CB_CUDA(cudaEventRecord(ev[2], st));
  std::vector<double> hR(9 * (size_t)n_seg), ht(3 * (size_t)n_seg);
  std::vector<long long> hc((size_t)n_seg);
  CB_CUDA(cudaMemcpyAsync(hR.data(), d_Rm, sizeof(double) * hR.size(), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(ht.data(), d_tmn, sizeof(double) * ht.size(), cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaMemcpyAsync(hc.data(), d_cnt, sizeof(long long) * hc.size(), cudaMemcpyDeviceToHost, st));
  if (rel_keep) CB_CUDA(cudaMemcpyAsync(rel_keep, d_keep, m, cudaMemcpyDeviceToHost, st));
  CB_CUDA(cudaStreamSynchronize(st));
  int np = 0;
  for (int s2 = 0; s2 < n_seg; ++s2) {
    if (hc[(size_t)s2] <= 0) continue;  // every sample rejected
    pair_a[np] = (int32_t)(uk[(size_t)s2] / span);
    pair_b[np] = (int32_t)(uk[(size_t)s2] % span);
    std::memcpy(R_out + 9 * (size_t)np, &hR[9 * (size_t)s2], 9 * sizeof(double));
    std::memcpy(t_out + 3 * (size_t)np, &ht[3 * (size_t)s2], 3 * sizeof(double));
    count_out[np] = hc[(size_t)s2];
    ++np;
  }
  *n_pairs_out = np;
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[0], ev[1]); stats->group_ms = ms;
    cudaEventElapsedTime(&ms, ev[1], ev[2]); stats->dlt_ms = ms;
    cudaEventElapsedTime(&ms, ev[0], ev[2]); stats->total_ms = ms;
    stats->kernel_launches = (int)(g_launches.load() - launches0);
  }
  return CB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// numeric CSV tables at the boundary (SURVEY.md §8(f) rank 4); see cb_io.h
// ------------------------------------------------------------------------------------------
#include "cb_io.h"

namespace {
struct MappedFile {
  const char* data = nullptr;
  size_t size = 0;
  int fd = -1;
  ~MappedFile() {
    if (data && size) munmap((void*)data, size);
    if (fd >= 0) close(fd);
  }
  int open_ro(const char* path) {
    fd = ::open(path, O_RDONLY);
    if (fd < 0) { g_last_error = std::string("cannot open ") + path + ": " + std::strerror(errno); return CB_E_INVALID; }
    struct stat sb;
    if (fstat(fd, &sb) != 0) { g_last_error = std::string("fstat ") + path; return CB_E_INVALID; }
    size = (size_t)sb.st_size;
    if (size == 0) return CB_OK;
    void* m = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (m == MAP_FAILED) { g_last_error = std::string("mmap ") + path + ": " + std::strerror(errno); data = nullptr; return CB_E_INVALID; }
    data = (const char*)m;
    return CB_OK;
  }
};

// start of the body (after the header line) or size
size_t csv_body_start(const MappedFile& f) {
  const char* nl = (const char*)memchr(f.data, '\n', f.size);
  return nl ? (size_t)(nl - f.data) + 1 : f.size;
}

// line-aligned chunk boundaries of [b0, size)
std::vector<size_t> csv_chunks(const MappedFile& f, size_t b0, int n) {
  std::vector<size_t> cut{b0};
  for (int t = 1; t < n; ++t) {
    size_t pos = b0 + (f.size - b0) * (size_t)t / (size_t)n;
    if (pos <= cut.back()) continue;
    const char* nl = (const char*)memchr(f.data + pos, '\n', f.size - pos);
    if (!nl) break;
    pos = (size_t)(nl - f.data) + 1;
    if (pos > cut.back() && pos < f.size) cut.push_back(pos);
  }
  cut.push_back(f.size);
  return cut;
}

inline bool blank_line(const char* b, const char* e) {
  for (const char* q = b; q < e; ++q)
    if (*q != '\r' && *q != ' ') return false;
  return true;
}
}  // namespace

extern "C" {

int cb_csv_write_numeric(const char* path, const char* header, int64_t n_rows, int32_t n_cols, const int32_t* col_kind,
                         const void* const* col_data, int32_t n_threads) {
  if (!path || !header || n_rows < 0 || n_cols <= 0 || !col_kind || !col_data) { g_last_error = "cb_csv_write_numeric: bad argument"; return CB_E_INVALID; }
  const int nt = cbio::n_workers(n_threads, (size_t)n_rows, 20000);
  std::vector<std::string> parts((size_t)nt);
  cbio::parallel_for(nt, [&](int t) {
    const int64_t r0 = n_rows * t / nt, r1 = n_rows * (t + 1) / nt;
    std::string& out = parts[(size_t)t];
    out.reserve((size_t)(r1 - r0) * (size_t)n_cols * 12);
    for (int64_t r = r0; r < r1; ++r) {
      for (int c = 0; c < n_cols; ++c) {
        if (c) out.push_back(',');
        if (col_kind[c] == 0) cbio::append_i64(out, ((const long long*)col_data[c])[r]);
        else cbio::append_f6(out, ((const double*)col_data[c])[r]);
      }
      out.push_back('\n');
    }
  });
  // temp file + fsync + atomic rename, as persistence._safe_write_csv (persistence.py:27-41)
  const std::string tmp = std::string(path) + ".tmp";
  const int fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) { g_last_error = "cannot create " + tmp + ": " + std::strerror(errno); return CB_E_INVALID; }
  auto write_all = [&](const char* p, size_t n) {
    while (n) {
      const ssize_t w = ::write(fd, p, n);
      if (w < 0) { if (errno == EINTR) continue; return false; }
      p += w; n -= (size_t)w;
    }
    return true;
  };
  bool ok = write_all(header, std::strlen(header)) && write_all("\n", 1);
  for (auto& s : parts) ok = ok && write_all(s.data(), s.size());
  ok = ok && fsync(fd) == 0;
  ::close(fd);
  if (!ok || std::rename(tmp.c_str(), path) != 0) {
    g_last_error = std::string("writing ") + path + ": " + std::strerror(errno);
    std::remove(tmp.c_str());
    return CB_E_INVALID;
  }
  return CB_OK;
}

// Host-side shard selection of a sharded solve: the observations whose point lies in [pt_lo, pt_hi), in the caller's
// order, with the point index made local.  Two passes over obs_pt by all host threads (count, then write at the prefix
// offsets); the NumPy version of the same selection (mask, flatnonzero, three fancy-index gathers) costs ~15 ms on a
// 2 M-observation list and sits inside every sharded call on every rank.
int cb_shard_select(int64_t n_obs, const int32_t* obs_cam, const int32_t* obs_pt, const double* obs_xy, int32_t pt_lo,
                    int32_t pt_hi, int64_t capacity, int64_t* n_sel_out, int64_t* sel_index, int32_t* cam_out,
                    int32_t* pt_out, double* xy_out, int32_t n_threads) {
  if (n_obs < 0 || !n_sel_out || (n_obs > 0 && (!obs_cam || !obs_pt || !obs_xy))) {
    g_last_error = "cb_shard_select: bad argument";
    return CB_E_INVALID;
  }
  const int nt = cbio::n_workers(n_threads, (size_t)n_obs, (size_t)1 << 16);
  std::vector<int64_t> cnt((size_t)nt + 1, 0);
  auto slice = [&](int t, int64_t* b, int64_t* e) { *b = n_obs * t / nt; *e = n_obs * (t + 1) / nt; };
  cbio::parallel_for(nt, [&](int t) {
    int64_t b, e, c = 0;
    slice(t, &b, &e);
    for (int64_t i = b; i < e; ++i) c += (obs_pt[i] >= pt_lo) & (obs_pt[i] < pt_hi);
    cnt[(size_t)t + 1] = c;
  });
  for (int t = 0; t < nt; ++t) cnt[(size_t)t + 1] += cnt[(size_t)t];
  *n_sel_out = cnt[(size_t)nt];
  if (!sel_index && !cam_out && !pt_out && !xy_out) return CB_OK;  // size query
  if (cnt[(size_t)nt] > capacity) {
    g_last_error = "cb_shard_select: capacity " + std::to_string(capacity) + " < " + std::to_string(cnt[(size_t)nt]) + " selected rows";
    return CB_E_INVALID;
  }
  cbio::parallel_for(nt, [&](int t) {
    int64_t b, e, o = cnt[(size_t)t];
    slice(t, &b, &e);
    for (int64_t i = b; i < e; ++i) {
      const int32_t pt = obs_pt[i];
      if (pt < pt_lo || pt >= pt_hi) continue;
      if (sel_index) sel_index[o] = i;
      if (cam_out) cam_out[o] = obs_cam[i];
      if (pt_out) pt_out[o] = pt - pt_lo;
      if (xy_out) { xy_out[2 * o] = obs_xy[2 * i]; xy_out[2 * o + 1] = obs_xy[2 * i + 1]; }
      ++o;
    }
  });
  return CB_OK;
}

int cb_csv_scan(const char* path, int64_t* n_rows, int32_t* n_cols) {
  if (!path || !n_rows || !n_cols) { g_last_error = "cb_csv_scan: bad argument"; return CB_E_INVALID; }
  MappedFile f;
  CB_TRY(f.open_ro(path));
  *n_rows = 0; *n_cols = 0;
  if (f.size == 0) return CB_OK;
  const size_t b0 = csv_body_start(f);
  int cols = 1;
  for (size_t i = 0; i + 1 < b0 || (i < b0 && f.data[i] != '\n'); ++i)
    if (f.data[i] == ',') ++cols;
  *n_cols = cols;
  const int nt = cbio::n_workers(0, f.size - b0, 1 << 20);
  const std::vector<size_t> cut = csv_chunks(f, b0, nt);
  std::vector<long long> cnt(cut.size(), 0);
  cbio::parallel_for((int)cut.size() - 1, [&](int t) {
    const char *p = f.data + cut[t], *e = f.data + cut[t + 1];
    long long c = 0;
    while (p < e) {
      const char* nl = (const char*)memchr(p, '\n', (size_t)(e - p));
      const char* le = nl ? nl : e;
      if (!blank_line(p, le)) ++c;
      p = nl ? nl + 1 : e;
    }
    cnt[(size_t)t] = c;
  });
  for (long long c : cnt) *n_rows += c;
  return CB_OK;
}

int cb_csv_parse_numeric(const char* path, int64_t n_rows, int32_t n_cols, double* out, int32_t* col_all_int,
                         int32_t* col_has_empty, int32_t n_threads) {
  if (!path || n_rows < 0 || n_cols <= 0 || !out || !col_all_int || !col_has_empty) { g_last_error = "cb_csv_parse_numeric: bad argument"; return CB_E_INVALID; }
  MappedFile f;
  CB_TRY(f.open_ro(path));
  for (int c = 0; c < n_cols; ++c) { col_all_int[c] = 1; col_has_empty[c] = 0; }
  if (f.size == 0 || n_rows == 0) return CB_OK;
  const size_t b0 = csv_body_start(f);
  const int nt = cbio::n_workers(n_threads, f.size - b0, 1 << 20);
  const std::vector<size_t> cut = csv_chunks(f, b0, nt);
  const int nc = (int)cut.size() - 1;
  // rows per chunk -> row offsets
  std::vector<long long> cnt((size_t)nc + 1, 0);
  cbio::parallel_for(nc, [&](int t) {
    const char *p = f.data + cut[t], *e = f.data + cut[t + 1];
    long long c = 0;
    while (p < e) {
      const char* nl = (const char*)memchr(p, '\n', (size_t)(e - p));
      const char* le = nl ? nl : e;
      if (!blank_line(p, le)) ++c;
      p = nl ? nl + 1 : e;
    }
    cnt[(size_t)t + 1] = c;
  });
  for (int t = 0; t < nc; ++t) cnt[(size_t)t + 1] += cnt[(size_t)t];
  if (cnt[(size_t)nc] != n_rows) { g_last_error = "cb_csv_parse_numeric: row count changed since cb_csv_scan"; return CB_E_INVALID; }
  std::vector<std::vector<int>> all_int((size_t)nc, std::vector<int>((size_t)n_cols, 1)), has_empty((size_t)nc, std::vector<int>((size_t)n_cols, 0));
  std::vector<long long> bad((size_t)nc, -1);
  const double nan = std::nan("");
  cbio::parallel_for(nc, [&](int t) {
    const char *p = f.data + cut[t], *e = f.data + cut[t + 1];
    long long row = cnt[(size_t)t];
    while (p < e) {
      const char* nl = (const char*)memchr(p, '\n', (size_t)(e - p));
      const char* le = nl ? nl : e;
      const char* next = nl ? nl + 1 : e;
      if (le > p && le[-1] == '\r') --le;
      if (blank_line(p, le)) { p = next; continue; }
      const char* q = p;
      for (int c = 0; c < n_cols; ++c) {
        const char* fe = (const char*)memchr(q, ',', (size_t)(le - q));
        if (!fe || c == n_cols - 1) fe = (c == n_cols - 1) ? le : (fe ? fe : le);
        double v = nan;
        if (fe == q) {
          has_empty[(size_t)t][(size_t)c] = 1;
          all_int[(size_t)t][(size_t)c] = 0;
        } else {
          const char* endp = cbio::precise_xstrtod(q, fe, &v);
          if (endp != fe) {
            // nan / inf spellings pandas accepts
            std::string tok(q, fe);
            if (tok == "nan" || tok == "NaN" || tok == "NA" || tok == "null" || tok == "NULL" || tok == "N/A" || tok == "n/a") { v = nan; has_empty[(size_t)t][(size_t)c] = 1; }
            else if (tok == "inf" || tok == "Inf" || tok == "+inf") v = INFINITY;
            else if (tok == "-inf" || tok == "-Inf") v = -INFINITY;
            else { bad[(size_t)t] = row; return; }
            all_int[(size_t)t][(size_t)c] = 0;
          } else {
            for (const char* z = q; z < fe; ++z)
              if (!((*z >= '0' && *z <= '9') || ((*z == '-' || *z == '+') && z == q))) { all_int[(size_t)t][(size_t)c] = 0; break; }
          }
        }
        out[(size_t)c * (size_t)n_rows + (size_t)row] = v;
        q = (fe < le) ? fe + 1 : le;
        if (fe >= le && c < n_cols - 1) {  // short row: remaining fields empty
          for (int c2 = c + 1; c2 < n_cols; ++c2) {
            out[(size_t)c2 * (size_t)n_rows + (size_t)row] = nan;
            has_empty[(size_t)t][(size_t)c2] = 1; all_int[(size_t)t][(size_t)c2] = 0;
          }
          break;
        }
      }
      ++row;
      p = next;
    }
  });
  for (int t = 0; t < nc; ++t) {
    if (bad[(size_t)t] >= 0) { g_last_error = "cb_csv_parse_numeric: non-numeric field in data row " + std::to_string(bad[(size_t)t]); return CB_E_INVALID; }
    for (int c = 0; c < n_cols; ++c) {
      if (!all_int[(size_t)t][(size_t)c]) col_all_int[c] = 0;
      if (has_empty[(size_t)t][(size_t)c]) col_has_empty[c] = 1;
    }
  }
  return CB_OK;
}

}  // extern "C"
