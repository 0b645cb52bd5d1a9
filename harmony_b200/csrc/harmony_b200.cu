// harmony_b200.cu — host side of libharmony_b200.so: the C ABI of include/harmony_b200.h on top of the
// kernels in kernels.cuh.  One hb_handle == one instance of the reference's `harmony` class
// (/root/reference/src/harmony.h:20-70).  sm_90a (H100) only; there is no CPU path.
#include "../../include/harmony_b200.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <numeric>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "kernels.cuh"
#include "io.cuh"
#include "update_per_step.cuh"
#include "update_two_pass.cuh"
#include "update_single_pass.cuh"
#include "assign_tc3.cuh"
#include "logits_tc.cuh"
#include "logits_wide.cuh"
#include "apply_tc3.cuh"
#include "stats_tc3.cuh"

namespace {

using namespace hb;

// ---- NCCL through dlopen (the process usually already holds torch's libnccl.so.2) ---------------
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
} g_nccl;

bool load_nccl(std::string* why) {
  if (g_nccl.ok) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    g_nccl.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.lib) break;
  }
  if (!g_nccl.lib) {
    if (why) *why = "cannot dlopen libnccl.so.2";
    return false;
  }
#define L(sym) *(void**)(&g_nccl.sym) = dlsym(g_nccl.lib, "nccl" #sym)
  L(GetUniqueId);
  L(CommInitRank);
  L(AllReduce);
  L(AllGather);
  L(CommDestroy);
  L(GetErrorString);
#undef L
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.AllGather && g_nccl.CommDestroy;
  if (!g_nccl.ok && why) *why = "libnccl lacks required symbols";
  return g_nccl.ok;
}

// one NCCL communicator per (device, rank, world) is kept for the life of the process and shared by every
// handle that asks for it with a NULL id (communicator set-up costs ~1 s; models come and go)
struct CommKey {
  int device, rank, world;
  bool operator<(const CommKey& o) const {
    return std::tie(device, rank, world) < std::tie(o.device, o.rank, o.world);
  }
};
std::map<CommKey, ncclComm_t> g_comms;

struct Region {
  double ms = 0;
  int64_t launches = 0;
};

// ---- host worker pool: widens float -> double into caller memory with several threads ---------------------
// A device -> host copy into pageable memory runs at the speed of one driver thread that also takes the page
// faults of a freshly allocated destination.  The download path (hb_get_field) instead DMA's
// floats into pinned staging and lets this pool widen + scatter them while the next chunk is in flight.
class WidenPool {
 public:
  explicit WidenPool(int nthreads) {
    for (int i = 1; i < nthreads; ++i) workers_.emplace_back([this] { run(); });
  }
  ~WidenPool() {
    {
      std::lock_guard<std::mutex> lk(m_);
      stop_ = true;
      ++gen_;
    }
    cv_job_.notify_all();
    for (auto& t : workers_) t.join();
  }
  int threads() const { return (int)workers_.size() + 1; }
  // dst[i] = (double) src[i], i < n; the caller takes part
  void widen(double* dst, const float* src, size_t n) {
    {
      std::lock_guard<std::mutex> lk(m_);
      dst_ = dst;
      src_ = src;
      n_ = n;
      next_.store(0);
      pending_ = (int)workers_.size();
      ++gen_;
    }
    cv_job_.notify_all();
    work();
    std::unique_lock<std::mutex> lk(m_);
    cv_done_.wait(lk, [this] { return pending_ == 0; });
  }

 private:
  static constexpr size_t kSlice = (size_t)1 << 18;  // elements per grab (2 MiB of doubles)
  void work() {
    for (;;) {
      const size_t i0 = next_.fetch_add(kSlice);
      if (i0 >= n_) break;
      const size_t i1 = std::min(n_, i0 + kSlice);
      for (size_t i = i0; i < i1; ++i) dst_[i] = (double)src_[i];
    }
  }
  void run() {
    uint64_t seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_job_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
      }
      work();
      {
        std::lock_guard<std::mutex> lk(m_);
        if (--pending_ == 0) cv_done_.notify_all();
      }
    }
  }
  std::vector<std::thread> workers_;
  std::mutex m_;
  std::condition_variable cv_job_, cv_done_;
  double* dst_ = nullptr;
  const float* src_ = nullptr;
  size_t n_ = 0;
  std::atomic<size_t> next_{0};
  int pending_ = 0;
  uint64_t gen_ = 0;
  bool stop_ = false;
};
WidenPool* widen_pool(int want = 0) {
  static std::mutex mk;
  static WidenPool* pool = nullptr;
  std::lock_guard<std::mutex> lk(mk);
  if (!pool) {
    int n = want;
    if (n <= 0) {
      const char* e = getenv("HB_HOST_THREADS");
      n = e ? atoi(e) : (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
    }
    pool = new WidenPool(std::max(1, n));  // lives until the process exits
  }
  return pool;
}

// Host-side phase timer for the one-off calls (HB_TRACE_HOST=1): every mark() drains the stream and prints the
// wall-clock time since the previous mark to stderr.  Off: a single branch per mark.
struct HostLap {
  cudaStream_t stream;
  const char* call;
  bool on;
  std::chrono::steady_clock::time_point t;
  HostLap(cudaStream_t s, const char* c) : stream(s), call(c), on(getenv("HB_TRACE_HOST") != nullptr) {
    if (on) t = std::chrono::steady_clock::now();
  }
  void mark(const char* what) {
    if (!on) return;
    cudaStreamSynchronize(stream);
    const auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[hb] %s: %-28s %9.3f ms\n", call, what, std::chrono::duration<double, std::milli>(now - t).count());
    t = now;
  }
};

// utils.cpp:102-108
int my_ceil(float num) {
  int inum = (int)num;
  if (num == (float)inum) return inum;
  return inum + 1;
}

// ---- kernel selection --------------------------------------------------------------------------------------
// One kernel per stage, chosen by select_kernels.  The values of UpdatePath are hb_debug_kernel_paths' numbers, those
// of Assign, ColdStart and Apply hb_debug_wide_paths'.
enum class UpdatePath { PerStep = 0, TwoPass = 1, SinglePass = 2 };
// assignment in natural order (init, legacy centroid step, cold start of the calls that do not run it in plan order):
// fused wgmma (assign_tc3.cuh), FFMA k_assign, or logits (logits_tc.cuh / logits_wide.cuh) + k_softmax_tiles
enum class Assign { FusedTc = 1, Ffma = 2, LogitsTc = 3, LogitsWide = 4 };
// cold-start assignment in the order of round 0 of the plan: fused wgmma, or logits + k_softmax_block_sums;
// None: no kernel for the shape, the cold start runs in natural order
enum class ColdStart { None = 0, FusedTc = 1, LogitsTc = 2, LogitsWide = 3 };
// ridge apply: wgmma k_apply_tc (one column range), FFMA k_ridge_apply, or k_apply_tc_cols over 128-column ranges
enum class Apply { Tc = 1, Ffma = 2, TcCols = 3 };
// native k-means initialisation: FFMA race and Lloyd steps, or both from logits with sigma = 1
enum class KmeansInit { Ffma, LogitsTc, LogitsWide };

struct KernelPaths {
  UpdatePath update = UpdatePath::PerStep;
  bool tuple_ranges = false;  // 2 J <= #SMs: the plan gives every CTA a slice of a block inside one tuple
  int k1_stages = 0;          // operand stages (1, 2) of the fused assignment kernel; 0: not fused
  Assign assign = Assign::Ffma;
  ColdStart cold = ColdStart::None;
  Apply apply = Apply::Ffma;
  KmeansInit kmeans = KmeansInit::Ffma;
};

int two_pass_nv(int KS) {
  int nv = 1;
  while (4 * UPD_LPR * nv < KS) nv <<= 1;
  return nv;
}
size_t two_pass_smem_bytes(int KS, int nb, int J) {
  const size_t tabn = (size_t)std::max(2, nb) * KS;
  const int nv = two_pass_nv(KS);
  const size_t rowbuf = (size_t)UPD_GWARPS * (upd_depth_upd(nv) + upd_depth_look(nv)) * UPD_RPW * KS;
  return sizeof(float) * ((size_t)KS + 2 * (tabn + (size_t)UPD_GWARPS * KS + 2 * (size_t)UPD_STAGE + (size_t)((J + 8) & ~3)) + rowbuf);
}

// The kernels of a shape (n: local cells, nb: update blocks); kernel_set: the HB_KS_* bits of the test hook.
// update_R runs the single-pass persistent kernel (update_single_pass.cuh) when every CTA's slice of a block can lie
// inside one covariate tuple (2 J <= #SMs), its ring fits shared memory and n KS < 2^32; else the two-pass
// persistent kernel (update_two_pass.cuh) when KS <= 256, J <= 8192 and its buffers fit shared memory; else three
// launches per block step (update_per_step.cuh).
// The other stages take their wgmma kernel where it fits, else their FFMA kernel where it fits (assign_ffma_fits,
// apply_ffma_fits, kmeans_ffma_fits), else the kernel of the wide shapes.  HB_KS_FFMA_CONTRACTIONS rules out the
// wgmma kernels, HB_KS_WIDE the wgmma and FFMA ones.  A stage that runs from logits takes k_logits_tc where it fits
// (not under HB_KS_WIDE), else the d-chunked k_logits_wide.  The plan-order cold start has no FFMA kernel: it runs
// from logits where k_logits_tc is among the wgmma kernels or the natural-order assignment runs from logits.
KernelPaths select_kernels(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set) {
  const int KS = (K + 3) & ~3, KD = (d + 7) & ~7, NP = (K + 15) & ~15;
  KernelPaths p;
  p.tuple_ranges = 2 * J <= num_sms;
  if (kernel_set & HB_KS_UPDATE_PER_STEP)
    p.update = UpdatePath::PerStep;
  else if (!(kernel_set & HB_KS_UPDATE_TWO_PASS) && p.tuple_ranges && sp_ring_rows(KS, SMEM_LIMIT) > 0 &&
           (uint64_t)n * (uint64_t)KS < (1ull << 32))
    p.update = UpdatePath::SinglePass;
  else if (KS <= 256 && J <= 8192 && two_pass_smem_bytes(KS, nb, J) <= SMEM_LIMIT)
    p.update = UpdatePath::TwoPass;
  const bool wide = kernel_set & HB_KS_WIDE;
  const bool tc = !(kernel_set & (HB_KS_FFMA_CONTRACTIONS | HB_KS_WIDE));
  const bool logits_tc = !wide && logits_tc_fits(d);
  if (tc) {
    const int ns = assign3_smem_bytes(2, KD, NP, KS) <= SMEM_LIMIT ? 2 : 1;
    if (d <= 64 && K <= 128 && assign3_smem_bytes(ns, KD, NP, KS) <= SMEM_LIMIT) p.k1_stages = ns;
  }
  if (p.k1_stages) {
    p.assign = Assign::FusedTc;
    p.cold = ColdStart::FusedTc;
  } else {
    if (wide || !assign_ffma_fits(K, d)) p.assign = logits_tc ? Assign::LogitsTc : Assign::LogitsWide;
    if ((tc && logits_tc) || p.assign != Assign::Ffma) p.cold = logits_tc ? ColdStart::LogitsTc : ColdStart::LogitsWide;
  }
  if (tc && apply_tc_fits(d))
    p.apply = Apply::Tc;  // cluster ranges of <= AP_MAXK per launch
  else if (wide || !apply_ffma_fits(K, d))
    p.apply = Apply::TcCols;
  if (tc && logits_tc && KS <= 256)
    p.kmeans = KmeansInit::LogitsTc;
  else if (wide || !kmeans_ffma_fits(K, d))
    p.kmeans = logits_tc ? KmeansInit::LogitsTc : KmeansInit::LogitsWide;
  return p;
}

// The update_R path of a cluster_cpp call of T rounds, and whether a cold-start assignment runs in the order of round
// 0 of the plan (and hands that round's removal sums to the single-pass kernel) instead of in natural order.  The
// two-pass kernel keeps its R-store rounds in a 32-bit mask: longer calls run per step, like every call with the
// legacy centroid step.
struct CallPath {
  UpdatePath update;
  bool plan_order_assign;
};
CallPath call_path(const KernelPaths& p, unsigned T, bool legacy_centroid) {
  CallPath c{p.update, false};
  if (legacy_centroid || (p.update == UpdatePath::TwoPass && T > 31)) c.update = UpdatePath::PerStep;
  c.plan_order_assign = c.update == UpdatePath::SinglePass && p.cold != ColdStart::None && T > 0;
  return c;
}

// exchange area of the persistent update kernel for sharded cells (see setup_peer_exchange)
struct XchArea {
  int device = 0, world = 0, rank = 0;
  size_t slots = 0, XH = 0, remT_floats = 0;
  float* base = nullptr;     // [inbox: slots * world * XH floats | flags: slots * world words | remT: remT_floats]
  void* peer[XCH_MAXWORLD] = {};
  unsigned epoch = 0;
  bool leased = false;
};

// Device buffers come from the device's default memory pool (stream-ordered allocator), whose release threshold
// hb_create raises to "keep everything": a model created after another one was dropped reuses the cached memory
// instead of paying cudaMalloc's OS mapping again (measured: 44 ms of a 100 ms end-to-end run at 1M cells).
// Frees keep cudaFree's contract: nothing of the device may still be using the memory.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release() {
    if (p) {
      cudaDeviceSynchronize();
      if (cudaFreeAsync(p, 0) != cudaSuccess) {
        cudaGetLastError();
        cudaFree(p);
      }
    }
    p = nullptr;
    n = 0;
  }
  cudaError_t alloc(size_t count) {
    release();
    if (count == 0) count = 1;
    cudaError_t e = cudaMallocAsync((void**)&p, count * sizeof(T), 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);  // ordered on the (idle) default stream: usable from any stream now
    if (e != cudaSuccess) {  // no pool support / pool exhausted: plain allocation
      cudaGetLastError();
      e = cudaMalloc((void**)&p, count * sizeof(T));
    }
    if (e == cudaSuccess) n = count;
    return e;
  }
};
void keep_pool_memory(int device) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  cudaGetLastError();
}

struct Plan;  // plan.cuh

}  // namespace

struct hb_handle {
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  std::string err;
  std::deque<std::string> warnings;

  // problem
  int64_t N_global = 0, cell_offset = 0, n = 0;
  bool shard_set = false;
  int d = 0, K = 0, B = 0, C = 0, J = 0;
  int KS = 0, DS = 0;  // row strides (multiples of 4 floats) of U/R/O/E and of Zo/Zc
  std::vector<int> B_vec, cov_of;
  float block_size = 0, epsilon_kmeans = 0, epsilon_harmony = 0, alpha = 0, cutoff = 0;
  unsigned max_iter_kmeans = 0, window_size = 3;
  bool lambda_estimation = false, ran_setup = false, ran_init = false;
  int verbose = 0;
  uint64_t seed = 0x5eedULL;
  int nb = 0;
  uint32_t cpb = 0;
  int half_bits = 1;
  int (*abort_cb)(void*) = nullptr;
  void* abort_user = nullptr;

  // device state
  DevBuf<float> Zo, Zc, U, R, Y, sigma, theta, Pr_b, N_b, lambda, O, E, P, Oacc, acc, S, V, Wfull, scratch, trace_d;
  DevBuf<float> ring, acc2, Psave, OEend, tmpT;  // persistent update kernel state
  DevBuf<double> obj2;
  DevBuf<unsigned> bar;
  std::unique_ptr<Plan> plan;  // update-order plan (plan.cuh)
  bool sigma_uniform = false;
  float sigma0 = 0.f;
  bool R_user_set = false;  // R was written through hb_set_field since the last assignment step
  int coop_grid = 0;
  DevBuf<double> obj_acc, stage;
  DevBuf<int> sort_perm, inv_sort, tuple_levels, cov_of_d, tile_cell0, tile_len, tile_tuple, iscratch, skipped, err_flag;
  DevBuf<int64_t> perms_d;
  DevBuf<int> tc_cell0, tc_len, tc_tuple;  // 128-cell tiles of the tensor-core kernels
  int tc_ntiles = 0;
  KernelPaths paths;             // kernels picked by hb_setup (select_kernels)
  int kernel_set = 0;            // HB_KERNEL_SET test hook (bits HB_KS_*), read by hb_setup
  bool legacy_centroid = false;  // HB_LEGACY_CENTROID_STEP: centroid update at the top of every clustering round
  DevBuf<float> Rkeep, OEkeep;   // R / O,E saved around the distance-only assignment of that step
  DevBuf<float> Ypad;            // Y padded for k_logits_wide
  DevBuf<double> objkeep;
  int ring_rows = 0;     // rows of a warp's private ring in the single-pass update kernel
  bool use_xch = false;  // sharded cells: block steps exchanged through peer memory (one cooperative launch per call)
  PeerXch xch{};
  XchArea* xarea = nullptr;  // leased exchange area (process-wide pool, see setup_peer_exchange)
  bool zc_pending_norm = false;  // Zc holds the un-normalised corrected embedding although cluster_cpp has run
  DevBuf<float> remT;    // [2][nb][J][KS] next round's removal sums per (block, tuple)
  DevBuf<float> remS;    // [nb][J][KS] sharded cells: the ranks' remT of one round, summed
  DevBuf<int> lvl_ptr, lvl_tup;  // CSR level -> tuples (+ one trailing word: B_vec[0])
  int ntiles = 0;
  int trace_cap = 0;
  std::vector<int> tuple_levels_h;  // [J][C]
  std::vector<int64_t> tuple_start_h;  // [J + 1] first sorted position of each tuple
  std::vector<int64_t> kmeans_cells;  // global cells chosen by the native initialize_centroids (test hook)

  // traces (harmony.h:55-56); values are produced on the device and pulled lazily
  int obj_count = 0;                      // objective evaluations so far (device slots)
  std::vector<float> obj_vals;            // 4 per slot, host mirror (first obj_synced slots valid)
  int obj_synced = 0;
  std::vector<int> harmony_slots;         // objective_harmony[i] = objective_kmeans[harmony_slots[i]]
  std::vector<int> kmeans_rounds;

  // multi-GPU
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;

  // instrumentation
  int64_t launches = 0;
  bool timing = false;
  std::map<std::string, Region> regions;
};

namespace {

int fail(hb_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  h->err = buf;
  return code;
}

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess) return fail(h, 10, "CUDA error %s at %s:%d", cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)
#define CKN(call)                                                                                  \
  do {                                                                                             \
    ncclResult_t r__ = (call);                                                                     \
    if (r__ != ncclSuccess)                                                                        \
      return fail(h, 11, "NCCL error %s at %s:%d", g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "?", __FILE__, __LINE__); \
  } while (0)
#define CKL()                                                                                      \
  do {                                                                                             \
    h->launches++;                                                                                 \
    cudaError_t e__ = cudaGetLastError();                                                          \
    if (e__ != cudaSuccess) return fail(h, 10, "kernel launch failed: %s at %s:%d", cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)
#define TRY(...)             \
  do {                       \
    int st__ = (__VA_ARGS__); \
    if (st__ != 0) return st__; \
  } while (0)

struct RegionScope {
  hb_handle* h;
  const char* name;
  int64_t l0;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  RegionScope(hb_handle* h_, const char* n) : h(h_), name(n), l0(h_->launches) {
    if (h->timing) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
      cudaEventRecord(e0, h->stream);
    }
  }
  ~RegionScope() {
    Region& r = h->regions[name];
    r.launches += h->launches - l0;
    if (e0) {
      cudaEventRecord(e1, h->stream);
      cudaEventSynchronize(e1);
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      r.ms += ms;
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
    }
  }
};

int grid_for(int64_t work_items, int threads, int cap) {
  int64_t g = (work_items + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

int allreduce_f(hb_handle* h, float* p, size_t count) {
  if (h->world <= 1) return 0;
  CKN(g_nccl.AllReduce(p, p, count, ncclFloat, ncclSum, h->comm, h->stream));
  return 0;
}
int allreduce_d(hb_handle* h, double* p, size_t count) {
  if (h->world <= 1) return 0;
  CKN(g_nccl.AllReduce(p, p, count, ncclDouble, ncclSum, h->comm, h->stream));
  return 0;
}

int kq_for(int K) {
  int q = (K + 31) / 32;
  int kq = 1;
  while (kq < q) kq <<= 1;
  return kq;
}

// Run-time value -> template argument: f(std::integral_constant<int, V>()) for the V of the list equal to v, whose
// status it returns; `unsupported` (formatted with K) when the list has no such V.
template <int... Vs, typename F>
int dispatch(hb_handle* h, int v, const char* unsupported, F&& f) {
  int st = 0;
  if (((v == Vs && ((st = f(std::integral_constant<int, Vs>())), true)) || ...)) return st;
  return fail(h, 2, unsupported, h->K);
}
constexpr const char* kUnsupportedK = "K = %d is not supported (K <= 1024)";
constexpr const char* kUnsupportedUpdateK = "K = %d is not supported by the persistent update kernel";

// U[i][k] = (2 / sigma_k) (z_i . y_k / |z_i| - 1) for all clusters on the tensor cores, 128 clusters per launch and d
// in chunks (logits_wide.cuh), after one pass that pads Y
int launch_logits_wide(hb_handle* h, const float* sigma, bool normalise) {
  const int KDc = (h->d + LW_DC - 1) / LW_DC * LW_DC, rows = (h->K + LW_NP - 1) / LW_NP * LW_NP;
  if (h->Ypad.n < (size_t)rows * KDc) CK(h->Ypad.alloc((size_t)rows * KDc));
  k_pad_rows<<<grid_for((int64_t)rows * KDc, 256, h->num_sms * 4), 256, 0, h->stream>>>(h->Y.p, h->Ypad.p, h->K, h->d, rows, KDc);
  CKL();
  LogitsWideArgs t{};
  t.Zc = h->Zc.p;
  t.Ypad = h->Ypad.p;
  t.sigma = sigma;
  t.U = h->U.p;
  t.n = h->n;
  t.d = h->d;
  t.K = h->K;
  t.DS = h->DS;
  t.KS = h->KS;
  t.KDc = KDc;
  t.normalise = normalise ? 1 : 0;
  const size_t smem = logits_wide_smem_bytes();
  CK(cudaFuncSetAttribute(k_logits_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((h->n + LW_TM - 1) / LW_TM, h->num_sms));
  for (t.n_off = 0; t.n_off < h->K; t.n_off += LW_NP) {
    k_logits_wide<<<grid, LW_THREADS, smem, h->stream>>>(t);
    CKL();
  }
  return 0;
}

// U[i][k] = (2 / sigma_k) (z_i . y_k / |z_i| - 1) for all clusters on the tensor cores, 64 clusters per launch
// (logits_tc.cuh), or from launch_logits_wide when `wide`; `sigma`: device array of K values
int launch_logits(hb_handle* h, const float* sigma, bool normalise, bool wide) {
  if (wide) return launch_logits_wide(h, sigma, normalise);
  LogitsArgs t{};
  t.Zc = h->Zc.p;
  t.Y = h->Y.p;
  t.sigma = sigma;
  t.U = h->U.p;
  t.n = h->n;
  t.d = h->d;
  t.K = h->K;
  t.DS = h->DS;
  t.KS = h->KS;
  t.KD = (h->d + 7) & ~7;
  t.normalise = normalise ? 1 : 0;
  const size_t smem_lg = logits_smem_bytes(t.KD);
  CK(cudaFuncSetAttribute(k_logits_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lg));
  const int grid_lg = (int)std::max<int64_t>(1, std::min<int64_t>((h->n + LG_TM - 1) / LG_TM, h->num_sms));
  for (t.n_off = 0; t.n_off < h->K; t.n_off += LG_NP) {
    k_logits_tc<<<grid_lg, LG_THREADS, smem_lg, h->stream>>>(t);
    CKL();
  }
  return 0;
}

}  // namespace

#include "plan.cuh"
#include "tuples.cuh"

namespace {

// ---- K1 launchers: assignment from centroids (init + cold start) -------------------------------
// the fused kernel (assign_tc3.cuh) over the tiles, R / Z_corr outputs and accumulators the caller set in t
int launch_assign_tc3(hb_handle* h, Assign3Args& t, int grid, bool normalise, bool want_obj) {
  t.Zc = h->Zc.p;
  t.Y = h->Y.p;
  t.sigma = h->sigma.p;
  t.U = h->U.p;
  t.tuple_levels = h->tuple_levels.p;
  t.obj_acc = h->obj_acc.p;
  t.d = h->d;
  t.K = h->K;
  t.C = h->C;
  t.B = h->B;
  t.DS = h->DS;
  t.KS = h->KS;
  t.KD = (h->d + 7) & ~7;
  t.NP = (h->K + 15) & ~15;
  t.SS = assign3_stage_stride(h->KS);
  t.ns = h->paths.k1_stages;
  t.normalise = normalise ? 1 : 0;
  t.want_obj = want_obj ? 1 : 0;
  const size_t smem = assign3_smem_bytes(t.ns, t.KD, t.NP, t.KS);
  if (want_obj) {
    CK(cudaFuncSetAttribute(k_assign_tc3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_assign_tc3<true><<<grid, A3_THREADS, smem, h->stream>>>(t);
  } else {
    CK(cudaFuncSetAttribute(k_assign_tc3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_assign_tc3<false><<<grid, A3_THREADS, smem, h->stream>>>(t);
  }
  CKL();
  return 0;
}

// natural order: R, the per-tile sums of O and of the row sums, then O and E; want_obj: objective sums (init)
int run_assign(hb_handle* h, bool normalise, bool want_obj) {
  RegionScope rs(h, "assign");
  const int K = h->K, d = h->d, B = h->B, KS = h->KS;
  float* O_acc = h->Oacc.p;
  float* rs_acc = h->Oacc.p + (size_t)B * KS;
  CK(cudaMemsetAsync(h->Oacc.p, 0, sizeof(float) * ((size_t)B * KS + KS), h->stream));
  switch (h->paths.assign) {
    case Assign::FusedTc: {
      Assign3Args t{};
      t.R = h->R.p;
      t.tile_p0 = h->tc_cell0.p;
      t.tile_len = h->tc_len.p;
      t.tile_tuple = h->tc_tuple.p;
      t.ntiles = h->tc_ntiles;
      t.O_acc = O_acc;
      t.rs_acc = rs_acc;
      t.Zc_out = normalise ? h->Zc.p : nullptr;  // the compatibility paths read the normalised embedding back
      TRY(launch_assign_tc3(h, t, std::max(1, std::min(h->tc_ntiles, h->num_sms)), normalise, want_obj));
      break;
    }
    case Assign::LogitsTc:
    case Assign::LogitsWide: {
      // shapes whose FFMA k_assign does not fit: logits on the tensor cores, then the softmax over the natural-order tiles
      TRY(launch_logits(h, h->sigma.p, normalise, h->paths.assign == Assign::LogitsWide));
      const int nv = sp_nv(KS);
      const size_t smem_sm = sizeof(float) * 8 * 128 * (size_t)nv;
      const int grid = std::max(1, std::min(h->ntiles, h->num_sms * 8));
      TRY(dispatch<1, 2, 4, 8>(h, nv, kUnsupportedK, [&](auto nvc) -> int {
        constexpr int NV = decltype(nvc)::value;
        k_softmax_tiles<NV><<<grid, 256, smem_sm, h->stream>>>(h->U.p, h->R.p, h->sigma.p, h->tile_cell0.p, h->tile_len.p,
                                                               h->tile_tuple.p, h->tuple_levels.p, O_acc, rs_acc,
                                                               h->obj_acc.p, h->ntiles, K, KS, h->C, want_obj ? 1 : 0);
        CKL();
        return 0;
      }));
      if (normalise) {  // the cold start leaves the normalised embedding in Z_corr (harmony.cpp:220)
        k_normalise_rows<<<grid_for((int64_t)h->n * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zc.p, h->Zc.p, h->n, d, h->DS);
        CKL();
      }
      break;
    }
    case Assign::Ffma: {
      AssignArgs a;
      a.Zc = h->Zc.p;
      a.Y = h->Y.p;
      a.sigma = h->sigma.p;
      a.U = h->U.p;
      a.R = h->R.p;
      a.tile_cell0 = h->tile_cell0.p;
      a.tile_len = h->tile_len.p;
      a.tile_tuple = h->tile_tuple.p;
      a.tuple_levels = h->tuple_levels.p;
      a.O_acc = O_acc;
      a.rs_acc = rs_acc;
      a.obj_acc = h->obj_acc.p;
      a.ntiles = h->ntiles;
      a.d = d;
      a.K = K;
      a.C = h->C;
      a.KP = (K + 63) & ~63;
      a.DS = h->DS;
      a.KS = KS;
      a.normalise = normalise ? 1 : 0;
      const size_t smem = assign_ffma_smem_bytes(K, d);
      TRY(dispatch<1, 2, 4, 8, 16, 32>(h, kq_for(K), kUnsupportedK, [&](auto kq) -> int {
        constexpr int KQ = decltype(kq)::value;
        CK(cudaFuncSetAttribute(k_assign<KQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 1;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_assign<KQ>, ASSIGN_THREADS, smem));
        if (occ < 1) occ = 1;
        int grid = std::min(h->ntiles, h->num_sms * occ);
        if (grid < 1) grid = 1;
        k_assign<KQ><<<grid, ASSIGN_THREADS, smem, h->stream>>>(a);
        CKL();
        return 0;
      }));
      break;
    }
  }
  h->R_user_set = false;
  TRY(allreduce_f(h, h->Oacc.p, (size_t)B * KS + KS));
  k_assign_finalize<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(O_acc, rs_acc, h->Pr_b.p, h->O.p, h->E.p, B, K, KS);
  CKL();
  return 0;
}

// cold start in the order of round 0 of the coming cluster_cpp call, where call_path chose that order
// (paths.cold != None): a tile's column sums are a share of its block's removal sums and go to the update kernel's
// accumulator slots; R is not stored and the objective is not evaluated
int run_assign_plan_order(hb_handle* h, bool normalise) {
  RegionScope rs(h, "assign");
  const int K = h->K, B = h->B, KS = h->KS;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  switch (h->paths.cold) {
    case ColdStart::FusedTc: {
      Assign3Args t{};
      t.row_index = r.order;
      t.tile_p0 = r.tile_p0;
      t.tile_len = r.tile_len;
      t.tile_tuple = r.tile_tuple;
      t.tile_blk = r.tile_blk;
      t.ntiles_ptr = r.tile_count;
      t.acc = h->acc2.p;
      TRY(launch_assign_tc3(h, t, h->num_sms, normalise, false));
      break;
    }
    case ColdStart::LogitsTc:
    case ColdStart::LogitsWide: {
      // shapes the fused kernel cannot hold (d > 64 or K > 128): logits on the tensor cores, then one gather pass over
      // U in the order of round 0 for the softmax + the blocks' removal sums (harmony.cpp:312-313)
      TRY(launch_logits(h, h->sigma.p, normalise, h->paths.cold == ColdStart::LogitsWide));
      const int nv = sp_nv(KS);
      const size_t smem_sm = sizeof(float) * 8 * 128 * (size_t)nv;
      TRY(dispatch<1, 2>(h, nv, kUnsupportedUpdateK, [&](auto nvc) -> int {
        constexpr int NV = decltype(nvc)::value;
        k_softmax_block_sums<NV><<<dim3(h->coop_grid, h->nb), 256, smem_sm, h->stream>>>(
            h->U.p, r.order, r.ranges, h->tuple_levels.p, h->acc2.p, h->coop_grid, K, KS, h->C, B);
        CKL();
        return 0;
      }));
      break;
    }
  }
  h->R_user_set = false;
  // O, E of the assignment = the sums of the blocks' removal terms (harmony.cpp:226-227)
  const size_t XH = (size_t)B * KS + KS;
  // sharded cells: the rem halves of slots 1 .. nb in ONE all-reduce (their add halves are still zero here)
  if (h->world > 1) TRY(allreduce_f(h, h->acc2.p + 2 * XH, 2 * XH * (size_t)h->nb));
  k_assign_finalize_plan<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(h->acc2.p, h->nb, h->Pr_b.p, h->O.p, h->E.p, B, K, KS);
  CKL();
  h->zc_pending_norm = normalise;  // the normalised embedding (harmony.cpp:220) is materialised on demand
  return 0;
}

int ensure_trace_cap(hb_handle* h, int slots) {
  if (slots <= h->trace_cap) return 0;
  int ncap = std::max(1024, h->trace_cap * 2);
  while (ncap < slots) ncap *= 2;
  float* np = nullptr;
  CK(cudaMalloc((void**)&np, sizeof(float) * 4 * (size_t)ncap));
  if (h->trace_d.p && h->obj_count > 0)
    CK(cudaMemcpyAsync(np, h->trace_d.p, sizeof(float) * 4 * (size_t)h->obj_count, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (h->trace_d.p) cudaFree(h->trace_d.p);
  h->trace_d.p = np;
  h->trace_d.n = 4 * (size_t)ncap;
  h->trace_cap = ncap;
  return 0;
}

// obj holds this rank's per-cell sums; fold in the K x B cross term of tables (O, E) and append to the trace
int push_objective_from(hb_handle* h, const float* O, const float* E, double* obj) {
  TRY(ensure_trace_cap(h, h->obj_count + 1));
  TRY(allreduce_d(h, obj, 2));
  k_objective_finalize<<<1, 256, 0, h->stream>>>(O, E, h->theta.p, h->sigma.p, obj, h->trace_d.p, h->obj_count, h->B,
                                                  h->K, h->KS, (double)h->N_global, 1.0);
  CKL();
  h->obj_count++;
  return 0;
}
int push_objective(hb_handle* h) { return push_objective_from(h, h->O.p, h->E.p, h->obj_acc.p); }

int sync_traces(hb_handle* h) {
  if (h->obj_synced == h->obj_count) return 0;
  h->obj_vals.resize(4 * (size_t)h->obj_count);
  CK(cudaMemcpyAsync(h->obj_vals.data() + 4 * (size_t)h->obj_synced, h->trace_d.p + 4 * (size_t)h->obj_synced,
                     sizeof(float) * 4 * (size_t)(h->obj_count - h->obj_synced), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->obj_synced = h->obj_count;
  return 0;
}

// harmony.cpp:173-205
int check_convergence_host(hb_handle* h, int type, int* out) {
  TRY(sync_traces(h));
  float obj_new, obj_old;
  auto ok = [&](int slot) { return h->obj_vals[4 * (size_t)slot]; };
  switch (type) {
    case 0: {
      if (h->obj_count < (int)h->window_size + 1) return fail(h, 3, "check_convergence(0): not enough objective values");
      obj_old = 0;
      obj_new = 0;
      for (unsigned i = 0; i < h->window_size; i++) {
        obj_old += ok(h->obj_count - 2 - (int)i);
        obj_new += ok(h->obj_count - 1 - (int)i);
      }
      *out = (std::abs(obj_old - obj_new) / std::abs(obj_old) < h->epsilon_kmeans) ? 1 : 0;
      return 0;
    }
    case 1: {
      if (h->harmony_slots.size() < 2) return fail(h, 3, "check_convergence(1): not enough objective values");
      obj_old = ok(h->harmony_slots[h->harmony_slots.size() - 2]);
      obj_new = ok(h->harmony_slots[h->harmony_slots.size() - 1]);
      *out = ((obj_old - obj_new) / std::abs(obj_old) < h->epsilon_harmony) ? 1 : 0;
      return 0;
    }
  }
  *out = 1;
  return 0;
}

// ---- per-step path: one update_R sweep (harmony.cpp:269-342), three launches per block step ---------------
int run_update_per_step(hb_handle* h) {
  RegionScope rs(h, "update_R");
  const int K = h->K, B = h->B, nb = h->nb, KS = h->KS;
  const int KP = (K + 63) & ~63;
  const size_t slot = 2 * ((size_t)B * KS + KS);  // [add_O | add_rs | rem_O | rem_rs]
  CK(cudaMemsetAsync(h->acc.p, 0, sizeof(float) * 2 * slot, h->stream));
  const PlanRound0 r = plan_round0(h, 0);  // the one round the per-step path plans
  StepArgs a;
  a.U = h->U.p;
  a.R = h->R.p;
  a.order = r.order;
  a.seg_start = r.seg_start;
  a.tile_base = r.tile_base;
  a.tuple_levels = h->tuple_levels.p;
  a.sigma = h->sigma.p;
  a.P = h->P.p;
  a.obj_acc = h->obj_acc.p;
  a.J = h->J;
  a.K = K;
  a.C = h->C;
  a.KP = KP;
  a.KS = KS;
  const int tiles_bound = (int)std::min<int64_t>((h->n / std::max(1, nb)) / TM + h->J + 8, (int64_t)h->num_sms * 8);
  const int grid = std::max(1, tiles_bound);
  const size_t sm_col = sizeof(float) * (size_t)NWARP * KP;
  const size_t sm_upd = sizeof(float) * ((size_t)NWARP * KP + 3 * (size_t)KP);
  return dispatch<1, 2, 4, 8, 16, 32>(h, kq_for(K), kUnsupportedK, [&](auto kq) -> int {
    constexpr int KQ = decltype(kq)::value;
    for (int j = 0; j <= nb; ++j) {
      float* sl = h->acc.p + (size_t)(j & 1) * slot;  // slot j = [add_{j-1} | rem_j]
      float* add_O = sl;
      float* add_rs = sl + (size_t)B * KS;
      float* rem_O = sl + (size_t)B * KS + KS;
      float* rem_rs = rem_O + (size_t)B * KS;
      if (j < nb) {
        a.blk = j;
        a.acc_O = rem_O;
        a.acc_rs = rem_rs;
        RegionScope r1(h, "k_block_colsum");
        k_block_colsum<KQ><<<grid, ROW_THREADS, sm_col, h->stream>>>(a);
        CKL();
      }
      TRY(allreduce_f(h, sl, slot));
      {
        RegionScope r2(h, "k_step_prepare");
        k_step_prepare<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(h->O.p, h->E.p, add_O, add_rs, rem_O, rem_rs,
                                                                     h->Pr_b.p, h->theta.p, (j < nb) ? h->P.p : nullptr, B, K, KS);
        CKL();
      }
      CK(cudaMemsetAsync(sl, 0, sizeof(float) * slot, h->stream));
      if (j < nb) {
        float* nx = h->acc.p + (size_t)((j + 1) & 1) * slot;  // add_j goes to slot j+1
        a.acc_O = nx;
        a.acc_rs = nx + (size_t)B * KS;
        RegionScope r3(h, "k_block_update");
        k_block_update<KQ><<<grid, ROW_THREADS, sm_upd, h->stream>>>(a);
        CKL();
      }
    }
    return 0;
  });
}

// ---- peer-memory exchange area of the persistent update kernel (sharded cells, one node) ----------------
// Areas live for the life of the process, like the communicators: another rank may still be writing into an
// area when its owner drops the handle, and unmapping needs a collective that a destructor cannot afford.  A
// handle leases an area; areas are created collectively, so area i here is paired with area i of every rank.
constexpr int XCH_MAX_AREAS = 16;
std::vector<XchArea*> g_xch_areas;

void release_peer_exchange(hb_handle* h) {
  if (h->xarea) {
    h->xarea->epoch = h->xch.epoch;  // the next lessee continues the epoch sequence
    h->xarea->leased = false;
    h->xarea = nullptr;
  }
  h->use_xch = false;
}
// layout of an area (floats): inbox [slots][world][XH] of 8-byte (value, epoch) words | remT [2][nb][J][KS]
uint2* xch_inbox(const XchArea* a, void* base) { return reinterpret_cast<uint2*>(base); }
float* xch_remT(const XchArea* a, void* base) { return reinterpret_cast<float*>(base) + 2 * a->slots * a->world * a->XH; }
// Collective over the handle's communicator.  Leases an area all ranks have free, or creates a new one:
// allocates this rank's part, exchanges the IPC handles and maps the other ranks' parts.  If any rank cannot
// map a peer the exchange stays off on all ranks (the update then runs one launch + all-reduce per block step).
int setup_peer_exchange(hb_handle* h, int Tplan) {
  const int W = h->world;
  const size_t BK = (size_t)h->B * h->KS, XH = BK + h->KS;
  const size_t slots = (size_t)Tplan * h->nb + 2;
  const size_t remT_floats = 2 * (size_t)h->nb * h->J * h->KS;
  release_peer_exchange(h);
  // 1. agree on a reusable area: free here AND on every other rank, same shape
  int64_t freev[XCH_MAX_AREAS + 2];
  for (int i = 0; i < XCH_MAX_AREAS; ++i) {
    const XchArea* a = i < (int)g_xch_areas.size() ? g_xch_areas[i] : nullptr;
    freev[i] = (a && !a->leased && a->device == h->device && a->world == W && a->rank == h->rank && a->slots == slots &&
                a->XH == XH && a->remT_floats == remT_floats) ? 1 : 0;
  }
  freev[XCH_MAX_AREAS] = (int64_t)g_xch_areas.size();       // min over ranks = smallest pool ...
  freev[XCH_MAX_AREAS + 1] = -(int64_t)g_xch_areas.size();  // ... and -(largest pool): they must agree
  DevBuf<int64_t> dv;
  CK(dv.alloc(XCH_MAX_AREAS + 2));
  CK(cudaMemcpyAsync(dv.p, freev, sizeof(freev), cudaMemcpyHostToDevice, h->stream));
  CKN(g_nccl.AllReduce(dv.p, dv.p, XCH_MAX_AREAS + 2, ncclInt64, ncclMin, h->comm, h->stream));
  CK(cudaMemcpyAsync(freev, dv.p, sizeof(freev), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  XchArea* area = nullptr;
  for (int i = 0; i < XCH_MAX_AREAS && !area; ++i)
    if (freev[i] == 1) area = g_xch_areas[i];
  if (!area) {
    // every rank sees the same reduced values, so every rank takes the same branch here
    if (freev[XCH_MAX_AREAS] != -freev[XCH_MAX_AREAS + 1] || freev[XCH_MAX_AREAS] >= XCH_MAX_AREAS) return 0;  // out of step / pool full
    // 2. create a new area (collective)
    XchArea tmp;
    tmp.slots = slots;
    tmp.world = W;
    tmp.XH = XH;
    const size_t total = (size_t)(xch_remT(&tmp, nullptr) - (float*)nullptr) + remT_floats;
    float* base = nullptr;
    CK(cudaMalloc((void**)&base, sizeof(float) * total));
    CK(cudaMemsetAsync(base, 0, sizeof(float) * total, h->stream));
    cudaIpcMemHandle_t mine;
    CK(cudaIpcGetMemHandle(&mine, base));
    DevBuf<char> ds, dr;
    CK(ds.alloc(sizeof(mine)));
    CK(dr.alloc(sizeof(mine) * W));
    CK(cudaMemcpyAsync(ds.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, h->stream));
    CKN(g_nccl.AllGather(ds.p, dr.p, sizeof(mine), ncclChar, h->comm, h->stream));
    std::vector<cudaIpcMemHandle_t> all(W);
    CK(cudaMemcpyAsync(all.data(), dr.p, sizeof(mine) * W, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    area = new XchArea();
    area->device = h->device;
    area->world = W;
    area->rank = h->rank;
    area->slots = slots;
    area->XH = XH;
    area->remT_floats = remT_floats;
    area->base = base;
    int64_t ok = 1;
    for (int r = 0; r < W; ++r) {
      if (r == h->rank) continue;
      if (cudaIpcOpenMemHandle(&area->peer[r], all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        area->peer[r] = nullptr;
        ok = 0;
      }
    }
    CK(cudaMemcpyAsync(dv.p, &ok, sizeof(ok), cudaMemcpyHostToDevice, h->stream));
    CKN(g_nccl.AllReduce(dv.p, dv.p, 1, ncclInt64, ncclMin, h->comm, h->stream));
    CK(cudaMemcpyAsync(&ok, dv.p, sizeof(ok), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    area->leased = !ok;            // an unusable area keeps its index (the ranks stay in step) but is never leased
    g_xch_areas.push_back(area);
    if (!ok) {
      h->warnings.push_back("peer-memory exchange unavailable (CUDA IPC mapping failed); using per-step all-reduce");
      return 0;
    }
  }
  area->leased = true;
  h->xarea = area;
  PeerXch& x = h->xch;
  x.world = W;
  x.rank = h->rank;
  x.epoch = area->epoch;
  x.XH = (int)XH;
  for (int r = 0; r < W; ++r) {
    void* b = (r == h->rank) ? (void*)area->base : area->peer[r];
    x.peer_inbox[r] = xch_inbox(area, b);
    x.peer_remT[r] = xch_remT(area, b);
  }
  x.inbox = x.peer_inbox[h->rank];
  h->use_xch = true;
  return 0;
}
float* remT_ptr(hb_handle* h) { return h->use_xch ? h->xch.peer_remT[h->rank] : h->remT.p; }

// ---- persistent update kernels over rounds [t0, t1) of this cluster_cpp call ---------------------------
TwoPassArgs make_two_pass_args(hb_handle* h, int T) {
  TwoPassArgs a;
  a.U = h->U.p;
  a.R = h->R.p;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  a.order = r.order;
  a.seg_start = r.seg_start;
  a.prev_at = r.prev_at;
  a.ranges = r.ranges;
  a.tuple_levels = h->tuple_levels.p;
  a.sigma = h->sigma.p;
  a.theta = h->theta.p;
  a.Pr_b = h->Pr_b.p;
  a.ring = h->ring.p;
  a.acc = h->acc2.p;
  a.Psave = h->Psave.p;
  a.OEend = h->OEend.p;
  a.obj = h->obj2.p;
  a.bar = h->bar.p;
  a.n = h->n;
  a.K = h->K;
  a.KS = h->KS;
  a.C = h->C;
  a.J = h->J;
  a.B = h->B;
  a.nb = h->nb;
  a.T = T;
  a.first_round_from_R = h->R_user_set ? 1 : 0;
  a.sigma_uniform = h->sigma_uniform ? 1 : 0;
  a.sigma0 = h->sigma0;
  return a;
}
SinglePassArgs make_single_pass_args(hb_handle* h, int T) {
  SinglePassArgs a;
  a.U = h->U.p;
  a.R = h->R.p;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  a.order = r.order;
  a.next_at = r.next_at;
  a.ranges = r.ranges;
  a.tuple_levels = h->tuple_levels.p;
  a.lvl_ptr = h->lvl_ptr.p;
  a.lvl_tup = h->lvl_tup.p;
  a.lvl_first1 = h->lvl_ptr.p + h->B + 1;
  a.sigma = h->sigma.p;
  a.theta = h->theta.p;
  a.Pr_b = h->Pr_b.p;
  a.ring = h->ring.p;
  a.acc = h->acc2.p;
  a.remT = remT_ptr(h);
  a.remS = h->remS.p;
  a.OEend = h->OEend.p;
  a.obj = h->obj2.p;
  a.bar = h->bar.p;
  a.n = h->n;
  a.K = h->K;
  a.KS = h->KS;
  a.C = h->C;
  a.J = h->J;
  a.B = h->B;
  a.nb = h->nb;
  a.T = T;
  a.s_begin = a.s_end = 0;
  a.write_from = std::min(T - 1, (int)h->window_size + 1);  // rounds after which cluster_cpp may stop (:250-256)
  a.has_next_from = T - 1;
  a.sigma_uniform = h->sigma_uniform ? 1 : 0;
  a.sigma0 = h->sigma0;
  a.ring_rows = h->ring_rows;
  a.coop = 1;
  return a;
}
// per-call state of the persistent update kernels for calls of up to T rounds: accumulator slots, the tables after
// every round, the objective sums and the step counters
int alloc_update_rounds(hb_handle* h, int T) {
  if (h->paths.update == UpdatePath::PerStep) return 0;
  const size_t BK = (size_t)h->B * h->KS;
  CK(h->acc2.alloc(2 * (BK + h->KS) * ((size_t)T * h->nb + 2)));
  CK(h->OEend.alloc((size_t)T * 2 * BK));
  CK(h->obj2.alloc(2 * (size_t)T));
  CK(h->bar.alloc(2 * ((size_t)T * h->nb + 2)));
  return 0;
}
// grows the buffers sized by the rounds of a call (a prebuilt plan is dropped: its buffers go)
int ensure_plan_rounds(hb_handle* h, int T) {
  if (T <= h->plan->rounds) return 0;
  TRY(plan_discard(h));
  CK(cudaStreamSynchronize(h->stream));
  TRY(plan_alloc_rounds(h, T));
  TRY(alloc_update_rounds(h, T));
  if (h->use_xch) TRY(setup_peer_exchange(h, T));  // collective: every rank grows its plan in the same call
  return 0;
}
// zero the per-step accumulators of a cluster_cpp call ...
int update_begin_zero(hb_handle* h, int T) {
  const size_t BK = (size_t)h->B * h->KS, SL = 2 * (BK + h->KS);
  CK(cudaMemsetAsync(h->acc2.p, 0, sizeof(float) * SL * ((size_t)T * h->nb + 2), h->stream));
  CK(cudaMemsetAsync(h->obj2.p, 0, sizeof(double) * 2 * (size_t)T, h->stream));
  CK(cudaMemsetAsync(h->bar.p, 0, sizeof(unsigned) * 2 * ((size_t)T * h->nb + 2), h->stream));
  if (h->paths.update == UpdatePath::SinglePass) CK(cudaMemsetAsync(remT_ptr(h), 0, sizeof(float) * 2 * (size_t)h->nb * h->J * h->KS, h->stream));
  if (h->use_xch) h->xch.epoch++;  // flags of earlier calls no longer match
  return 0;
}
// ... and seed ring[1] (= "O_{-1}") with the tables the call starts from
int update_begin_seed(hb_handle* h) {
  const size_t BK = (size_t)h->B * h->KS;
  CK(cudaMemcpyAsync(h->ring.p + 2 * BK, h->O.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->ring.p + 3 * BK, h->E.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}
int launch_two_pass(hb_handle* h, TwoPassArgs a, bool cooperative) {
  const size_t smem = two_pass_smem_bytes(h->KS, h->nb, h->J);
  return dispatch<1, 2, 4>(h, two_pass_nv(h->KS), kUnsupportedUpdateK, [&](auto nvc) -> int {
    constexpr int NV = decltype(nvc)::value;
    CK(cudaFuncSetAttribute(k_update_two_pass<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    a.use_barrier = cooperative ? 1 : 0;
    if (cooperative) {
      void* args[] = {&a};
      CK(cudaLaunchCooperativeKernel((void*)k_update_two_pass<NV>, dim3(h->coop_grid), dim3(UPD_THREADS), args, smem, h->stream));
    } else {
      k_update_two_pass<NV><<<h->coop_grid, UPD_THREADS, smem, h->stream>>>(a);
    }
    CKL();
    return 0;
  });
}
template <int NV, bool SIGU>
int launch_single_pass_nv(hb_handle* h, SinglePassArgs& a, bool cooperative) {
  const size_t smem = sp_smem_bytes(NV, a.ring_rows, a.KS);
  CK(cudaFuncSetAttribute(k_update_single_pass<NV, SIGU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  a.coop = cooperative ? 1 : 0;
  SinglePassLaunch lp;
  lp.a = a;
  if (h->use_xch) lp.x = h->xch;
  if (cooperative) {
    void* args[] = {&lp};
    CK(cudaLaunchCooperativeKernel((void*)k_update_single_pass<NV, SIGU>, dim3(h->coop_grid), dim3(SP_THREADS), args, smem,
                                   h->stream));
  } else {
    k_update_single_pass<NV, SIGU><<<h->coop_grid, SP_THREADS, smem, h->stream>>>(lp);
  }
  CKL();
  return 0;
}
int launch_single_pass(hb_handle* h, SinglePassArgs a, bool cooperative) {
  return dispatch<1, 2>(h, sp_nv(h->KS), kUnsupportedUpdateK, [&](auto nvc) -> int {
    constexpr int NV = decltype(nvc)::value;
    // sigma_uniform, the default: scalar sigma (objective terms simplify)
    return h->sigma_uniform ? launch_single_pass_nv<NV, true>(h, a, cooperative) : launch_single_pass_nv<NV, false>(h, a, cooperative);
  });
}
// compute_objective() of every round in [t0, t1) (harmony.cpp:248) from the kernels' per-round sums and tables
int push_round_objectives(hb_handle* h, int t0, int t1) {
  const size_t BK = (size_t)h->B * h->KS;
  for (int t = t0; t < t1; ++t) {
    const float* O = (t == t1 - 1) ? h->O.p : h->OEend.p + (size_t)t * 2 * BK;
    const float* E = (t == t1 - 1) ? h->E.p : h->OEend.p + (size_t)t * 2 * BK + BK;
    TRY(push_objective_from(h, O, E, h->obj2.p + 2 * (size_t)t));
  }
  return 0;
}
// single-pass kernel (update_single_pass.cuh), rounds [t0, t1)
int run_update_single_pass(hb_handle* h, int T, int t0, int t1, bool rem_ready) {
  RegionScope rs(h, "update_R");
  const int nb = h->nb;
  const size_t BK = (size_t)h->B * h->KS, XH = BK + h->KS, SL = 2 * XH;
  SinglePassArgs a = make_single_pass_args(h, T);
  if (t0 == 0 && !rem_ready) {
    // removal sums of round 0 from the R in memory (assignment step / user), harmony.cpp:312-313
    RegionScope r0(h, "k_rem_sums");
    k_rem_sums<<<dim3(h->coop_grid, nb), 256, sizeof(float) * 8 * (size_t)h->KS, h->stream>>>(
        h->R.p, a.order, a.ranges, a.tuple_levels, a.acc, 0, h->coop_grid, h->K, h->KS, h->C, h->B);
    CKL();
    if (h->world > 1) TRY(allreduce_f(h, h->acc2.p + SL, SL * (size_t)nb));  // rem halves of slots 1 .. nb (add halves: zero)
  }
  if (h->world <= 1 || h->use_xch) {
    a.s_begin = t0 * nb;
    a.s_end = t1 * nb;
    RegionScope r3(h, "k_update_steps");
    TRY(launch_single_pass(h, a, true));
  } else {
    // sharded cells without peer memory: one launch per block step, the step's add half all-reduced in between; the next round's
    // removal sums (remT) are all-reduced and folded once per round
    RegionScope r3(h, "k_update_steps");
    for (int t = t0; t < t1; ++t) {
      if (t > 0) {
        TRY(allreduce_f(h, h->remT.p + (size_t)(t & 1) * nb * h->J * h->KS, (size_t)nb * h->J * h->KS));
        k_fold_round<<<grid_for((int64_t)nb * h->K, 256, h->num_sms), 256, 0, h->stream>>>(a, t);
        CKL();
      }
      for (int s = t * nb; s < (t + 1) * nb; ++s) {
        if (s > t0 * nb) TRY(allreduce_f(h, h->acc2.p + (size_t)(s + 1) * SL, XH));  // add_{s-1}
        a.s_begin = s;
        a.s_end = s + 1;
        TRY(launch_single_pass(h, a, false));
      }
    }
    TRY(allreduce_f(h, h->acc2.p + (size_t)(t1 * nb + 1) * SL, XH));  // add_{S-1}
  }
  {
    RegionScope r4(h, "k_update_finalize");
    k_single_pass_finalize<<<grid_for(BK, 256, 64), 256, 0, h->stream>>>(a, h->use_xch ? h->xch : PeerXch{}, t1 * nb, h->O.p, h->E.p);
    CKL();
  }
  return push_round_objectives(h, t0, t1);
}
// two-pass kernel (update_two_pass.cuh): look-ahead + update warp groups.  rounds [t0, t1): t0 == 0 runs the
// prologue look-ahead.  write_mask: rounds that store R.
int run_update_two_pass(hb_handle* h, int T, int t0, int t1, unsigned write_mask) {
  RegionScope rs(h, "update_R");
  const int nb = h->nb;
  const size_t BK = (size_t)h->B * h->KS, SL = 2 * (BK + h->KS);
  TwoPassArgs a = make_two_pass_args(h, T);
  a.write_R_mask = write_mask;
  if (h->world <= 1) {
    a.s_begin = t0 * nb;
    a.s_end = t1 * nb;
    a.prologue = (t0 == 0) ? 1 : 0;
    RegionScope r3(h, "k_update_steps");
    TRY(launch_two_pass(h, a, true));
  } else {
    // sharded cells: one launch per step, the step's slot [add_{s-1} | rem_s] all-reduced in between
    RegionScope r3(h, "k_update_steps");
    if (t0 == 0) {
      a.s_begin = a.s_end = 0;
      a.prologue = 1;
      TRY(launch_two_pass(h, a, false));
    }
    a.prologue = 0;
    for (int s = t0 * nb; s < t1 * nb; ++s) {
      TRY(allreduce_f(h, h->acc2.p + (size_t)(s + 1) * SL, SL));
      a.s_begin = s;
      a.s_end = s + 1;
      TRY(launch_two_pass(h, a, false));
    }
    TRY(allreduce_f(h, h->acc2.p + (size_t)(t1 * nb + 1) * SL, SL));  // slot(S): add_{S-1} (+ look-ahead rem_S)
  }
  // tables at the end of round t1-1 -> O, E (the chain itself continues from the ring)
  {
    RegionScope r4(h, "k_update_finalize");
    k_two_pass_finalize<<<grid_for(BK, 256, 64), 256, 0, h->stream>>>(a, t1 * nb, h->O.p, h->E.p);
    CKL();
  }
  return push_round_objectives(h, t0, t1);
}


// S[q][k][:] += R_q^T [Z_q | 1] on the tensor cores (stats_tc3.cuh): one launch per 128 clusters x 64 or 128 columns
// of [Z | 1] (K = 100, d = 50: one launch).  The caller zeroes S.
int run_stats_tc(hb_handle* h, const float* Zsrc) {
  const int K = h->K, D1 = h->d + 1;
  StatsTcArgs t;
  t.R = h->R.p;
  t.Zo = Zsrc;
  t.tile_cell0 = h->tile_cell0.p;
  t.tile_len = h->tile_len.p;
  t.tile_tuple = h->tile_tuple.p;
  t.S = h->S.p;
  t.ntiles = h->ntiles;
  t.d = h->d;
  t.K = K;
  t.KS = h->KS;
  t.DS = h->DS;
  t.tiles_per_cta = std::max(1, (h->ntiles + h->num_sms - 1) / h->num_sms);
  const int grid_tc = (h->ntiles + t.tiles_per_cta - 1) / t.tiles_per_cta;
  const int nb = D1 > 64 ? 128 : 64;
  for (t.k_off = 0; t.k_off < K; t.k_off += 128)
    for (t.c_off = 0; t.c_off < D1; t.c_off += nb) {
      const size_t smem = stats_tc_smem_bytes(stats_tc_rk(h->KS, t.k_off), stats_tc_rc(h->DS, t.c_off, nb), nb);
      if (nb == 64) {
        CK(cudaFuncSetAttribute(k_stats_tc<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_stats_tc<1><<<grid_tc, ST_THREADS, smem, h->stream>>>(t);
      } else {
        CK(cudaFuncSetAttribute(k_stats_tc<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_stats_tc<2><<<grid_tc, ST_THREADS, smem, h->stream>>>(t);
      }
      CKL();
    }
  return 0;
}

// ---- moe_correct_ridge_cpp (harmony.cpp:345-638) -------------------------------------------------
int run_correct(hb_handle* h) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, C = h->C;
  const int D1 = d + 1;
  {
    RegionScope rs(h, "ridge_stats");
    CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * D1, h->stream));
    TRY(run_stats_tc(h, h->Zo.p));
    TRY(allreduce_f(h, h->S.p, (size_t)J * K * D1));
  }
  {
    RegionScope rs(h, "ridge_solve");
    SolveArgs a;
    a.S = h->S.p;
    a.O = h->O.p;
    a.E = h->E.p;
    a.N_b = h->N_b.p;
    a.lambda = h->lambda_estimation ? nullptr : h->lambda.p;
    a.tuple_levels = h->tuple_levels.p;
    a.cov_of = h->cov_of_d.p;
    a.Y = h->Y.p;
    a.V = h->V.p;
    a.Wfull = h->Wfull.p;
    a.skipped = h->skipped.p;
    a.scratch = h->scratch.p;
    a.iscratch = h->iscratch.p;
    a.err_flag = h->err_flag.p;
    a.J = J;
    a.K = K;
    a.B = B;
    a.C = C;
    a.d = d;
    a.KS = h->KS;
    a.alpha = h->alpha;
    a.cutoff = h->cutoff;
    k_ridge_solve<<<K, 256, sizeof(int) * (size_t)(B + C), h->stream>>>(a);
    CKL();
  }
  RegionScope rs(h, "ridge_apply");
  switch (h->paths.apply) {
    case Apply::Tc:
    case Apply::TcCols: {
      // Tc: one range of all columns; TcCols (d > 256, or K x d beyond the FFMA apply): ranges of <= 128 columns.
      // Each column range runs in cluster ranges of at most AP_MAXK clusters, equal sizes, multiples of 8, and small
      // enough for two raw stages of shared memory: the first launch subtracts its share from Zo, the following ones
      // from the partial result in Zc
      const bool cols = h->paths.apply == Apply::TcCols;
      ApplyTcArgs a;
      a.R = h->R.p;
      a.V = h->V.p;
      a.Zc = h->Zc.p;
      a.tile_cell0 = h->tile_cell0.p;
      a.tile_len = h->tile_len.p;
      a.tile_tuple = h->tile_tuple.p;
      a.ntiles = h->ntiles;
      a.d = d;
      a.K = K;
      a.KS = h->KS;
      a.DS = h->DS;
      a.tiles_per_cta = std::max(1, (h->ntiles + h->num_sms - 1) / h->num_sms);
      const int grid = (h->ntiles + a.tiles_per_cta - 1) / a.tiles_per_cta;
      const int DC = cols ? 128 : h->DS;
      auto kernel = cols ? k_apply_tc_cols : d <= 64 ? k_apply_tc<1> : k_apply_tc<2>;
      for (a.c_off = 0; a.c_off < h->DS; a.c_off += DC) {
        a.DC = std::min(DC, h->DS - a.c_off);
        auto stages = [&](int RS) { return cols ? apply_cols_stages(RS, a.DC) : apply_tc_stages(RS, d, h->DS); };
        int npass = (K + AP_MAXK - 1) / AP_MAXK, Kpass = 0;
        for (;; ++npass) {
          Kpass = (((K + npass - 1) / npass) + 7) & ~7;
          if (stages(apply_tc_rs(Kpass, h->KS, 0)) >= 2) break;
        }
        for (int k_off = 0; k_off < K; k_off += Kpass) {
          a.k_off = k_off;
          a.Kp = std::min(Kpass, K - k_off);
          a.KD = (a.Kp + 7) & ~7;
          a.minuend = (k_off == 0) ? h->Zo.p : h->Zc.p;
          const int RS = apply_tc_rs(a.KD, h->KS, k_off);
          const size_t smem = cols ? apply_cols_smem_bytes(RS, a.DC) : apply_tc_smem_bytes(RS, d, h->DS);
          CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
          kernel<<<grid, AP_THREADS, smem, h->stream>>>(a);
          CKL();
        }
      }
      break;
    }
    case Apply::Ffma: {
      ApplyArgs a;
      a.R = h->R.p;
      a.Zo = h->Zo.p;
      a.V = h->V.p;
      a.Zc = h->Zc.p;
      a.tile_cell0 = h->tile_cell0.p;
      a.tile_len = h->tile_len.p;
      a.tile_tuple = h->tile_tuple.p;
      a.ntiles = h->ntiles;
      a.d = d;
      a.K = K;
      a.ldR = h->KS;
      a.ldZ = h->DS;
      const int DP = (d + 3) & ~3;
      dim3 block(DP / 4, TM / 4);
      const size_t smem = apply_ffma_smem_bytes(K, d);
      CK(cudaFuncSetAttribute(k_ridge_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      a.tiles_per_cta = std::max(1, (h->ntiles + h->num_sms * 4 - 1) / (h->num_sms * 4));
      int grid = (h->ntiles + a.tiles_per_cta - 1) / a.tiles_per_cta;
      k_ridge_apply<<<grid, block, smem, h->stream>>>(a);
      CKL();
      break;
    }
  }
  return 0;
}

int check_err_flag(hb_handle* h) {
  int flag = 0;
  CK(cudaMemcpyAsync(&flag, h->err_flag.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (flag) {
    int z = 0;
    cudaMemcpyAsync(h->err_flag.p, &z, sizeof(int), cudaMemcpyHostToDevice, h->stream);
    if (flag == 1) return fail(h, 4, "update order holds an index outside [0, N)");
    if (flag == 2) return fail(h, 5, "inv(): matrix is singular");
    if (flag == 3) return fail(h, 4, "update order is not a permutation of the cells");
    return fail(h, 6, "device error flag %d", flag);
  }
  return 0;
}

// rows of a per-cell field (device row stride ld), un-sorted and widened to double.  Rows are gathered on the device
// as floats (half the PCIe bytes), DMA'd into two pinned staging buffers and widened into the caller's array by the
// host pool while the next chunk is in flight: a device -> host copy of doubles into a freshly allocated pageable
// array runs at the speed of ONE driver thread that also takes the array's page faults (measured: 88 ms for
// 1M x 50 against ~20 ms this way).  The pinned buffers live for the life of the process and are allocated with the
// first handle (hb_create), not inside the first download.
float* g_pinned[2] = {nullptr, nullptr};
constexpr size_t kPinnedFloats = (size_t)8 << 20;  // 32 MiB per buffer
bool ensure_pinned_staging() {
  static std::mutex mk;
  std::lock_guard<std::mutex> lk(mk);
  if (g_pinned[0]) return true;
  for (int i = 0; i < 2; ++i)
    if (cudaHostAlloc((void**)&g_pinned[i], sizeof(float) * kPinnedFloats, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      if (i == 1) cudaFreeHost(g_pinned[0]);
      g_pinned[0] = g_pinned[1] = nullptr;
      return false;  // no pinned memory: the plain path serves
    }
  return true;
}
int download_rows_mt(hb_handle* h, const float* src, int cols, int ld, double* out, bool* done) {
  float** pinned = g_pinned;
  const size_t kFloats = kPinnedFloats;
  *done = false;
  if (!ensure_pinned_staging()) return 0;
  WidenPool* pool = widen_pool();
  const int64_t n = h->n;
  float* dev = reinterpret_cast<float*>(h->stage.p);  // two halves of the device staging buffer
  const size_t dev_half = std::min(kFloats, h->stage.n);  // stage.n doubles = 2 * stage.n floats
  const int64_t rows_per = std::max<int64_t>(1, (int64_t)(dev_half / (size_t)cols));
  const int64_t nchunks = (n + rows_per - 1) / rows_per;
  cudaEvent_t ev[2];
  CK(cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming));
  auto enqueue = [&](int64_t i) -> int {
    const int64_t r0 = i * rows_per, rows = std::min(rows_per, n - r0);
    float* d = dev + (size_t)(i & 1) * dev_half;
    copy_rows(src, ld, d, cols, h->inv_sort.p, r0, false, rows, cols, h->num_sms, h->stream);
    CKL();
    CK(cudaMemcpyAsync(pinned[i & 1], d, sizeof(float) * (size_t)rows * cols, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaEventRecord(ev[i & 1], h->stream));
    return 0;
  };
  int rc = nchunks > 0 ? enqueue(0) : 0;
  for (int64_t i = 0; i < nchunks && rc == 0; ++i) {
    if (i + 1 < nchunks) rc = enqueue(i + 1);  // its buffers were released by widen(i - 1)
    if (rc) break;
    if (cudaEventSynchronize(ev[i & 1]) != cudaSuccess) {
      rc = fail(h, 10, "CUDA error while downloading rows");
      break;
    }
    const int64_t r0 = i * rows_per, rows = std::min(rows_per, n - r0);
    pool->widen(out + r0 * cols, pinned[i & 1], (size_t)rows * cols);
  }
  cudaStreamSynchronize(h->stream);
  cudaEventDestroy(ev[0]);
  cudaEventDestroy(ev[1]);
  *done = (rc == 0);
  return rc;
}
int download_rows(hb_handle* h, const float* src, int cols, int ld, double* out) {
  RegionScope rs(h, "download");
  {
    bool done = false;
    TRY(download_rows_mt(h, src, cols, ld, out, &done));
    if (done) return 0;
  }
  const int64_t n = h->n;
  const int64_t rows_per = std::max<int64_t>(1, (int64_t)(h->stage.n / (size_t)cols));
  for (int64_t r0 = 0; r0 < n; r0 += rows_per) {
    int64_t rows = std::min(rows_per, n - r0);
    copy_rows(src, ld, h->stage.p, cols, h->inv_sort.p, r0, false, rows, cols, h->num_sms, h->stream);
    CKL();
    CK(cudaMemcpyAsync(out + r0 * cols, h->stage.p, sizeof(double) * (size_t)rows * cols, cudaMemcpyDeviceToHost,
                       h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return 0;
}
int upload_rows(hb_handle* h, const double* in, int cols, int ld, float* dst) {
  RegionScope rs(h, "upload");
  const int64_t n = h->n;
  const int64_t rows_per = std::max<int64_t>(1, (int64_t)(h->stage.n / (size_t)cols));
  for (int64_t r0 = 0; r0 < n; r0 += rows_per) {
    int64_t rows = std::min(rows_per, n - r0);
    CK(cudaMemcpyAsync(h->stage.p, in + r0 * cols, sizeof(double) * (size_t)rows * cols, cudaMemcpyHostToDevice,
                       h->stream));
    copy_rows<double, float>(h->stage.p, cols, dst, ld, h->inv_sort.p, r0, true, rows, cols, h->num_sms, h->stream);
    CKL();
    CK(cudaStreamSynchronize(h->stream));
  }
  return 0;
}

// ---- device-memory boundary (hb_setup_device / hb_get_field_device) -------------------------------------------------
// Source of Z for setup: host doubles (d per row, dense) or a device array of `dtype` with row stride `ld`, read on the
// library stream after the work queued on `stream`.
struct ZInput {
  const double* host = nullptr;
  const void* dev = nullptr;
  int dtype = HB_FLOAT64;
  int64_t ld = 0;
  cudaStream_t stream = nullptr;
};
// A caller buffer must be device or managed memory of the handle's device: the kernels dereference it directly.
int check_device_ptr(hb_handle* h, const void* p, const char* what) {
  if (!p) return fail(h, 2, "null %s", what);
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  cudaGetLastError();
  if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged))
    return fail(h, 2, "%s is not device or managed memory (host buffers go through hb_setup / hb_get_field)", what);
  if (a.device != h->device)
    return fail(h, 2, "%s lives on device %d, the handle on device %d", what, a.device, h->device);
  return 0;
}
// Where the labels phi_i lie, found with check_device_ptr's query: *type = cudaMemoryTypeDevice or
// cudaMemoryTypeManaged of the handle's device, else cudaMemoryTypeHost (pageable or pinned).  Another device's
// memory: status 2.  NULL is left to setup's checks.
int phi_location(hb_handle* h, const void* p, cudaMemoryType* type) {
  *type = cudaMemoryTypeHost;
  if (!p) return 0;
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  cudaGetLastError();
  if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)) return 0;
  if (a.device != h->device) return fail(h, 2, "phi_i lives on device %d, the handle on device %d", a.device, h->device);
  *type = a.type;
  return 0;
}
// `later` waits for the work queued on `earlier` so far (no host synchronisation)
int stream_after(hb_handle* h, cudaStream_t later, cudaStream_t earlier) {
  if (later == earlier) return 0;
  cudaEvent_t ev;
  CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  const cudaError_t e1 = cudaEventRecord(ev, earlier);
  const cudaError_t e2 = e1 == cudaSuccess ? cudaStreamWaitEvent(later, ev, 0) : e1;
  cudaEventDestroy(ev);
  CK(e2);
  return 0;
}
// Z (n rows of d values, row stride ld elements, fp32 / fp64 device memory) -> Zo in tuple-sorted order, on the
// library stream after the work queued on `caller`
int upload_rows_device(hb_handle* h, const void* Z, int dtype, int64_t ld, cudaStream_t caller) {
  RegionScope rs(h, "upload");
  TRY(stream_after(h, h->stream, caller));
  if (dtype == HB_FLOAT32)
    copy_rows((const float*)Z, ld, h->Zo.p, h->DS, h->inv_sort.p, 0, true, h->n, h->d, h->num_sms, h->stream);
  else
    copy_rows((const double*)Z, ld, h->Zo.p, h->DS, h->inv_sort.p, 0, true, h->n, h->d, h->num_sms, h->stream);
  CKL();
  return 0;
}
// K x B tables are stored [B][KS]; the boundary wants them dense
int download_table(hb_handle* h, const float* src, double* out) {
  k_compact<<<(h->B * h->K + 255) / 256, 256, 0, h->stream>>>(src, h->tmpT.p, h->B, h->K, h->KS);
  CKL();
  std::vector<float> tmp((size_t)h->B * h->K);
  CK(cudaMemcpyAsync(tmp.data(), h->tmpT.p, sizeof(float) * tmp.size(), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < tmp.size(); ++i) out[i] = (double)tmp[i];
  return 0;
}
int upload_table(hb_handle* h, const double* in, float* dst) {
  std::vector<float> tmp((size_t)h->B * h->K);
  for (size_t i = 0; i < tmp.size(); ++i) tmp[i] = (float)in[i];
  CK(cudaMemcpyAsync(h->tmpT.p, tmp.data(), sizeof(float) * tmp.size(), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemsetAsync(dst, 0, sizeof(float) * (size_t)h->B * h->KS, h->stream));
  k_expand<<<(h->B * h->K + 255) / 256, 256, 0, h->stream>>>(h->tmpT.p, dst, h->B, h->K, h->KS);
  CKL();
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}
int download_small(hb_handle* h, const float* src, size_t count, double* out) {
  std::vector<float> tmp(count);
  CK(cudaMemcpyAsync(tmp.data(), src, sizeof(float) * count, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < count; ++i) out[i] = (double)tmp[i];
  return 0;
}
int upload_small(hb_handle* h, const double* in, size_t count, float* dst) {
  std::vector<float> tmp(count);
  for (size_t i = 0; i < count; ++i) tmp[i] = (float)in[i];
  CK(cudaMemcpyAsync(dst, tmp.data(), sizeof(float) * count, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // namespace

// =================================================================================================
extern "C" {

int hb_version(void) { return 300; }

int hb_create(hb_handle** out, int device) {
  if (!out) return 1;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return 10;  // no CUDA device: there is no CPU path
  hb_handle* h = new hb_handle();
  if (device < 0) cudaGetDevice(&device);
  h->device = device;
  if (cudaSetDevice(device) != cudaSuccess) {
    delete h;
    return 10;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->num_sms = prop.multiProcessorCount;
  cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  h->plan.reset(new Plan());
  ensure_pinned_staging();  // process-wide; the first handle pays for it, not the first download
  keep_pool_memory(device);
  widen_pool();
  *out = h;
  return 0;
}

void hb_destroy(hb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  release_peer_exchange(h);
  cudaStream_t s = h->stream;
  delete h;  // frees device buffers
  if (s) cudaStreamDestroy(s);
}

const char* hb_last_error(const hb_handle* h) { return h ? h->err.c_str() : "null handle"; }

int hb_pop_warning(hb_handle* h, char* buf, size_t cap) {
  if (!h || h->warnings.empty()) return 0;
  if (buf && cap) {
    strncpy(buf, h->warnings.front().c_str(), cap - 1);
    buf[cap - 1] = 0;
  }
  h->warnings.pop_front();
  return 1;
}

int hb_comm_unique_id(char id[HB_COMM_ID_BYTES]) {
  static_assert(sizeof(ncclUniqueId) <= HB_COMM_ID_BYTES, "id size");
  std::string why;
  if (!load_nccl(&why)) return 11;
  ncclUniqueId uid;
  if (g_nccl.GetUniqueId(&uid) != ncclSuccess) return 11;
  memset(id, 0, HB_COMM_ID_BYTES);
  memcpy(id, &uid, sizeof(uid));
  return 0;
}

int hb_comm_init(hb_handle* h, int rank, int world_size, const char id[HB_COMM_ID_BYTES]) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "hb_comm_init must precede hb_setup");
  if (world_size < 1 || rank < 0 || rank >= world_size) return fail(h, 2, "bad rank/world_size");
  h->rank = rank;
  h->world = world_size;
  if (world_size == 1) return 0;
  std::string why;
  if (!load_nccl(&why)) return fail(h, 11, "%s", why.c_str());
  CK(cudaSetDevice(h->device));
  const CommKey key{h->device, rank, world_size};
  if (!id) {  // reuse the process-wide communicator created by an earlier handle
    auto it = g_comms.find(key);
    if (it == g_comms.end()) return fail(h, 3, "hb_comm_init(NULL id): no communicator has been created yet for this rank/world");
    h->comm = it->second;
    return 0;
  }
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  CKN(g_nccl.CommInitRank(&h->comm, world_size, uid, rank));
  g_comms[key] = h->comm;  // kept until process exit
  return 0;
}

int hb_set_shard(hb_handle* h, int64_t N_global, int64_t cell_offset) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "hb_set_shard must precede hb_setup");
  h->N_global = N_global;
  h->cell_offset = cell_offset;
  h->shard_set = true;
  return 0;
}

int hb_set_seed(hb_handle* h, uint64_t seed) {
  if (!h) return 1;
  TRY(plan_discard(h));
  h->seed = seed;
  h->plan->round_counter = 0;
  return 0;
}

int hb_set_abort_callback(hb_handle* h, int (*cb)(void*), void* user) {
  if (!h) return 1;
  h->abort_cb = cb;
  h->abort_user = user;
  return 0;
}

// hb_setup and hb_setup_device: everything but the source of Z
static int setup_common(hb_handle* h, const ZInput& Z, int d, int64_t N, const int32_t* phi_i, bool phi_on_device,
                        const int32_t* B_vec, int C, const double* sigma, const double* theta, const double* lambda, double alpha,
                        int max_iter_kmeans, double epsilon_kmeans, double epsilon_harmony, int K, double block_size,
                        double batch_proportion_cutoff, int verbose) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "setup was already run on this object");
  if (!(Z.host || Z.dev) || !phi_i || !B_vec || !sigma || !theta) return fail(h, 2, "null argument");
  if (d < 1 || N < 1 || C < 1 || K < 1) return fail(h, 2, "bad dimensions");
  if (K > 1024) return fail(h, 2, "K = %d is not supported (K <= 1024)", K);
  if (N > 2000000000LL) return fail(h, 2, "more than 2e9 cells per GPU are not supported");
  CK(cudaSetDevice(h->device));
  h->n = N;
  if (!h->shard_set) {
    if (h->world > 1) return fail(h, 3, "hb_set_shard is required when world_size > 1");
    h->N_global = N;
    h->cell_offset = 0;
  }
  const int64_t NG = h->N_global;
  h->d = d;
  h->C = C;
  h->K = K;
  h->KS = (K + 3) & ~3;
  h->DS = (d + 3) & ~3;
  h->B_vec.assign(B_vec, B_vec + C);
  h->B = std::accumulate(h->B_vec.begin(), h->B_vec.end(), 0);
  const int B = h->B;
  h->cov_of.resize(B);
  {
    int b = 0;
    for (int c = 0; c < C; ++c)
      for (int l = 0; l < B_vec[c]; ++l) h->cov_of[b++] = c;
  }
  // harmony.cpp:83-91
  if (NG < 6) return fail(h, 1, "Refusing to run with less than 6 cells");
  if (NG < 40) {
    h->warnings.push_back("Too few cells. Setting block_size to 0.2");
    h->block_size = 0.2f;
  } else {
    h->block_size = (float)block_size;
  }
  h->epsilon_kmeans = (float)epsilon_kmeans;
  h->epsilon_harmony = (float)epsilon_harmony;
  h->alpha = (float)alpha;
  h->cutoff = (float)batch_proportion_cutoff;
  h->max_iter_kmeans = (unsigned)max_iter_kmeans;
  h->verbose = verbose;
  h->lambda_estimation = (lambda == nullptr) || (lambda[0] == -1);  // harmony.cpp:75
  // update_R block geometry, harmony.cpp:280-281 (float arithmetic on the GLOBAL cell count)
  h->nb = my_ceil(1.0f / h->block_size);
  h->cpb = (uint32_t)((float)NG * h->block_size);
  if (h->cpb == 0) return fail(h, 2, "block_size * N < 1");
  {
    int bits = 1;
    while ((1ull << bits) < (uint64_t)NG) bits++;
    h->half_bits = (bits + 1) / 2;
  }

  HostLap lap(h->stream, "hb_setup");
  // ---- joint covariate tuples; cells get sorted by tuple (stable), on the device (tuples.cuh)
  std::vector<uint64_t> radix(C);
  uint64_t key_space = 1;
  {
    long double prod = 1;
    for (int c = 0; c < C; ++c) prod *= (long double)B_vec[c];
    if (prod > 9e18L) return fail(h, 2, "covariate level product overflows 64 bits");
    for (int c = C - 1; c >= 0; --c) {
      radix[c] = key_space;
      key_space *= (uint64_t)B_vec[c];
    }
  }
  std::vector<int> base(C, 0);
  for (int c = 1; c < C; ++c) base[c] = base[c - 1] + B_vec[c - 1];
  TupleIndex ti;
  {
    RegionScope rs(h, "tuple_index");
    DevBuf<int> phi_up;  // host labels: one upload, then the same kernels
    const int* phi_d = phi_i;
    if (phi_on_device) {
      TRY(stream_after(h, h->stream, Z.stream));  // read after the caller's work, like Z
    } else {
      CK(phi_up.alloc((size_t)N * C));
      CK(cudaMemcpyAsync(phi_up.p, phi_i, sizeof(int) * (size_t)N * C, cudaMemcpyDefault, h->stream));
      phi_d = phi_up.p;
    }
    TRY(build_tuple_index(h, phi_d, N, base, radix, key_space, ti));
  }
  const std::vector<int64_t>& lvl_count = ti.lvl_count;
  const std::vector<int64_t>& tstart = ti.tstart;
  const int J = (int)ti.uniq.size();
  h->J = J;
  h->tuple_levels_h.resize((size_t)J * C);
  for (int q = 0; q < J; ++q) {
    uint64_t kk = ti.uniq[q];
    for (int c = 0; c < C; ++c) {
      h->tuple_levels_h[(size_t)q * C + c] = base[c] + (int)(kk / radix[c]);
      kk %= radix[c];
    }
  }
  h->tuple_start_h = tstart;
  // static tiles (<= TM cells of one tuple)
  std::vector<int> t_cell0, t_len, t_tuple;
  for (int q = 0; q < J; ++q)
    for (int64_t s = tstart[q]; s < tstart[q + 1]; s += TM) {
      t_cell0.push_back((int)s);
      t_len.push_back((int)std::min<int64_t>(TM, tstart[q + 1] - s));
      t_tuple.push_back(q);
    }
  std::vector<int> tc0, tcl, tct;  // 128-cell tiles for the tensor-core kernels
  for (int q = 0; q < J; ++q)
    for (int64_t s2 = tstart[q]; s2 < tstart[q + 1]; s2 += TC_TM) {
      tc0.push_back((int)s2);
      tcl.push_back((int)std::min<int64_t>(TC_TM, tstart[q + 1] - s2));
      tct.push_back(q);
    }
  h->tc_ntiles = (int)tc0.size();
  h->ntiles = (int)t_cell0.size();

  lap.mark("tuple index (device)");
  // ---- device allocations
  const int KS = h->KS, DS = h->DS;
  const size_t nK = (size_t)N * KS, nd = (size_t)N * DS, BK = (size_t)B * KS;
  const int Tplan = std::max(1, (int)h->max_iter_kmeans);
  h->coop_grid = h->num_sms;  // one persistent CTA per SM
  h->paths = select_kernels(K, d, J, N, h->nb, h->coop_grid, h->kernel_set);
  h->ring_rows = sp_ring_rows(KS, SMEM_LIMIT);
  const bool single_pass = h->paths.update == UpdatePath::SinglePass;
  CK(h->Zo.alloc(nd));
  CK(h->Zc.alloc(nd));
  CK(h->U.alloc(nK));
  CK(h->R.alloc(nK));
  CK(h->Y.alloc((size_t)K * d));
  CK(h->sigma.alloc(K));
  CK(h->theta.alloc(B));
  CK(h->Pr_b.alloc(B));
  CK(h->N_b.alloc(B));
  CK(h->lambda.alloc(B + 1));
  CK(h->O.alloc(BK));
  CK(h->E.alloc(BK));
  CK(h->P.alloc(BK));
  CK(h->tmpT.alloc((size_t)B * K));
  CK(h->Oacc.alloc(BK + KS));
  CK(h->acc.alloc(4 * (BK + KS)));
  CK(h->S.alloc((size_t)J * K * (d + 1)));
  CK(h->V.alloc((size_t)J * K * d));
  CK(h->Wfull.alloc((size_t)K * (B + 1) * d));
  CK(h->scratch.alloc((size_t)K * (2 * (size_t)(B + 1) * (B + 1) + (size_t)(B + 1) * d)));
  CK(h->iscratch.alloc((size_t)K * (2 * (size_t)B + J)));
  CK(h->skipped.alloc(K));
  CK(h->err_flag.alloc(1));
  CK(h->obj_acc.alloc(2));
  CK(h->stage.alloc((size_t)8 << 20));  // 64 MiB of doubles
  CK(h->tuple_levels.alloc((size_t)J * C));
  CK(h->cov_of_d.alloc(B));
  CK(h->tile_cell0.alloc(h->ntiles));
  CK(h->tile_len.alloc(h->ntiles));
  CK(h->tile_tuple.alloc(h->ntiles));
  CK(h->tc_cell0.alloc(h->tc_ntiles));
  CK(h->tc_len.alloc(h->tc_ntiles));
  CK(h->tc_tuple.alloc(h->tc_ntiles));
  TRY(plan_setup(h, tstart, Tplan));
  TRY(ensure_plan_rounds(h, Tplan));
  if (h->paths.update != UpdatePath::PerStep) {
    CK(h->ring.alloc(4 * BK));
    CK(h->Psave.alloc(single_pass ? 1 : 2 * (size_t)h->nb * BK));
    if (single_pass) CK(h->remT.alloc(2 * (size_t)h->nb * J * KS));
    if (single_pass && h->world > 1) CK(h->remS.alloc((size_t)h->nb * J * KS));
    release_peer_exchange(h);
    if (single_pass && h->world > 1 && h->world <= XCH_MAXWORLD && !(h->kernel_set & HB_KS_NO_PEER_EXCHANGE))
      TRY(setup_peer_exchange(h, Tplan));
    CK(cudaMemsetAsync(h->Psave.p, 0, sizeof(float) * h->Psave.n, h->stream));
    CK(cudaMemsetAsync(h->ring.p, 0, sizeof(float) * 4 * BK, h->stream));
  }
  lap.mark("device allocations");
  CK(cudaMemsetAsync(h->err_flag.p, 0, sizeof(int), h->stream));
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  CK(cudaMemsetAsync(h->O.p, 0, sizeof(float) * BK, h->stream));
  CK(cudaMemsetAsync(h->E.p, 0, sizeof(float) * BK, h->stream));
  CK(cudaMemsetAsync(h->Wfull.p, 0, sizeof(float) * (size_t)K * (B + 1) * d, h->stream));
  CK(cudaMemsetAsync(h->skipped.p, 0, sizeof(int) * K, h->stream));
  CK(cudaMemsetAsync(h->R.p, 0, sizeof(float) * nK, h->stream));
  CK(cudaMemsetAsync(h->Zo.p, 0, sizeof(float) * nd, h->stream));
  CK(cudaMemsetAsync(h->Zc.p, 0, sizeof(float) * nd, h->stream));
  k_fill_f<<<grid_for((int64_t)nK, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->U.p, (int64_t)nK, U_PAD);
  CKL();
  CK(cudaMemsetAsync(h->Y.p, 0, sizeof(float) * (size_t)K * d, h->stream));
#define UP(buf, vec) CK(cudaMemcpyAsync(h->buf.p, (vec).data(), sizeof((vec)[0]) * (vec).size(), cudaMemcpyHostToDevice, h->stream))
  UP(tuple_levels, h->tuple_levels_h);
  // CSR level -> tuples containing it, ascending tuple order; trailing word: the number of levels of covariate 0
  std::vector<int> lvl_ptr_h(B + 2, 0), lvl_tup_h((size_t)J * C);
  {
    for (size_t i = 0; i < h->tuple_levels_h.size(); ++i) lvl_ptr_h[h->tuple_levels_h[i] + 1]++;
    for (int b = 0; b < B; ++b) lvl_ptr_h[b + 1] += lvl_ptr_h[b];
    std::vector<int> fill(lvl_ptr_h.begin(), lvl_ptr_h.begin() + B);
    for (int q = 0; q < J; ++q)
      for (int c = 0; c < C; ++c) lvl_tup_h[fill[h->tuple_levels_h[(size_t)q * C + c]]++] = q;
    lvl_ptr_h[B + 1] = h->B_vec[0];
    CK(h->lvl_ptr.alloc(B + 2));
    CK(h->lvl_tup.alloc(std::max<size_t>(1, lvl_tup_h.size())));
    UP(lvl_ptr, lvl_ptr_h);
    UP(lvl_tup, lvl_tup_h);
  }
  UP(cov_of_d, h->cov_of);
  UP(tile_cell0, t_cell0);
  UP(tile_len, t_len);
  UP(tile_tuple, t_tuple);
  UP(tc_cell0, tc0);
  UP(tc_len, tcl);
  UP(tc_tuple, tct);
  {
    std::vector<float> f(K);
    for (int k = 0; k < K; ++k) f[k] = (float)sigma[k];
    h->sigma0 = f[0];
    h->sigma_uniform = true;
    for (int k = 1; k < K; ++k) h->sigma_uniform = h->sigma_uniform && (f[k] == f[0]);
    UP(sigma, f);
    f.resize(B);
    for (int b = 0; b < B; ++b) f[b] = (float)theta[b];
    UP(theta, f);
    std::vector<float> nbv(B), prb(B);
    for (int b = 0; b < B; ++b) {
      nbv[b] = (float)lvl_count[b];
      prb[b] = (float)lvl_count[b] / (float)NG;  // harmony.cpp:67
    }
    UP(N_b, nbv);
    UP(Pr_b, prb);
    std::vector<float> lam(B + 1, 0.f);
    if (!h->lambda_estimation)
      for (int b = 0; b <= B; ++b) lam[b] = (float)lambda[b];
    UP(lambda, lam);
    CK(cudaStreamSynchronize(h->stream));
  }
#undef UP
  lap.mark("memsets + small uploads");
  // Z: double -> float, into tuple-sorted order (harmony.cpp:41); Z_corr = normalise(Z_orig) (:42)
  if (Z.dev)
    TRY(upload_rows_device(h, Z.dev, Z.dtype, Z.ld, Z.stream));
  else
    TRY(upload_rows(h, Z.host, d, h->DS, h->Zo.p));
  k_normalise_rows<<<grid_for(N * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zo.p, h->Zc.p, N, d, h->DS);
  CKL();
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("Z upload + normalise");
  h->ran_setup = true;
  return 0;
}

int hb_setup(hb_handle* h, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
             const double* sigma, const double* theta, const double* lambda, double alpha, int max_iter_kmeans,
             double epsilon_kmeans, double epsilon_harmony, int K, double block_size,
             double batch_proportion_cutoff, int verbose) {
  if (!h) return 1;
  cudaMemoryType phi_type;  // managed labels are read like host ones (one copy to the device)
  TRY(phi_location(h, phi_i, &phi_type));
  if (phi_type == cudaMemoryTypeDevice)
    return fail(h, 2, "phi_i is device memory: hb_setup takes host labels (device labels go through hb_setup_device)");
  ZInput z;
  z.host = Z;
  return setup_common(h, z, d, N, phi_i, false, B_vec, C, sigma, theta, lambda, alpha, max_iter_kmeans, epsilon_kmeans,
                      epsilon_harmony, K, block_size, batch_proportion_cutoff, verbose);
}

int hb_setup_device(hb_handle* h, const void* Z, int z_dtype, int64_t z_ld, void* stream, int d, int64_t N,
                    const int32_t* phi_i, const int32_t* B_vec, int C, const double* sigma, const double* theta,
                    const double* lambda, double alpha, int max_iter_kmeans, double epsilon_kmeans,
                    double epsilon_harmony, int K, double block_size, double batch_proportion_cutoff, int verbose) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "setup was already run on this object");
  if (z_dtype != HB_FLOAT32 && z_dtype != HB_FLOAT64) return fail(h, 2, "unknown dtype %d of Z", z_dtype);
  if (z_ld < d) return fail(h, 2, "row stride of Z (%lld) is smaller than d = %d", (long long)z_ld, d);
  TRY(check_device_ptr(h, Z, "Z"));
  cudaMemoryType phi_type;
  TRY(phi_location(h, phi_i, &phi_type));
  ZInput z;
  z.dev = Z;
  z.dtype = z_dtype;
  z.ld = z_ld;
  z.stream = (cudaStream_t)stream;
  return setup_common(h, z, d, N, phi_i, phi_type != cudaMemoryTypeHost, B_vec, C, sigma, theta, lambda, alpha, max_iter_kmeans, epsilon_kmeans,
                      epsilon_harmony, K, block_size, batch_proportion_cutoff, verbose);
}

int hb_init_cluster(hb_handle* h, const double* Y0) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  CK(cudaSetDevice(h->device));
  HostLap lap(h->stream, "hb_init_cluster");
  if (Y0) {
    // Y = normalise(kmeans_centers(..)) (harmony.cpp:133-136), centroids injected by the caller
    TRY(upload_small(h, Y0, (size_t)h->K * h->d, h->Y.p));
  } else {
    // native kmeans_centers (utils.cpp:10-64) on the cosine-normalised cells, sharded like everything else:
    // initialize_centroids' rule (K start cells, then per centroid the winner of an exponential race weighted by the
    // distance from its start cell, already-taken cells skipped) with keyed-hash uniforms, then 10 Lloyd iterations
    // (10 x arma::kmeans(.., keep_existing, 1): Euclidean assignment, means of the members).
    const int K = h->K, d = h->d;
    const size_t Kd = (size_t)K * d;
    if (h->N_global >= (1ll << 32)) return fail(h, 2, "native k-means initialisation supports < 2^32 cells; pass Y0");
    DevBuf<float> ysum;
    CK(ysum.alloc(Kd + K));
    const uint64_t seed = hb_mix64(h->seed ^ 0x6b6d65616e73ull);
    DevBuf<int64_t> cells_d;
    DevBuf<unsigned long long> best_d;
    CK(cells_d.alloc(K));
    CK(best_d.alloc(K));
    std::vector<int64_t> cells(K);
    auto gather = [&](int only) -> int {  // Y rows <- cells (all, or one centroid), summed over the ranks that own them
      CK(cudaMemcpyAsync(cells_d.p, cells.data(), sizeof(int64_t) * K, cudaMemcpyHostToDevice, h->stream));
      float* dst = (only >= 0) ? h->Y.p + (size_t)only * d : h->Y.p;
      const size_t cnt = (only >= 0) ? (size_t)d : Kd;
      CK(cudaMemsetAsync(dst, 0, sizeof(float) * cnt, h->stream));
      k_kmeans_gather<<<K, 64, 0, h->stream>>>(h->Zc.p, h->inv_sort.p, h->Y.p, cells_d.p, K, d, h->DS, h->cell_offset, h->n, only);
      CKL();
      return allreduce_f(h, dst, cnt);
    };
    // (1) start cells: floor(u (N - 1))  (utils.cpp:12-16)
    for (int k = 0; k < K; ++k)
      cells[k] = (int64_t)std::floor((double)kmeans_uniform(seed, (uint64_t)K, (uint64_t)k) * (double)(h->N_global - 1));
    TRY(gather(-1));
    // (2) the races of all centroids in one pass over the cells (a centroid's race only looks at its own start cell)
    // both steps run from tensor-core logits U = 2 (z . y - 1) (sigma = 1) when select_kernels chose them; else from
    // the FFMA kernels (thread per cell)
    DevBuf<float> ones, yy;
    const KmeansInit km = h->paths.kmeans;
    const int km_nv = sp_nv(h->KS);
    const size_t smem = sizeof(float) * Kd;
    if (km == KmeansInit::Ffma) {
      CK(cudaFuncSetAttribute(k_kmeans_race, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      CK(cudaFuncSetAttribute(k_kmeans_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    } else {
      CK(ones.alloc(K));
      CK(yy.alloc(K));
      k_fill_f<<<1, 256, 0, h->stream>>>(ones.p, (int64_t)K, 1.0f);
      CKL();
    }
    std::vector<unsigned long long> best(K);
    bool logits_of_start = false;  // U holds the logits of the start cells
    auto race = [&](int i0, int i1, const std::vector<int64_t>& taken) -> int {
      DevBuf<int64_t> taken_d;
      if (!taken.empty()) {
        CK(taken_d.alloc(taken.size()));
        CK(cudaMemcpyAsync(taken_d.p, taken.data(), sizeof(int64_t) * taken.size(), cudaMemcpyHostToDevice, h->stream));
      }
      CK(cudaMemsetAsync(best_d.p + i0, 0xff, sizeof(unsigned long long) * (i1 - i0), h->stream));
      switch (km) {
        case KmeansInit::Ffma:
          k_kmeans_race<<<grid_for(h->n, 128, h->num_sms * 4), 128, sizeof(float) * (size_t)(i1 - i0) * d, h->stream>>>(
              h->Zc.p, h->sort_perm.p, h->Y.p, best_d.p, taken.empty() ? nullptr : taken_d.p, (int)taken.size(), h->n, K, d, h->DS,
              h->cell_offset, seed, i0, i1);
          CKL();
          break;
        case KmeansInit::LogitsTc:
        case KmeansInit::LogitsWide: {
          if (!logits_of_start) {
            TRY(launch_logits(h, ones.p, false, km == KmeansInit::LogitsWide));
            logits_of_start = true;
          }
          const int grid_r = grid_for(h->n * 32, 256, h->num_sms * 8);
          TRY(dispatch<1, 2, 4, 8>(h, km_nv, kUnsupportedK, [&](auto nvc) -> int {
            constexpr int NV = decltype(nvc)::value;
            k_kmeans_race_u<NV><<<grid_r, 256, 0, h->stream>>>(h->U.p, h->sort_perm.p, best_d.p, taken.empty() ? nullptr : taken_d.p,
                                                             (int)taken.size(), h->n, K, h->KS, h->cell_offset, seed, i0, i1);
            CKL();
            return 0;
          }));
          break;
        }
      }
      if (h->world > 1) CKN(g_nccl.AllReduce(best_d.p + i0, best_d.p + i0, (size_t)(i1 - i0), ncclUint64, ncclMin, h->comm, h->stream));
      CK(cudaMemcpyAsync(best.data() + i0, best_d.p + i0, sizeof(unsigned long long) * (i1 - i0), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      return 0;
    };
    TRY(race(0, K, {}));
    // (3) accept in centroid order; a winner that is already taken re-runs that centroid's race without the taken cells
    // (utils.cpp:38-45); the race of centroid i reads its START cell, so Y is only rewritten afterwards
    std::vector<int64_t> taken;
    for (int i = 0; i < K; ++i) {
      int64_t w = (int64_t)(best[i] & 0xffffffffull);
      if (best[i] == ~0ull) return fail(h, 3, "native k-means initialisation: no free cell for centroid %d", i);
      if (std::find(taken.begin(), taken.end(), w) != taken.end()) {
        TRY(race(i, i + 1, taken));
        if (best[i] == ~0ull) return fail(h, 3, "native k-means initialisation: no free cell for centroid %d", i);
        w = (int64_t)(best[i] & 0xffffffffull);
      }
      taken.push_back(w);
      cells[i] = w;
    }
    h->kmeans_cells = cells;
    TRY(gather(-1));
    for (int iter = 0; iter < 10; ++iter) {
      switch (km) {
        case KmeansInit::Ffma:
          CK(cudaMemsetAsync(ysum.p, 0, sizeof(float) * (Kd + K), h->stream));
          k_kmeans_assign<<<grid_for(h->n, 128, h->num_sms * 4), 128, smem, h->stream>>>(h->Zc.p, h->Y.p, ysum.p, ysum.p + Kd,
                                                                                           h->n, K, d, h->DS);
          CKL();
          TRY(allreduce_f(h, ysum.p, Kd + K));
          k_kmeans_update<<<(int)((Kd + 255) / 256), 256, 0, h->stream>>>(h->Y.p, ysum.p, ysum.p + Kd, K, d);
          CKL();
          break;
        case KmeansInit::LogitsTc:
        case KmeansInit::LogitsWide: {
          // Lloyd iteration on the tensor cores: logits -> one-hot rows of R -> members' sums and counts (K3) -> means
          TRY(launch_logits(h, ones.p, false, km == KmeansInit::LogitsWide));
          k_kmeans_norms<<<(K + 127) / 128, 128, 0, h->stream>>>(h->Y.p, yy.p, K, d);
          CKL();
          const int grid_p = grid_for(h->n * 32, 256, h->num_sms * 8);
          TRY(dispatch<1, 2, 4, 8>(h, km_nv, kUnsupportedK, [&](auto nvc) -> int {
            constexpr int NV = decltype(nvc)::value;
            k_kmeans_pick<NV><<<grid_p, 256, 0, h->stream>>>(h->U.p, yy.p, h->R.p, h->n, K, h->KS);
            CKL();
            return 0;
          }));
          CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)h->J * K * (d + 1), h->stream));
          TRY(run_stats_tc(h, h->Zc.p));
          TRY(allreduce_f(h, h->S.p, (size_t)h->J * K * (d + 1)));
          k_kmeans_means_from_stats<<<(int)((Kd + 255) / 256), 256, 0, h->stream>>>(h->S.p, h->Y.p, h->J, K, d);
          CKL();
          break;
        }
      }
    }
    CK(cudaStreamSynchronize(h->stream));
  }
  // Y = arma::normalise(Y, 2, 0)  (harmony.cpp:136)
  lap.mark("centroids (Y0 / native k-means)");
  k_normalise_rows<<<grid_for((int64_t)h->K * 32, 256, 64), 256, 0, h->stream>>>(h->Y.p, h->Y.p, h->K, h->d, h->d);
  CKL();
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  TRY(run_assign(h, false, true));
  TRY(push_objective(h));                       // compute_objective() (:152)
  lap.mark("assignment + objective");
  h->harmony_slots.push_back(h->obj_count - 1);  // objective_harmony.push_back (:153)
  h->ran_init = true;
  return 0;
}

// STEP 1 of harmony::cluster_cpp as it ran before 2.0.4 (harmony.cpp:235-238):
//   Y = arma::normalise(Z_corr * R.t(), 2, 0);   dist_mat = 2 * (1 - Y.t() * Z_corr);
// built from the kernels of the ridge statistics (R^T [Z_corr | 1] per tuple) and of the assignment.  The
// assignment kernels also rewrite R, O, E and the objective sums, which this step must leave alone: they are
// saved and restored around the call (compatibility path, not a fast one).
int legacy_centroid_step(hb_handle* h) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, KS = h->KS;
  const int D1 = d + 1;
  const size_t nK = (size_t)h->n * KS, BK = (size_t)B * KS;
  CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * D1, h->stream));
  TRY(run_stats_tc(h, h->Zc.p));  // the statistics of the corrected, normalised embedding
  TRY(allreduce_f(h, h->S.p, (size_t)J * K * D1));
  k_centroids_from_stats<<<K, 64, sizeof(float) * (size_t)d, h->stream>>>(h->S.p, h->Y.p, J, K, d);
  CKL();
  // distances to the new centroids -> U; everything else the assignment writes is put back
  if (h->Rkeep.n < nK) CK(h->Rkeep.alloc(nK));
  if (h->OEkeep.n < 2 * BK) CK(h->OEkeep.alloc(2 * BK));
  if (h->objkeep.n < 2) CK(h->objkeep.alloc(2));
  CK(cudaMemcpyAsync(h->Rkeep.p, h->R.p, sizeof(float) * nK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->OEkeep.p, h->O.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->OEkeep.p + BK, h->E.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->objkeep.p, h->obj_acc.p, 2 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  TRY(run_assign(h, false, true));
  CK(cudaMemcpyAsync(h->R.p, h->Rkeep.p, sizeof(float) * nK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->O.p, h->OEkeep.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->E.p, h->OEkeep.p + BK, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->obj_acc.p, h->objkeep.p, 2 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}


int hb_cluster(hb_handle* h, const int64_t* update_orders) {
  if (!h) return 1;
  if (!h->ran_init) return fail(h, 3, "init_cluster_cpp has not been run");
  CK(cudaSetDevice(h->device));
  const unsigned T = h->max_iter_kmeans;
  const bool cold = h->harmony_slots.size() != 1;  // harmony.cpp:214-228 cold start
  TRY(ensure_plan_rounds(h, (int)std::max(1u, T)));
  const CallPath call = call_path(h->paths, T, h->legacy_centroid);
  const bool plan_assign = cold && call.plan_order_assign;
  if (cold && !plan_assign) {
    TRY(run_assign(h, true, false));  // the cold start does not evaluate the objective
    CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  }
  if (update_orders && T > 0) {
    size_t cnt = (size_t)T * (size_t)h->N_global;
    if (h->perms_d.n < cnt) CK(h->perms_d.alloc(cnt));
    CK(cudaMemcpyAsync(h->perms_d.p, update_orders, sizeof(int64_t) * cnt, cudaMemcpyHostToDevice, h->stream));
  }
  if (h->abort_cb && h->abort_cb(h->abort_user)) return -1;  // Progress::check_abort (:233)
  // the call's first native round: a prebuilt plan drew its rounds from here on
  const uint64_t first_round = h->plan->round_counter - (h->plan->next_ready ? (uint64_t)h->plan->next_T : 0);
  unsigned iter = 0;
  if (call.update == UpdatePath::PerStep) {
    TRY(plan_discard(h));  // a plan prebuilt by an earlier call is not used here
    for (iter = 0; iter < T; iter++) {
      if (iter > 0 && h->abort_cb && h->abort_cb(h->abort_user)) return -1;
      if (h->legacy_centroid) TRY(legacy_centroid_step(h));  // :235-238
      TRY(build_plans(h, 1, update_orders ? h->perms_d.p + (size_t)iter * (size_t)h->N_global : nullptr, 0, h->stream, true));
      TRY(run_update_per_step(h));  // :241
      TRY(push_objective(h));          // :248
      if (iter > h->window_size) {  // :250-256
        int conv = 0;
        TRY(check_convergence_host(h, 0, &conv));
        if (conv) {
          iter++;
          break;
        }
      }
    }
  } else {
    // all T update orders are drawn up front (they do not depend on the data), then the rounds run in
    // chunks: [0, window_size + 2) in one launch, afterwards one round per launch (convergence checks)
    TRY(plan_acquire(h, (int)T, update_orders ? h->perms_d.p : nullptr));
    if (T > 0) TRY(update_begin_zero(h, (int)T));
    if (plan_assign) {
      TRY(run_assign_plan_order(h, true));
      CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
    }
    if (T > 0) TRY(update_begin_seed(h));
    unsigned t0 = 0;
    while (t0 < T) {
      unsigned t1 = (t0 == 0) ? std::min(T, h->window_size + 2) : t0 + 1;
      unsigned mask = 0;
      for (unsigned t = t0; t < t1; ++t)
        if (t < 32 && (t == T - 1 || t > h->window_size)) mask |= 1u << t;  // rounds after which cluster_cpp may stop
      if (t0 > 0 && h->abort_cb && h->abort_cb(h->abort_user)) return -1;
      if (call.update == UpdatePath::SinglePass)
        TRY(run_update_single_pass(h, (int)T, (int)t0, (int)t1, plan_assign));
      else
        TRY(run_update_two_pass(h, (int)T, (int)t0, (int)t1, mask));
      iter = t1;
      if (t1 - 1 > h->window_size) {  // :250-256
        int conv = 0;
        TRY(check_convergence_host(h, 0, &conv));
        if (conv) break;
      }
      t0 = t1;
    }
  }
  // the reference draws one shuffle per executed update_R (:268): rounds drawn but not run, after an early stop or in
  // an adopted plan longer than the call, go back to the counter, so the orders do not depend on the update path
  if (!update_orders) h->plan->round_counter = first_round + iter;
  if (call.update != UpdatePath::PerStep && !update_orders && T > 0 && !h->timing)
    TRY(plan_prebuild(h, (int)T));  // the next call's plan, while this call's correction and the next assignment run
  if (T > 0) h->R_user_set = false;
  if (update_orders) TRY(check_err_flag(h));
  h->kmeans_rounds.push_back((int)iter);         // :259
  h->harmony_slots.push_back(h->obj_count - 1);  // :260
  return 0;
}

int hb_moe_correct_ridge(hb_handle* h) {
  if (!h) return 1;
  if (!h->ran_init) return fail(h, 3, "init_cluster_cpp has not been run");
  CK(cudaSetDevice(h->device));
  TRY(run_correct(h));
  h->zc_pending_norm = false;  // Z_corr was rebuilt from Z_orig
  if (h->C > 1) TRY(check_err_flag(h));
  return 0;
}

int hb_check_convergence(hb_handle* h, int type) {
  if (!h) return -1;
  int out = 1;
  int st = check_convergence_host(h, type, &out);
  if (st != 0) return -st;
  return out;
}

int hb_compute_objective(hb_handle* h) {
  if (!h) return 1;
  if (!h->ran_init) return fail(h, 3, "init_cluster_cpp has not been run");
  CK(cudaSetDevice(h->device));
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  k_objective_cells<<<grid_for(h->n * 32, ROW_THREADS, h->num_sms * 8), ROW_THREADS, 0, h->stream>>>(
      h->R.p, h->U.p, h->sigma.p, h->n, h->K, h->KS, h->obj_acc.p);
  CKL();
  return push_objective(h);
}

int64_t hb_field_size(const hb_handle* h, int field) {
  if (!h || !h->ran_setup) return 0;
  switch (field) {
    case HB_Z_CORR:
    case HB_Z_ORIG: return (int64_t)h->n * h->d;
    case HB_R: return (int64_t)h->n * h->K;
    case HB_Y: return (int64_t)h->K * h->d;
    case HB_O:
    case HB_E: return (int64_t)h->K * h->B;
    case HB_W: return (int64_t)(h->B + 1) * h->d;
    case HB_PR_B:
    case HB_THETA: return h->B;
    case HB_SIGMA: return h->K;
    case HB_LAMBDA: return (int64_t)h->K * (h->B + 1);
    case HB_LAMBDA_VEC: return h->B + 1;
  }
  return 0;
}

// cluster_cpp leaves Z_corr cosine-normalised (harmony.cpp:220); the library normalises on the first read of Z_corr
static int normalise_pending_zc(hb_handle* h) {
  if (!h->zc_pending_norm) return 0;
  k_normalise_rows<<<grid_for((int64_t)h->n * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zc.p, h->Zc.p, h->n, h->d, h->DS);
  CKL();
  h->zc_pending_norm = false;
  return 0;
}

int hb_get_field(hb_handle* h, int field, double* out) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  if (!out) return fail(h, 2, "null output");
  CK(cudaSetDevice(h->device));
  const int K = h->K, B = h->B, d = h->d;
  switch (field) {
    case HB_Z_CORR: {
      HostLap lap(h->stream, "hb_get_field");
      TRY(normalise_pending_zc(h));
      const int rc = download_rows(h, h->Zc.p, d, h->DS, out);
      lap.mark("Z_corr download");
      return rc;
    }
    case HB_Z_ORIG: return download_rows(h, h->Zo.p, d, h->DS, out);
    case HB_R: return download_rows(h, h->R.p, K, h->KS, out);
    case HB_Y: return download_small(h, h->Y.p, (size_t)K * d, out);
    case HB_O: return download_table(h, h->O.p, out);
    case HB_E: return download_table(h, h->E.p, out);
    case HB_PR_B: return download_small(h, h->Pr_b.p, B, out);
    case HB_THETA: return download_small(h, h->theta.p, B, out);
    case HB_SIGMA: return download_small(h, h->sigma.p, K, out);
    case HB_LAMBDA_VEC: return download_small(h, h->lambda.p, B + 1, out);
    case HB_LAMBDA: {  // getLambda, harmony.cpp:657-669: K x (B+1) column-major
      std::vector<double> E((size_t)K * B), lam(B + 1);
      TRY(download_table(h, h->E.p, E.data()));
      TRY(download_small(h, h->lambda.p, B + 1, lam.data()));
      for (int k = 0; k < K; ++k) {
        out[k] = h->lambda_estimation ? 0.0 : lam[0];
        for (int b = 0; b < B; ++b)
          out[(size_t)(b + 1) * K + k] =
              h->lambda_estimation ? (double)((float)E[(size_t)b * K + k] * h->alpha) : lam[b + 1];
      }
      return 0;
    }
    case HB_W: {  // (B+1) x d column-major; betas of the last cluster that was corrected
      std::vector<int> sk(K);
      CK(cudaMemcpyAsync(sk.data(), h->skipped.p, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      int last = -1;
      for (int k = 0; k < K; ++k)
        if (!sk[k]) last = k;
      std::vector<double> w((size_t)(B + 1) * d, 0.0);
      if (last >= 0) TRY(download_small(h, h->Wfull.p + (size_t)last * (B + 1) * d, (size_t)(B + 1) * d, w.data()));
      for (int b = 0; b <= B; ++b)
        for (int c = 0; c < d; ++c) out[(size_t)c * (B + 1) + b] = w[(size_t)b * d + c];
      return 0;
    }
  }
  return fail(h, 2, "unknown field %d", field);
}

int hb_get_field_device(hb_handle* h, int field, void* out, int dtype, int64_t ld, void* stream) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  if (field != HB_Z_CORR && field != HB_Z_ORIG && field != HB_R)
    return fail(h, 2, "field %d has no device getter (HB_Z_CORR, HB_Z_ORIG, HB_R)", field);
  if (dtype != HB_FLOAT32 && dtype != HB_FLOAT64) return fail(h, 2, "unknown dtype %d", dtype);
  const int cols = field == HB_R ? h->K : h->d;
  if (ld < cols) return fail(h, 2, "row stride %lld is smaller than the field's %d columns", (long long)ld, cols);
  TRY(check_device_ptr(h, out, "output"));
  CK(cudaSetDevice(h->device));
  const cudaStream_t caller = (cudaStream_t)stream;
  TRY(stream_after(h, h->stream, caller));  // the caller's earlier work on `out` comes first
  if (field == HB_Z_CORR) TRY(normalise_pending_zc(h));
  {
    RegionScope rs(h, "download");
    const float* src = field == HB_Z_CORR ? h->Zc.p : field == HB_Z_ORIG ? h->Zo.p : h->R.p;
    const int src_ld = field == HB_R ? h->KS : h->DS;
    if (dtype == HB_FLOAT32)
      copy_rows(src, src_ld, (float*)out, ld, h->inv_sort.p, 0, false, h->n, cols, h->num_sms, h->stream);
    else
      copy_rows(src, src_ld, (double*)out, ld, h->inv_sort.p, 0, false, h->n, cols, h->num_sms, h->stream);
    CKL();
  }
  return stream_after(h, caller, h->stream);
}

int hb_set_field(hb_handle* h, int field, const double* in) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  if (!in) return fail(h, 2, "null input");
  CK(cudaSetDevice(h->device));
  const int K = h->K, B = h->B, d = h->d;
  switch (field) {
    case HB_Z_CORR:
      h->zc_pending_norm = false;
      return upload_rows(h, in, d, h->DS, h->Zc.p);
    case HB_R:
      h->R_user_set = true;
      return upload_rows(h, in, K, h->KS, h->R.p);
    case HB_Y: return upload_small(h, in, (size_t)K * d, h->Y.p);
    case HB_O: return upload_table(h, in, h->O.p);
    case HB_E: return upload_table(h, in, h->E.p);
    case HB_THETA: return upload_small(h, in, B, h->theta.p);
    case HB_SIGMA: {
      for (int k = 0; k < K; ++k)
        if (!(std::isfinite(in[k]) && (float)in[k] > 0.f))
          return fail(h, 2, "sigma[%d] = %g: sigma must be finite and positive", k, in[k]);
      if (h->ran_init) {
        // U holds -dist / sigma_old (the reference keeps dist_mat and divides by the current sigma in every update_R and
        // compute_objective, harmony.cpp:158-162, 318-319): rescale column k by sigma_old[k] / sigma_new[k]
        std::vector<double> old(K);
        TRY(download_small(h, h->sigma.p, K, old.data()));
        std::vector<double> ratio(K);
        for (int k = 0; k < K; ++k) ratio[k] = old[k] / (double)(float)in[k];
        DevBuf<float> s;
        CK(s.alloc(K));
        TRY(upload_small(h, ratio.data(), K, s.p));
        k_scale_cols<<<grid_for(h->n * K, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->U.p, s.p, h->n, K, h->KS);
        CKL();
        CK(cudaStreamSynchronize(h->stream));
      }
      h->sigma0 = (float)in[0];
      h->sigma_uniform = true;
      for (int k = 1; k < K; ++k) h->sigma_uniform = h->sigma_uniform && ((float)in[k] == (float)in[0]);
      return upload_small(h, in, K, h->sigma.p);
    }
    case HB_LAMBDA_VEC:
      h->lambda_estimation = false;
      return upload_small(h, in, B + 1, h->lambda.p);
  }
  return fail(h, 2, "field %d is not writable", field);
}

int hb_get_scalar(const hb_handle* h, int which, double* out) {
  if (!h || !out) return 1;
  switch (which) {
    case HB_N: *out = (double)h->N_global; return 0;
    case HB_N_LOCAL: *out = (double)h->n; return 0;
    case HB_B: *out = h->B; return 0;
    case HB_K: *out = h->K; return 0;
    case HB_D: *out = h->d; return 0;
    case HB_C: *out = h->C; return 0;
    case HB_ALPHA: *out = h->alpha; return 0;
    case HB_MAX_ITER_KMEANS: *out = h->max_iter_kmeans; return 0;
    case HB_BLOCK_SIZE: *out = h->block_size; return 0;
    case HB_EPSILON_KMEANS: *out = h->epsilon_kmeans; return 0;
    case HB_EPSILON_HARMONY: *out = h->epsilon_harmony; return 0;
    case HB_LAMBDA_ESTIMATION: *out = h->lambda_estimation ? 1 : 0; return 0;
    case HB_WINDOW_SIZE: *out = h->window_size; return 0;
    case HB_LEGACY_CENTROID_STEP: *out = h->legacy_centroid ? 1 : 0; return 0;
    case HB_KERNEL_SET: *out = h->kernel_set; return 0;
    case HB_DEVICE: *out = h->device; return 0;
  }
  return 2;
}

int hb_set_scalar(hb_handle* h, int which, double value) {
  if (!h) return 1;
  switch (which) {
    case HB_ALPHA: h->alpha = (float)value; return 0;
    case HB_MAX_ITER_KMEANS:
      if (value < 0) return fail(h, 2, "max_iter_kmeans must be >= 0");
      h->max_iter_kmeans = (unsigned)value;
      return 0;
    case HB_EPSILON_KMEANS: h->epsilon_kmeans = (float)value; return 0;
    case HB_EPSILON_HARMONY: h->epsilon_harmony = (float)value; return 0;
    case HB_LEGACY_CENTROID_STEP: h->legacy_centroid = value != 0.0; return 0;
    case HB_KERNEL_SET: h->kernel_set = (int)value; return 0;  // takes effect at the next hb_setup
  }
  return fail(h, 2, "scalar %d is not writable", which);
}

int hb_get_B_vec(const hb_handle* h, int32_t* out) {
  if (!h || !out) return 1;
  for (int c = 0; c < h->C; ++c) out[c] = h->B_vec[c];
  return 0;
}

int64_t hb_trace(const hb_handle* hc, int trace, double* out, int64_t cap) {
  hb_handle* h = const_cast<hb_handle*>(hc);
  if (!h) return -1;
  if (trace == HB_KMEANS_ROUNDS) {
    if (out)
      for (int64_t i = 0; i < (int64_t)h->kmeans_rounds.size() && i < cap; ++i) out[i] = h->kmeans_rounds[i];
    return (int64_t)h->kmeans_rounds.size();
  }
  if (sync_traces(h) != 0) return -1;
  if (trace >= HB_OBJECTIVE_KMEANS && trace <= HB_OBJECTIVE_KMEANS_CROSS) {
    if (out)
      for (int64_t i = 0; i < h->obj_count && i < cap; ++i) out[i] = h->obj_vals[4 * (size_t)i + trace];
    return h->obj_count;
  }
  if (trace == HB_OBJECTIVE_HARMONY) {
    if (out)
      for (int64_t i = 0; i < (int64_t)h->harmony_slots.size() && i < cap; ++i)
        out[i] = h->obj_vals[4 * (size_t)h->harmony_slots[i]];
    return (int64_t)h->harmony_slots.size();
  }
  return -1;
}

int64_t hb_kernel_launches(const hb_handle* h) { return h ? h->launches : 0; }
void* hb_stream(const hb_handle* h) { return h ? (void*)h->stream : nullptr; }

int hb_synchronize(hb_handle* h) {
  if (!h) return 1;
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int hb_region_time(hb_handle* h, const char* region, double* ms, int64_t* launches) {
  if (!h || !region) return 1;
  auto it = h->regions.find(region);
  if (it == h->regions.end()) return 2;
  if (ms) *ms = it->second.ms;
  if (launches) *launches = it->second.launches;
  return 0;
}

// Host evaluation of the keyed cell-order permutation used for the native update orders (test hook; the
// same __host__ __device__ code runs in k_plan_block_native / k_kmeans_seed).
uint64_t hb_debug_permute(uint64_t i, uint64_t n, uint64_t key, int inverse) {
  if (n == 0 || i >= n) return ~0ull;
  int bits = 1;
  while ((1ull << bits) < n) bits++;
  const int half_bits = (bits + 1) / 2;
  return inverse ? hb_permute_inv(i, n, half_bits, key) : hb_permute(i, n, half_bits, key);
}

// Host worker pool (test hook, host only): out[i] = (double) in[i] with `threads` threads (first call fixes the
// pool size for the process).  Returns the number of threads of the pool.
int hb_debug_widen(double* out, const float* in, int64_t n, int threads) {
  WidenPool* p = widen_pool(threads);
  if (n > 0) p->widen(out, in, (size_t)n);
  return p->threads();
}

// Ring geometry of the persistent update kernel for rows of KS floats (test hook, host only):
// out = {float4 per lane, groups per warp ring, rows per group, shared-memory bytes, warps}; 0 if the kernel cannot run the shape.
int hb_debug_update_geometry(int KS, int nb, int64_t out[9]) {
  (void)nb;
  if (KS <= 0 || (KS & 3)) return 0;
  const int D = sp_ring_rows(KS, SMEM_LIMIT);
  if (D <= 0) return 0;
  const int nv = sp_nv(KS), ru = sp_ru(nv);
  const int64_t v[9] = {nv, D / ru, ru, (int64_t)sp_smem_bytes(nv, D, KS), SP_NW, 0, 0, 0, 0};
  for (int i = 0; i < 9; ++i) out[i] = v[i];
  return 1;
}

// Kernels hb_setup picks for a shape, and the update path of a cluster_cpp call (test hook, host only).
// Fields 2 and 4 are derived from the stage choices: "wgmma logits" is a k_logits_tc cold start without
// HB_KS_FFMA_CONTRACTIONS (with it, only shapes past FFMA k_assign take that cold start), "tensor-core k-means" a
// k_logits_tc initialisation at KS <= 256.
int hb_debug_kernel_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[8]) {
  const KernelPaths p = select_kernels(K, d, J, n, nb, num_sms, kernel_set);
  const bool cold_logits_tc = p.cold == ColdStart::LogitsTc && !(kernel_set & HB_KS_FFMA_CONTRACTIONS);
  const bool kmeans_tc = p.kmeans == KmeansInit::LogitsTc && ((K + 3) & ~3) <= 256;
  const int64_t v[8] = {(int64_t)p.update, p.k1_stages, cold_logits_tc, p.apply == Apply::Tc, kmeans_tc,
                        call_path(p, 20, false).plan_order_assign, (int64_t)call_path(p, 40, false).update,
                        (int64_t)call_path(p, 20, true).update};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
  return 0;
}

// The kernels of the stages whose FFMA kernels stop at a shared-memory limit, and the kernels that take those shapes
// instead (test hook, host only).  out = {natural-order assignment: 1 fused wgmma, 2 FFMA k_assign, 3 k_logits_tc +
// softmax pass, 4 k_logits_wide + softmax pass; plan-order cold start of a 20-round call: 0 none (natural order),
// 1 fused wgmma, 2 k_logits_tc + block sums, 3 k_logits_wide + block sums; ridge apply: 1 wgmma, 2 FFMA, 3 column
// ranges; native k-means initialisation: 1 FFMA, 2 k_logits_tc logits (KS <= 256), 3 k_logits_tc logits, 4
// k_logits_wide logits}.  The k-means values 2 and 3 run the same kernels; they tell KS <= 256 from KS > 256.
int hb_debug_wide_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[4]) {
  const KernelPaths p = select_kernels(K, d, J, n, nb, num_sms, kernel_set);
  out[0] = (int64_t)p.assign;
  out[1] = call_path(p, 20, false).plan_order_assign ? (int64_t)p.cold : 0;
  out[2] = (int64_t)p.apply;
  out[3] = p.kmeans == KmeansInit::Ffma ? 1 : p.kmeans == KmeansInit::LogitsWide ? 4 : ((K + 3) & ~3) <= 256 ? 2 : 3;
  return 0;
}

// The covariate-tuple index setup built (test hook): J, and the non-null ones of sort_perm (N_local cells, sorted
// position -> caller's cell), tuple_levels (J x C global levels) and tuple_start (J + 1 first sorted positions).
int hb_debug_tuple_index(const hb_handle* h, int32_t* sort_perm, int32_t* tuple_levels, int64_t* tuple_start) {
  if (!h || !h->ran_setup) return -1;
  if (sort_perm &&
      (cudaSetDevice(h->device) != cudaSuccess ||
       cudaMemcpy(sort_perm, h->sort_perm.p, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToHost) != cudaSuccess))
    return -1;
  if (tuple_levels) std::copy(h->tuple_levels_h.begin(), h->tuple_levels_h.end(), tuple_levels);
  if (tuple_start) std::copy(h->tuple_start_h.begin(), h->tuple_start_h.end(), tuple_start);
  return h->J;
}

// Test hooks of the native kmeans_centers: the uniform of (centroid i, global cell g) under the handle's seed, and
// the cells initialize_centroids chose (K values; 0 if the native initialisation has not run).
double hb_debug_kmeans_uniform(const hb_handle* h, uint64_t i, uint64_t g) {
  return (double)kmeans_uniform(hb_mix64(h->seed ^ 0x6b6d65616e73ull), i, g);
}
int hb_debug_kmeans_cells(const hb_handle* h, int64_t* out) {
  if (!h || h->kmeans_cells.empty()) return 0;
  for (size_t i = 0; i < h->kmeans_cells.size(); ++i) out[i] = h->kmeans_cells[i];
  return (int)h->kmeans_cells.size();
}

int hb_enable_timing(hb_handle* h, int on) {
  if (!h) return 1;
  h->timing = on != 0;
  return 0;
}

}  // extern "C"
