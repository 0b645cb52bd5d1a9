// handle.cuh — hb_handle and what every host module uses with it: buffers, errors, counted launches, timing regions.
#pragma once

namespace {

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
  // at least `count` elements: a smaller buffer is replaced (its contents go), a large enough one is kept as it is
  cudaError_t reserve(size_t count) { return n < count ? alloc(count) : cudaSuccess; }
};
void keep_pool_memory(int device) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  cudaGetLastError();
}

// Tiles of at most `rows` consecutive cells of one covariate tuple in sorted order (build_tiles)
struct Tiles {
  DevBuf<int> cell0, len, tuple;
  int count = 0;
  // the tile fields of a kernel's arguments, with its tiles dealt out to at most `ctas` CTAs; returns the grid
  template <typename A>
  int deal(A& a, int ctas) const {
    a.tile_cell0 = cell0.p;
    a.tile_len = len.p;
    a.tile_tuple = tuple.p;
    a.ntiles = count;
    a.tiles_per_cta = std::max(1, (count + ctas - 1) / ctas);
    return (count + a.tiles_per_cta - 1) / a.tiles_per_cta;
  }
};

struct Region {
  double ms = 0;
  int64_t launches = 0;
};

struct Plan;         // plan.cuh
struct UpdateState;  // update_host.cuh
struct AssignState;  // assign_host.cuh
struct MapState;     // map_host.cuh
struct ScoreScratch;  // score_host.cuh

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
  bool sigma_uniform = false;
  float sigma0 = 0.f;
  bool R_user_set = false;       // R was written through hb_set_field since the last assignment step
  bool zc_pending_norm = false;  // Zc holds the un-normalised corrected embedding although cluster_cpp has run
  bool mapping = false;          // set up by hb_map_setup: a query mapped onto a reference, not a Harmony run
  bool ran_map = false;
  std::vector<int> tuple_levels_h;     // [J][C]
  std::vector<int64_t> tuple_start_h;  // [J + 1] first sorted position of each tuple
  std::vector<int64_t> kmeans_cells;   // global cells chosen by the native initialize_centroids (test hook)
  bool kmeans_keep_means = false;      // record Y after the race's gather and after every Lloyd step (test hook)
  std::vector<float> kmeans_means;     // [steps][K][d] recorded while kmeans_keep_means is on

  // kernels
  KernelPaths paths;             // kernels picked by hb_setup (select_kernels)
  int kernel_set = 0;            // HB_KERNEL_SET test hook (bits HB_KS_*), read by hb_setup
  bool legacy_centroid = false;  // HB_LEGACY_CENTROID_STEP: centroid update at the top of every clustering round
  int coop_grid = 0;             // CTAs of the persistent update kernels and of the plan's ranges

  // device state
  DevBuf<float> Zo, Zc, U, R, Y, sigma, theta, Pr_b, N_b, lambda, O, E, Oacc, S, V, Wfull, scratch, tmpT;
  DevBuf<double> obj_acc, stage;
  DevBuf<int> sort_perm, inv_sort, tuple_levels, cov_of_d, iscratch, skipped, err_flag;
  DevBuf<int64_t> perms_d;
  Tiles tiles;     // TM-cell tiles of the FFMA kernels and the stats / apply kernels
  Tiles tc_tiles;  // TC_TM-cell tiles of the fused assignment kernel
  std::unique_ptr<Plan> plan;
  std::unique_ptr<UpdateState> upd;
  std::unique_ptr<AssignState> asg;
  std::unique_ptr<MapState> map;  // hb_map_setup only
  std::unique_ptr<ScoreScratch> scores;  // the scratch of the score calls (score_host.cuh), from the first such call

  // traces (harmony.h:55-56); values are produced on the device and pulled lazily
  DevBuf<float> trace_d;
  int trace_cap = 0;
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

// kernel<<<grid, block, smem, h->stream>>>(args...) with the kernel's dynamic shared-memory limit raised to smem
template <typename... P, typename... A>
int launch(hb_handle* h, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<grid, block, smem, h->stream>>>(std::forward<A>(args)...);
  CKL();
  return 0;
}
// the same for a kernel of one argument, as a cooperative launch when `cooperative`
template <typename P>
int launch_coop(hb_handle* h, void (*kernel)(P), bool cooperative, dim3 grid, dim3 block, size_t smem, P arg) {
  if (!cooperative) return launch(h, kernel, grid, block, smem, arg);
  CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  void* args[] = {&arg};
  CK(cudaLaunchCooperativeKernel((void*)kernel, grid, block, args, smem, h->stream));
  CKL();
  return 0;
}

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

int grid_for(int64_t work_items, int threads, int cap) {
  int64_t g = (work_items + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

int kq_for(int K) {  // the smallest power of two with 32 kq >= K
  int kq = 1;
  while (32 * kq < K) kq <<= 1;
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

// The tiles of at most `rows` cells of the tuples whose sorted cells are [tstart[q], tstart[q + 1]), uploaded
int build_tiles(hb_handle* h, Tiles& t, const std::vector<int64_t>& tstart, int rows) {
  std::vector<int> cell0, len, tuple;
  for (int q = 0; q + 1 < (int)tstart.size(); ++q)
    for (int64_t s = tstart[q]; s < tstart[q + 1]; s += rows) {
      cell0.push_back((int)s);
      len.push_back((int)std::min<int64_t>(rows, tstart[q + 1] - s));
      tuple.push_back(q);
    }
  t.count = (int)cell0.size();
  for (auto u : {std::make_pair(&t.cell0, &cell0), std::make_pair(&t.len, &len), std::make_pair(&t.tuple, &tuple)}) {
    CK(u.first->alloc(u.second->size()));
    CK(cudaMemcpyAsync(u.first->p, u.second->data(), sizeof(int) * u.second->size(), cudaMemcpyHostToDevice, h->stream));
  }
  return 0;
}

}  // namespace
