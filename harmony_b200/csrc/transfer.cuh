// transfer.cuh — host <-> device transfers of the C ABI: per-cell rows (un-sorted on download, sorted on upload),
// the K x B tables and small arrays, and the checks and stream ordering of caller device memory.  Included by
// harmony_b200.cu after trace.cuh.
#pragma once

namespace {

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
  *done = false;
  if (!ensure_pinned_staging()) return 0;
  WidenPool* pool = widen_pool();
  const int64_t n = h->n;
  float* dev = reinterpret_cast<float*>(h->stage.p);  // two halves of the device staging buffer
  const size_t dev_half = std::min(kPinnedFloats, h->stage.n);  // stage.n doubles = 2 * stage.n floats
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
    CK(cudaMemcpyAsync(g_pinned[i & 1], d, sizeof(float) * (size_t)rows * cols, cudaMemcpyDeviceToHost, h->stream));
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
    pool->widen(out + r0 * cols, g_pinned[i & 1], (size_t)rows * cols);
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

// The device buffer, column count and row stride of a per-cell field (HB_Z_CORR, HB_Z_ORIG, HB_R); buf is null for
// any other field
struct RowField {
  float* buf;
  int cols, ld;
};
RowField row_field(hb_handle* h, int field) {
  switch (field) {
    case HB_Z_CORR: return {h->Zc.p, h->d, h->DS};
    case HB_Z_ORIG: return {h->Zo.p, h->d, h->DS};
    case HB_R: return {h->R.p, h->K, h->KS};
  }
  return {nullptr, 0, 0};
}

// cluster_cpp leaves Z_corr cosine-normalised (harmony.cpp:220); the library normalises on the first read of Z_corr
int normalise_pending_zc(hb_handle* h) {
  if (!h->zc_pending_norm) return 0;
  k_normalise_rows<<<grid_for((int64_t)h->n * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zc.p, h->Zc.p, h->n, h->d, h->DS);
  CKL();
  h->zc_pending_norm = false;
  return 0;
}

// ---- device-memory boundary (hb_setup_device / hb_get_field_device) -------------------------------------------------
// Where a caller buffer lies: *type = cudaMemoryTypeDevice or cudaMemoryTypeManaged of the handle's device, else
// cudaMemoryTypeHost (pageable or pinned).  Another device's memory: status 2.
int memory_type(hb_handle* h, const void* p, const char* what, cudaMemoryType* type) {
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  cudaGetLastError();
  *type = e == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.type : cudaMemoryTypeHost;
  if (*type != cudaMemoryTypeHost && a.device != h->device)
    return fail(h, 2, "%s lives on device %d, the handle on device %d", what, a.device, h->device);
  return 0;
}
// A caller buffer must be device or managed memory of the handle's device: the kernels dereference it directly.
int check_device_ptr(hb_handle* h, const void* p, const char* what) {
  if (!p) return fail(h, 2, "null %s", what);
  cudaMemoryType type;
  TRY(memory_type(h, p, what, &type));
  if (type == cudaMemoryTypeHost)
    return fail(h, 2, "%s is not device or managed memory (host buffers go through hb_setup / hb_get_field)", what);
  return 0;
}
// Where the labels phi_i lie.  NULL is left to setup's checks.
int phi_location(hb_handle* h, const void* p, cudaMemoryType* type) {
  *type = cudaMemoryTypeHost;
  return p ? memory_type(h, p, "phi_i", type) : 0;
}
// A caller's device array of n rows: fp32 or fp64 (enum hb_dtype), row stride ld elements
struct DevRows {
  const void* p;
  int dtype;
  int64_t ld, n;
};
// Caller rows of `cols` values, which the kernels access in place: a known dtype, ld >= cols, device memory (status 2)
int check_rows(hb_handle* h, const DevRows& r, int cols, const char* what) {
  if (r.dtype != HB_FLOAT32 && r.dtype != HB_FLOAT64) return fail(h, 2, "unknown dtype %d of %s", r.dtype, what);
  if (r.ld < cols) return fail(h, 2, "row stride of %s (%lld) is smaller than its %d columns", what, (long long)r.ld, cols);
  return check_device_ptr(h, r.p, what);
}
// f(p) with the rows' pointer as `const float*` or `const double*`, by their checked dtype
template <typename F>
auto with_rows(const DevRows& r, F&& f) {
  return r.dtype == HB_FLOAT32 ? f((const float*)r.p) : f((const double*)r.p);
}
// The element type of the pointer with_rows passes: row_t<decltype(p)> is float or double
template <typename P>
using row_t = std::remove_const_t<std::remove_pointer_t<P>>;
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
// work() on the library stream after the work queued on `caller` so far, and before the work queued there next
template <typename F>
int on_caller_stream(hb_handle* h, cudaStream_t caller, F&& work) {
  TRY(stream_after(h, h->stream, caller));
  TRY(work());
  return stream_after(h, caller, h->stream);
}
// Z (h->n rows of d values) -> Zo in tuple-sorted order, on the library stream after the work queued on `caller`
int upload_rows_device(hb_handle* h, const DevRows& Z, cudaStream_t caller) {
  RegionScope rs(h, "upload");
  TRY(stream_after(h, h->stream, caller));
  with_rows(Z, [&](auto z) { copy_rows(z, Z.ld, h->Zo.p, h->DS, h->inv_sort.p, 0, true, h->n, h->d, h->num_sms, h->stream); });
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
// a host vector into the front of a device buffer of its element type, on the handle's stream
template <typename T>
int upload_vector(hb_handle* h, DevBuf<T>& buf, const std::vector<T>& v) {
  CK(cudaMemcpyAsync(buf.p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, h->stream));
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
