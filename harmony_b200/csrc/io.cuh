// io.cuh — the per-cell row transfers at the library's boundary (sm_90a): every upload of Z / Z_corr / R into the
// tuple-sorted device rows and every download back into the caller's cell order goes through k_copy_rows.
//
//   upload   (map_dst): dst[map[map0 + r]][c] = (TD) src[r][c]
//   download (!map_dst): dst[r][c]           = (TD) src[map[map0 + r]][c]      r < rows, c < cols
//
// A sub-warp of `lanes` threads (a power of two, <= 32) moves one whole row; each lane moves V consecutive elements
// per access (V * sizeof(T) bytes, 8 or 16-byte accesses where both sides' base address and row stride allow it, a
// scalar path otherwise) and the last cols % V elements one by one.  Columns >= cols are never touched, so the zero
// padding of the device rows (d..DS-1, K..KS-1) stays zero.  Offsets are int64 (a 6.25M x 200 R is 1.25e9 floats).
// float <-> double conversions are exact or round to nearest like a C cast, so the result does not depend on V.
#pragma once
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace hb {

template <int BYTES> struct RawVec;
template <> struct RawVec<4> { using type = unsigned; };
template <> struct RawVec<8> { using type = uint2; };
template <> struct RawVec<16> { using type = uint4; };

// V elements of T from / to an address aligned to min(16, V sizeof(T)) bytes, in accesses of at most 16 bytes
template <typename T, int V>
__device__ __forceinline__ void load_elems(const T* p, T (&v)[V]) {
  constexpr int BYTES = V * (int)sizeof(T), W = BYTES < 16 ? BYTES : 16;
  using R = typename RawVec<W>::type;
  R r[BYTES / W];
#pragma unroll
  for (int i = 0; i < BYTES / W; ++i) r[i] = reinterpret_cast<const R*>(p)[i];
  memcpy(v, r, BYTES);
}
template <typename T, int V>
__device__ __forceinline__ void store_elems(T* p, const T (&v)[V]) {
  constexpr int BYTES = V * (int)sizeof(T), W = BYTES < 16 ? BYTES : 16;
  using R = typename RawVec<W>::type;
  R r[BYTES / W];
  memcpy(r, v, BYTES);
#pragma unroll
  for (int i = 0; i < BYTES / W; ++i) reinterpret_cast<R*>(p)[i] = r[i];
}

template <typename TS, typename TD, int V>
__global__ void __launch_bounds__(256) k_copy_rows(const TS* __restrict__ src, int64_t src_ld, TD* __restrict__ dst,
                                                   int64_t dst_ld, const int* __restrict__ map, int64_t map0,
                                                   bool map_dst, int64_t rows, int cols, int lanes_log2) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int lanes = 1 << lanes_log2, sub = (int)(t & (lanes - 1));
  const int64_t stride = ((int64_t)gridDim.x * blockDim.x) >> lanes_log2;
  const int nvec = cols / V, c_tail = nvec * V;
  for (int64_t r = t >> lanes_log2; r < rows; r += stride) {
    const int64_t m = map[map0 + r];
    const TS* s = src + (map_dst ? r : m) * src_ld;
    TD* o = dst + (map_dst ? m : r) * dst_ld;
    for (int j = sub; j < nvec; j += lanes) {
      TS a[V];
      TD b[V];
      load_elems<TS, V>(s + j * V, a);
#pragma unroll
      for (int i = 0; i < V; ++i) b[i] = (TD)a[i];
      store_elems<TD, V>(o + j * V, b);
    }
    for (int c = c_tail + sub; c < cols; c += lanes) o[c] = (TD)s[c];  // the last cols % V elements
  }
}

// widest V in {4, 2, 1} whose accesses are aligned on a side: base address and row stride (in bytes)
template <typename T>
inline bool copy_aligned(const void* p, int64_t ld, int V) {
  const int64_t a = std::min<int64_t>(16, (int64_t)V * (int64_t)sizeof(T));
  return (uintptr_t)p % (uintptr_t)a == 0 && (ld * (int64_t)sizeof(T)) % a == 0;
}
template <typename TS, typename TD>
inline int copy_width(const TS* src, int64_t src_ld, const TD* dst, int64_t dst_ld, int cols) {
  for (int V = 4; V > 1; V >>= 1)
    if (cols >= V && copy_aligned<TS>(src, src_ld, V) && copy_aligned<TD>(dst, dst_ld, V)) return V;
  return 1;
}

// Enqueues k_copy_rows on `stream` (the caller checks the launch).  Sub-warp of the smallest power of two >= the
// row's accesses, so short rows share a warp.
template <typename TS, typename TD>
void copy_rows(const TS* src, int64_t src_ld, TD* dst, int64_t dst_ld, const int* map, int64_t map0, bool map_dst,
               int64_t rows, int cols, int num_sms, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return;
  const int V = copy_width(src, src_ld, dst, dst_ld, cols);
  const int acc = (cols + V - 1) / V;
  int lanes_log2 = 0;
  while ((1 << lanes_log2) < acc && lanes_log2 < 5) ++lanes_log2;
  const int threads = 256;
  const int64_t want = (rows << lanes_log2) / threads + 1;
  const int grid = (int)std::min<int64_t>(want, (int64_t)num_sms * 64);
#define HB_COPY(VV) \
  k_copy_rows<TS, TD, VV><<<grid, threads, 0, stream>>>(src, src_ld, dst, dst_ld, map, map0, map_dst, rows, cols, lanes_log2)
  if (V == 4)
    HB_COPY(4);
  else if (V == 2)
    HB_COPY(2);
  else
    HB_COPY(1);
#undef HB_COPY
}

}  // namespace hb
