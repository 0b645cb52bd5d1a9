// common.cuh — shared device helpers for libharmony_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define HB_WARP 32

namespace hb {
constexpr float U_PAD = -1.0e30f;  // logit stored in the padding columns of U (exp -> 0)
constexpr int TC_TM = 128;         // cells per tile of the tensor-core kernels (two wgmma M = 64 halves)
// dynamic shared memory a kernel may request: the 227 KB opt-in limit of sm_90 less room for static shared memory
constexpr size_t SMEM_LIMIT = (size_t)227 * 1024 - 256;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Row norms in fp32.  The plain sum of squares underflows for rows below |v| ~ 1e-19 (the squares fall under the
// smallest normal float) and overflows above |v| ~ 1.8e19.  Such sums are rejected by norm_sq_ok, and the row is measured
// again after dividing by its largest magnitude.  That path is rare and costs nothing on ordinary rows.
__device__ __forceinline__ bool norm_sq_ok(float ss) { return ss >= 1.17549435e-38f && ss <= 3.40282347e38f; }
// |x| of n values v(0) .. v(n - 1) held by one thread; 0 for a zero row
template <typename Get>
__device__ __forceinline__ float norm_rescaled(int n, Get v) {
  float m = 0.f;
  for (int i = 0; i < n; ++i) m = fmaxf(m, fabsf(v(i)));
  if (m == 0.f || !isfinite(m)) return m;
  float s = 0.f;
  for (int i = 0; i < n; ++i) {
    const float t = v(i) / m;
    s += t * t;
  }
  return m * sqrtf(s);
}
// the same for a row x[0 .. d) read by a whole warp (lane l reads x[l], x[l + 32], ..); every lane gets the result
__device__ __forceinline__ float warp_norm_rescaled(const float* x, int d, int lane) {
  float m = 0.f;
  for (int c = lane; c < d; c += 32) m = fmaxf(m, fabsf(x[c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (m == 0.f || !isfinite(m)) return m;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) {
    const float t = x[c] / m;
    s += t * t;
  }
  return m * sqrtf(warp_sum(s));
}

// Single-instruction transcendental approximations (MUFU, flush-to-zero): the intrinsics __expf / __logf /
// __frcp_rn expand to range-handling sequences (extra FSETP / FMUL / branches) that the issue-bound row
// loops cannot afford.  Relative error ~2^-22.
__device__ __forceinline__ float fast_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_log(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y * 0.6931471805599453f;
}

// Streaming (read-once) global loads: keep them out of L1 so the small tables stay resident.
__device__ __forceinline__ float ld_stream(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float4 ld_stream4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(float* p, float v) {
  asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v));
}

// 64-bit mix (splitmix64 finaliser) — round function of the cell-order permutation and the k-means seeder.
__host__ __device__ __forceinline__ uint64_t hb_mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Keyed pseudo-random permutation of [0, n): 6-round balanced Feistel network on 2*half_bits bits with
// cycle walking.  pos = hb_permute(i) plays the role of reverse_index[i] of the reference's
// arma::shuffle (harmony.cpp:272-277): cell i sits at position pos in the round's update order.
__host__ __device__ __forceinline__ uint64_t hb_permute(uint64_t i, uint64_t n, int half_bits, uint64_t key) {
  const uint64_t mask = (1ull << half_bits) - 1ull;
  uint64_t x = i;
  do {
    uint64_t l = x >> half_bits, r = x & mask;
#pragma unroll
    for (int round = 0; round < 6; ++round) {
      uint64_t f = hb_mix64(r ^ (key + 0x632BE59BD9B4E019ull * (uint64_t)(round + 1))) & mask;
      uint64_t nl = r;
      r = l ^ f;
      l = nl;
    }
    x = (l << half_bits) | r;
  } while (x >= n);
  return x;
}

// Inverse of hb_permute: the cell that sits at position `pos`.
__host__ __device__ __forceinline__ uint64_t hb_permute_inv(uint64_t pos, uint64_t n, int half_bits, uint64_t key) {
  const uint64_t mask = (1ull << half_bits) - 1ull;
  uint64_t x = pos;
  do {
    uint64_t l = x >> half_bits, r = x & mask;
#pragma unroll
    for (int round = 5; round >= 0; --round) {
      // forward round: (l, r) -> (r, l ^ f(r));  inverse: (l', r') -> (r' ^ f(l'), l')
      uint64_t f = hb_mix64(l ^ (key + 0x632BE59BD9B4E019ull * (uint64_t)(round + 1))) & mask;
      uint64_t pl = r ^ f;
      r = l;
      l = pl;
    }
    x = (l << half_bits) | r;
  } while (x >= n);
  return x;
}
