// components.cuh — connected components of a neighbour graph (DESIGN §12), sm_90a.  The graph is the symmetric
// closure of idx [N][k] (row stride idx_ld, -1: no neighbour), optionally cut between rows of different labels.
//   k_cc_check     read-only range pass: the smallest row (k + 1) + m of an entry m < k outside -1..N-1, or of a label
//                  (m = k) outside 0..n_labels-1
//   k_cc_init      parent[i] = i (the caller's comp is the parent array)
//   k_cc_hook      lock-free union-find, one thread per entry: the larger root is linked under the smaller by CAS
//   k_cc_compress  comp[i] = the root of i, the smallest row of its component
//   k_cc_count     size[root] += 1, warp-aggregated over lanes with the same root
//   k_cc_largest   largest[label[r]] = max size over the roots r of that label
#pragma once
#include <cuda/atomic>

#include "common.cuh"

namespace hb {

// Every read of the parent array while links are being made is a relaxed device-scope atomic load: a plain load may
// be served from a stale L1 line or hoisted out of the retry loop, and the loop would never see another SM's link.
__device__ __forceinline__ int cc_load(int* parent, int v) {
  return cuda::atomic_ref<int, cuda::thread_scope_device>(parent[v]).load(cuda::memory_order_relaxed);
}
__device__ __forceinline__ void cc_store(int* parent, int v, int p) {
  cuda::atomic_ref<int, cuda::thread_scope_device>(parent[v]).store(p, cuda::memory_order_relaxed);
}

// The root of v, halving the path on the way.  Invariant: every non-root has parent[v] < v and parent[v] in v's set.
// A halving store writes v's grandparent, an ancestor smaller than v, so the invariant holds under any interleaving;
// roots are only ever written by the CAS of cc_union (a non-root never becomes a root again), so a halving store never
// overwrites a link.  The root is therefore the smallest row of its tree, and there are no cycles.
__device__ __forceinline__ int cc_find(int* parent, int v) {
  for (;;) {
    const int p = cc_load(parent, v);
    if (p == v) return v;
    const int gp = cc_load(parent, p);
    if (gp != p) cc_store(parent, v, gp);
    v = gp;
  }
}

// Joins the sets of a and b: the larger root goes under the smaller.  A failed CAS means another thread linked rb
// first, so some union made progress: the loop is lock-free and no thread waits on another.
__device__ __forceinline__ void cc_union(int* parent, int a, int b) {
  for (;;) {
    a = cc_find(parent, a);
    b = cc_find(parent, b);
    if (a == b) return;
    const int ra = min(a, b), rb = max(a, b);
    if (atomicCAS(parent + rb, rb, ra) == rb) return;
    a = ra;
    b = rb;
  }
}

__global__ void __launch_bounds__(256) k_cc_check(const int32_t* __restrict__ idx, int64_t idx_ld, int64_t N, int k,
                                                  const int32_t* __restrict__ labels, int n_labels,
                                                  unsigned long long* __restrict__ bad) {
  const int64_t k1 = (int64_t)k + 1, total = N * k1;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / k1;
    const int m = (int)(t - i * k1);
    bool ok;
    if (m < k) {
      const int j = idx[i * idx_ld + m];
      ok = j >= -1 && j < N;
    } else {
      ok = !labels || (labels[i] >= 0 && labels[i] < n_labels);
    }
    if (!ok) atomicMin(bad, (unsigned long long)t);
  }
}

__global__ void __launch_bounds__(256) k_cc_init(int64_t N, int* __restrict__ parent) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x)
    parent[i] = (int)i;
}

// One thread per entry (int64 entry indices: N k passes 2^31).  Skipped: -1, self entries and, with labels, edges
// between rows of different labels.
__global__ void __launch_bounds__(256) k_cc_hook(const int32_t* __restrict__ idx, int64_t idx_ld, int64_t N, int k,
                                                 const int32_t* __restrict__ labels, int* parent) {
  const int64_t total = N * k;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / k;
    const int j = idx[i * idx_ld + (e - i * k)];
    if (j < 0 || j == i) continue;
    if (labels && labels[i] != labels[j]) continue;
    cc_union(parent, (int)i, j);
  }
}

// After every link (the kernel boundary orders it after k_cc_hook): comp[i] = root(i).  A thread's own store races
// with other threads' walks through i, which then read either i's old parent or its root: both ancestors.
__global__ void __launch_bounds__(256) k_cc_compress(int64_t N, int* comp) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    int r = (int)i, p;
    while ((p = cc_load(comp, r)) != r) r = p;
    cc_store(comp, (int)i, r);
  }
}

// size[comp[i]] += 1, one atomic per distinct root among a warp's 32 rows: one large component costs N / 32 atomics
// on its root's word, not N
__global__ void __launch_bounds__(256) k_cc_count(const int* __restrict__ comp, int64_t N, int* __restrict__ size) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i0 = warp * 32; i0 < N; i0 += warps * 32) {  // warp-uniform bound: every lane takes part in the ballot
    const int64_t i = i0 + lane;
    const unsigned active = __ballot_sync(0xffffffffu, i < N);
    if (i < N) {
      const int r = comp[i];
      const unsigned peers = __match_any_sync(active, r);
      if (lane == __ffs(peers) - 1) atomicAdd(size + r, __popc(peers));
    }
  }
}

// For every root r: largest[label[r]] = max(largest[label[r]], size[r]) (label 0 without labels).  A component lies
// within one label, so its root's label is its label.
__global__ void __launch_bounds__(256) k_cc_largest(const int* __restrict__ comp, const int* __restrict__ size,
                                                    const int32_t* __restrict__ labels, int64_t N,
                                                    int* __restrict__ largest) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x)
    if (comp[i] == i) atomicMax(largest + (labels ? labels[i] : 0), size[i]);
}

}  // namespace hb
