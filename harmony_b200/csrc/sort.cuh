// sort.cuh — the chained exclusive scan and the stable LSD radix sort of int codes built on it: the kernels and the one
// host driver of each (chained_scan, sort_by_code).  The update-order plan scans with it, the covariate-tuple index
// sorts the cells by tuple id and hb_umap_graph / hb_leiden do every grouping with it.  Included by harmony_b200.cu
// after handle.cuh and before plan.cuh.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int TI_CHUNK = 2048;  // cells per warp in the radix passes
constexpr int TI_WARPS = 8;     // warps (chunks) per CTA of the radix passes

// Exclusive scan of `nseg` independent int arrays of n elements (back to back in `data`, in place) by many CTAs:
// chained scan with dynamic tile numbers.  A CTA draws the next tile (8192 elements) of its segment from a counter
// — so a tile's predecessor has always been drawn, i.e. runs or has run: no deadlock whatever the dispatch order —,
// scans it locally, waits for the inclusive prefix of the tile before it, publishes its own (value and flag in one
// 64-bit word) and writes the results.  state: [nseg][1 + tiles] words, zeroed by the caller (word 0: the counter).
constexpr int SCAN_TILE = 8192;  // 1024 threads x 8 elements
__global__ void __launch_bounds__(1024) k_scan_chained(int* __restrict__ data, int64_t n, unsigned long long* __restrict__ state,
                                                       int tiles_per_seg) {
  __shared__ int wsum[32];
  __shared__ int sh_tile, sh_carry;
  const int seg = blockIdx.y;
  data += (size_t)seg * (size_t)n;
  unsigned long long* st = state + (size_t)seg * (tiles_per_seg + 1);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) sh_tile = (int)atomicAdd(st, 1ull);
  __syncthreads();
  const int tile = sh_tile;
  if (tile >= tiles_per_seg) return;
  const int64_t base = (int64_t)tile * SCAN_TILE + (int64_t)tid * 8;
  int v[8];
  int s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = (base + i < n) ? data[base + i] : 0;
    s += v[i];
  }
  // exclusive scan of the threads' sums within the CTA
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const int w = wsum[lane];
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    wsum[lane] = winc - w;  // exclusive prefix of the warps
    if (lane == 31) {
      // tile aggregate = winc; chain: inclusive prefix of this tile = prefix of the previous one + aggregate
      int carry = 0;
      if (tile > 0) {
        unsigned long long p;
        do {
          asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(p) : "l"(st + tile) : "memory");  // word 1 + (tile - 1)
        } while ((p >> 32) == 0ull);
        carry = (int)(unsigned)(p & 0xffffffffull);
      }
      const unsigned long long mine = (1ull << 32) | (unsigned)(carry + winc);
      asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(st + tile + 1), "l"(mine) : "memory");
      sh_carry = carry;
    }
  }
  __syncthreads();
  int run = sh_carry + wsum[warp] + (inc - s);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (base + i < n) data[base + i] = run;
    run += v[i];
  }
}

// ---- stable LSD radix sort of int keys, 8-bit digits.  One warp per chunk of TI_CHUNK cells; the digit histograms
// are laid out digit-major, H[digit * nchunks + chunk], so that one exclusive scan of H gives every (digit, chunk) its
// first output position.
__global__ void __launch_bounds__(TI_WARPS * 32) k_radix_hist(const int* __restrict__ key, int64_t n, int shift,
                                                              int nchunks, int* __restrict__ H) {
  __shared__ int cnt[TI_WARPS][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * TI_WARPS + warp;
  if (c >= nchunks) return;
  for (int j = lane; j < 256; j += 32) cnt[warp][j] = 0;
  __syncwarp();
  const int64_t s0 = (int64_t)c * TI_CHUNK, s1 = min(n, s0 + TI_CHUNK);
  for (int64_t s = s0 + lane; s < s1; s += 32) atomicAdd(&cnt[warp][(key[s] >> shift) & 255], 1);
  __syncwarp();
  for (int j = lane; j < 256; j += 32) H[(size_t)j * nchunks + c] = cnt[warp][j];
}
// The chunk's cells in ascending order, 32 at a time: lanes with the same digit are ranked by lane (match), so equal
// digits keep their input order.  val_in null: the values are the positions (the first pass).  inv non-null (the
// last pass): inv[value] = output position.
__global__ void __launch_bounds__(TI_WARPS * 32) k_radix_scatter(const int* __restrict__ key_in, const int* __restrict__ val_in,
                                                                 int64_t n, int shift, int nchunks, const int* __restrict__ Hoff,
                                                                 int* __restrict__ key_out, int* __restrict__ val_out,
                                                                 int* __restrict__ inv) {
  __shared__ int cur[TI_WARPS][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * TI_WARPS + warp;
  if (c >= nchunks) return;
  for (int j = lane; j < 256; j += 32) cur[warp][j] = Hoff[(size_t)j * nchunks + c];
  __syncwarp();
  const int64_t s0 = (int64_t)c * TI_CHUNK, s1 = min(n, s0 + TI_CHUNK);
  for (int64_t base = s0; base < s1; base += 32) {
    const int64_t s = base + lane;
    const bool act = s < s1;
    const int k = act ? key_in[s] : 0;
    const int v = act ? (val_in ? val_in[s] : (int)s) : 0;
    const int dig = act ? (k >> shift) & 255 : 256 + lane;  // inactive lanes get keys of their own
    const unsigned m = __match_any_sync(0xffffffffu, dig);
    const int leader = __ffs(m) - 1;
    int start = 0;
    if (act && lane == leader) {
      start = cur[warp][dig];
      cur[warp][dig] = start + __popc(m);
    }
    start = __shfl_sync(0xffffffffu, start, leader);
    if (act) {
      const int p = start + __popc(m & ((1u << lane) - 1u));
      key_out[p] = k;
      val_out[p] = v;
      if (inv) inv[v] = p;
    }
    __syncwarp();
  }
}
// J = 1: every cell keeps its place
__global__ void k_identity_perm(int64_t n, int* __restrict__ perm, int* __restrict__ inv) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    perm[i] = (int)i;
    inv[i] = (int)i;
  }
}
// tstart[q] = first sorted position of tuple q, tstart[J] = n (tuples without local cells start where the next does)
__global__ void k_tuple_starts(const int* __restrict__ sorted, int64_t n, int J, int* __restrict__ tstart) {
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s <= n; s += (int64_t)gridDim.x * blockDim.x) {
    const int prev = s > 0 ? sorted[s - 1] : -1, cur = s < n ? sorted[s] : J;
    for (int q = prev + 1; q <= cur; ++q) tstart[q] = (int)s;
  }
}

}  // namespace hb
namespace {

// Exclusive scan in place of nseg int arrays of len elements, back to back, on `st`.  `state` is grown to and zeroed
// over nseg * (tiles + 1) words; no other scan may use it while this one runs.
int chained_scan(hb_handle* h, cudaStream_t st, int* data, int64_t len, int nseg, DevBuf<unsigned long long>& state) {
  const int tiles = (int)((len + SCAN_TILE - 1) / SCAN_TILE);
  const size_t words = (size_t)nseg * (tiles + 1);
  CK(state.reserve(words));
  CK(cudaMemsetAsync(state.p, 0, sizeof(unsigned long long) * words, st));
  k_scan_chained<<<dim3(tiles, nseg), 1024, 0, st>>>(data, len, state.p, tiles);
  CKL();
  return 0;
}

// The scratch of sort_by_code, grown on demand: the keys' second buffer, the values between passes, the digit
// histograms and the chain state of their scans
struct SortScratch {
  DevBuf<int> key, val[2], hist;
  DevBuf<unsigned long long> scan;
};

// Stable sort of the n codes in `key` (each in [0, n_codes); overwritten) on h->stream, ceil(log2(n_codes) / 8)
// passes of 8 bits: vin (null: the positions) into vout in the codes' order; inv (if not null) gets each value's
// sorted position, and starts (if not null) the n_codes + 1 first sorted positions of the codes.  With no pass, vout
// is a copy of vin, or the positions (and so is inv, or s.val[0]).  n = 0 sorts nothing.
int sort_by_code(hb_handle* h, SortScratch& s, int* key, int64_t n, int n_codes, const int* vin, int* vout, int* inv,
                 int* starts) {
  const cudaStream_t st = h->stream;
  int bits = 0;
  while (bits < 31 && (1ll << bits) < (long long)n_codes) ++bits;
  const int passes = (bits + 7) / 8;
  int* kin = key;
  if (n > 0 && passes == 0) {
    if (vin) {
      CK(cudaMemcpyAsync(vout, vin, sizeof(int) * n, cudaMemcpyDeviceToDevice, st));
    } else {
      if (!inv) CK(s.val[0].reserve((size_t)n));
      k_identity_perm<<<grid_for(n, 256, h->num_sms * 8), 256, 0, st>>>(n, vout, inv ? inv : s.val[0].p);
      CKL();
    }
  } else if (n > 0) {
    const int nchunks = (int)((n + TI_CHUNK - 1) / TI_CHUNK);
    const int cta = (nchunks + TI_WARPS - 1) / TI_WARPS;
    CK(s.key.reserve((size_t)n));
    if (passes > 1) CK(s.val[0].reserve((size_t)n));
    if (passes > 2) CK(s.val[1].reserve((size_t)n));
    CK(s.hist.reserve((size_t)256 * nchunks));
    int* kout = s.key.p;
    const int* v = vin;
    for (int p = 0; p < passes; ++p) {
      const bool last = p == passes - 1;
      int* vo = last ? vout : s.val[p & 1].p;
      k_radix_hist<<<cta, TI_WARPS * 32, 0, st>>>(kin, n, 8 * p, nchunks, s.hist.p);
      CKL();
      TRY(chained_scan(h, st, s.hist.p, (int64_t)256 * nchunks, 1, s.scan));
      k_radix_scatter<<<cta, TI_WARPS * 32, 0, st>>>(kin, v, n, 8 * p, nchunks, s.hist.p, kout, vo, last ? inv : nullptr);
      CKL();
      v = vo;
      std::swap(kin, kout);
    }
  }
  if (starts) {
    k_tuple_starts<<<grid_for(n + 1, 256, h->num_sms * 8), 256, 0, st>>>(kin, n, n_codes, starts);
    CKL();
  }
  return 0;
}

}  // namespace
