// plan.cuh — the update-order plan of update_R (replaces the physical shuffles of harmony.cpp:272-291): a round's
// cells sorted by (block, tuple, block in the next round) and the tables derived from that order.  The kernels that
// build it and the host code that owns it; included by harmony_b200.cu once hb_handle and its helpers exist.
#pragma once
#include "common.cuh"

namespace hb {

// Injected order: for global position p, cell update_order[p] belongs to block min(p/cpb, nb-1).
__global__ void k_plan_block_injected(const int64_t* __restrict__ update_order, int64_t N_global, int64_t cell_offset,
                                      int64_t n_local, const int* __restrict__ inv_sort, uint32_t cpb, int nb,
                                      int* __restrict__ blk_of, int* __restrict__ err_flag) {
  update_order += (size_t)blockIdx.y * (size_t)N_global;  // blockIdx.y: round of the call
  blk_of += (size_t)blockIdx.y * (size_t)n_local;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < N_global;
       p += (int64_t)gridDim.x * blockDim.x) {
    int64_t g = update_order[p];
    if (g < 0 || g >= N_global) {
      atomicExch(err_flag, 1);
      continue;
    }
    int64_t l = g - cell_offset;
    if (l < 0 || l >= n_local) continue;
    int64_t b = p / cpb;
    if (b > nb - 1) b = nb - 1;
    blk_of[inv_sort[l]] = (int)b;
  }
}
// Native order: position of global cell g is hb_permute(g) (a keyed bijection of [0, N)); the key of a round
// depends on (seed, round counter) only.  blockIdx.y: round of the call.
__host__ __device__ __forceinline__ uint64_t plan_round_key(uint64_t seed, uint64_t round_counter) {
  return hb_mix64(seed ^ hb_mix64(round_counter + 0x1234567ull));
}
__global__ void k_plan_block_native(int64_t N_global, int64_t cell_offset, int64_t n_local,
                                    const int* __restrict__ sort_perm, uint32_t cpb, int nb, int half_bits,
                                    uint64_t seed, uint64_t round_counter0, int* __restrict__ blk_of) {
  const uint64_t key = plan_round_key(seed, round_counter0 + blockIdx.y);
  blk_of += (size_t)blockIdx.y * (size_t)n_local;
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < n_local;
       s += (int64_t)gridDim.x * blockDim.x) {
    uint64_t g = (uint64_t)(cell_offset + sort_perm[s]);
    uint64_t pos = hb_permute(g, (uint64_t)N_global, half_bits, key);
    uint64_t b = pos / cpb;
    if (b > (uint64_t)(nb - 1)) b = nb - 1;
    blk_of[s] = (int)b;
  }
}
// Sort key of a cell in round t: (block in round t, tuple, block in round t+1, chunk, cell).  Chunks are runs of
// consecutive (tuple-sorted) cells of one tuple, so with the histogram laid out as
//   H[blk][ nsub * cq0[c] + sub * cnq[c] + (c - cq0[c]) ]      (cq0 / cnq: first chunk / #chunks of c's tuple)
// one plain exclusive scan of H yields the offsets of that order (nsub = nb, sub = next-round block; nsub = 1
// switches the third key off).
__device__ __forceinline__ size_t plan_hidx(int blk, int sub, int c, int nchunks, int nsub, const int* __restrict__ cq0,
                                            const int* __restrict__ cnq) {
  const int c0 = cq0[c];
  return (size_t)blk * nsub * nchunks + (size_t)nsub * c0 + (size_t)sub * cnq[c] + (c - c0);
}
// One warp per chunk: H[..] = #cells of the chunk with (block, next-round block) = (blk, sub).
__global__ void k_plan_hist(const int* __restrict__ blk_of, const int* __restrict__ chunk_start, const int* __restrict__ cq0,
                            const int* __restrict__ cnq, int nchunks, int nb, int nsub, int* __restrict__ H,
                            int* __restrict__ err_flag, int64_t n_local, int rounds_with_next) {
  extern __shared__ int sh[];
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* cnt = sh + warp * nb * nsub;
  int c = blockIdx.x * (blockDim.x >> 5) + warp;
  if (c >= nchunks) return;
  // blockIdx.y: round of the batch (rounds are n_local apart in blk_of; the next round's blocks follow a round's)
  blk_of += (size_t)blockIdx.y * (size_t)n_local;
  const int* blk_next = ((int)blockIdx.y < rounds_with_next) ? blk_of + n_local : nullptr;
  H += (size_t)blockIdx.y * (size_t)nb * nsub * nchunks;
  for (int j = lane; j < nb * nsub; j += 32) cnt[j] = 0;
  __syncwarp();
  int s0 = chunk_start[c], s1 = chunk_start[c + 1];
  for (int s = s0 + lane; s < s1; s += 32) {
    const int b = blk_of[s];
    if (b < 0 || b >= nb) {  // an injected update order that is not a permutation left this cell without a block
      atomicCAS(err_flag, 0, 3);  // an out-of-range index (flag 1) is the more specific report
      continue;
    }
    const int sub = (nsub > 1 && blk_next) ? blk_next[s] : 0;
    atomicAdd(cnt + b * nsub + ((sub >= 0 && sub < nsub) ? sub : 0), 1);
  }
  __syncwarp();
  for (int j = lane; j < nb * nsub; j += 32) H[plan_hidx(j / nsub, j % nsub, c, nchunks, nsub, cq0, cnq)] = cnt[j];
}
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
// Stable scatter: order[offset(key, chunk) + rank] = cell, cells of a chunk visited in ascending order;
// next_at[same position] = block of the cell in the next round, prev_at = its block in the previous round.
__global__ void k_plan_scatter(const int* __restrict__ blk_of, const int* __restrict__ chunk_start, const int* __restrict__ cq0,
                               const int* __restrict__ cnq, int nchunks, int nb, int nsub, const int* __restrict__ Hoff,
                               int* __restrict__ order, int* __restrict__ prev_at, int* __restrict__ next_at,
                               int64_t n_local, int rounds_with_next, int first_has_prev) {
  extern __shared__ int sh[];
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* cur = sh + warp * nb * nsub;
  int c = blockIdx.x * (blockDim.x >> 5) + warp;
  if (c >= nchunks) return;
  const int *blk_next, *blk_prev;
  {  // blockIdx.y: round of the batch (rounds are n_local apart in blk_of)
    const size_t ro = (size_t)blockIdx.y * (size_t)n_local;
    blk_of += ro;
    blk_next = ((int)blockIdx.y < rounds_with_next) ? blk_of + n_local : nullptr;
    blk_prev = (blockIdx.y > 0 || first_has_prev) ? blk_of - n_local : nullptr;
    Hoff += (size_t)blockIdx.y * (size_t)nb * nsub * nchunks;
    order += ro;
    if (prev_at) prev_at += ro;
    if (next_at) next_at += ro;
  }
  for (int j = lane; j < nb * nsub; j += 32) cur[j] = Hoff[plan_hidx(j / nsub, j % nsub, c, nchunks, nsub, cq0, cnq)];
  __syncwarp();
  int s0 = chunk_start[c], s1 = chunk_start[c + 1];
  for (int base = s0; base < s1; base += 32) {
    int s = base + lane;
    bool act = s < s1;
    int b = act ? blk_of[s] : -1;
    act = act && b >= 0 && b < nb;  // cells without a block were flagged by k_plan_hist
    int nx = (act && blk_next) ? blk_next[s] : 0;
    if (nx < 0 || nx >= nb) nx = 0;
    int key = act ? b * nsub + (nsub > 1 ? nx : 0) : -1 - lane;  // inactive lanes get unique keys
    unsigned m = __match_any_sync(0xffffffffu, key);
    int rank = __popc(m & ((1u << lane) - 1u));
    int leader = __ffs(m) - 1;
    int start = 0;
    if (act && lane == leader) {
      start = cur[key];
      cur[key] = start + __popc(m);
    }
    start = __shfl_sync(0xffffffffu, start, leader);
    if (act) {
      order[start + rank] = s;
      if (prev_at) prev_at[start + rank] = blk_prev ? blk_prev[s] : 0;
      if (next_at) next_at[start + rank] = nx;
    }
    __syncwarp();
  }
}
// Segment (block, tuple) boundaries: seg s = blk*J + q starts at the offset of (blk, first chunk of q, sub 0).
__global__ void k_plan_segments(const int* __restrict__ Hoff, const int* __restrict__ tuple_chunk0, int nchunks,
                                int nb, int nsub, int J, int n_local, int* __restrict__ seg_start) {
  int S = nb * J;
  Hoff += (size_t)blockIdx.y * (size_t)nb * nsub * nchunks;  // blockIdx.y: round of the batch
  seg_start += (size_t)blockIdx.y * (S + 1);
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= S; s += gridDim.x * blockDim.x) {
    int v;
    if (s == S) {
      v = n_local;
    } else {
      int blk = s / J, q = s - blk * J;
      int c = tuple_chunk0[q];  // first chunk of tuple q (tuples without local cells point at the first later chunk)
      v = Hoff[(size_t)blk * nsub * nchunks + (size_t)nsub * c];
    }
    seg_start[s] = v;
  }
}
// Tuple-aligned work split of every block for the persistent update kernel (G CTAs): each CTA gets a contiguous
// slice of ONE (block, tuple) segment.  The block step ends when its most loaded CTA does, so the CTAs are dealt out
// to minimise the largest slice: every non-empty segment starts with one CTA and the remaining ones go, one at a
// time, to the segment with the most rows per CTA (exact comparison L_a n_b > L_b n_a; ties to the lower tuple).
// One CTA (256 threads) per (block j = blockIdx.x, round = blockIdx.y); J <= 2 J <= G <= 1024.
constexpr int PLAN_MAXJ = 512;
__global__ void __launch_bounds__(256) k_plan_ranges(const int* __restrict__ seg_start, int nb, int J, int G,
                                                     int4* __restrict__ ranges) {
  __shared__ int L[PLAN_MAXJ], nq[PLAN_MAXJ], first[PLAN_MAXJ + 1];
  seg_start += (size_t)blockIdx.y * ((size_t)nb * J + 1);  // blockIdx.y: round of the batch
  ranges += (size_t)blockIdx.y * (size_t)nb * G;
  const int j = blockIdx.x;
  const int* segs = seg_start + (size_t)j * J;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int q = tid; q < J; q += blockDim.x) {
    L[q] = segs[q + 1] - segs[q];
    nq[q] = L[q] > 0 ? 1 : 0;
  }
  __syncthreads();
  if (tid < 32) {
    int nonempty = 0;
    for (int q = lane; q < J; q += 32) nonempty += nq[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nonempty += __shfl_xor_sync(0xffffffffu, nonempty, o);
    for (int rem = (nonempty > 0) ? G - nonempty : 0; rem > 0; --rem) {
      long long bl = 0, bn = 1;  // best ratio bl / bn of this lane
      int bq = J;
      for (int q = lane; q < J; q += 32)
        if (nq[q] > 0 && (long long)L[q] * bn > bl * (long long)nq[q]) {
          bl = L[q];
          bn = nq[q];
          bq = q;
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const long long ol = __shfl_xor_sync(0xffffffffu, bl, o), on = __shfl_xor_sync(0xffffffffu, bn, o);
        const int oq = __shfl_xor_sync(0xffffffffu, bq, o);
        const long long lhs = ol * bn, rhs = bl * on;
        if (lhs > rhs || (lhs == rhs && oq < bq)) {
          bl = ol;
          bn = on;
          bq = oq;
        }
      }
      if (lane == 0 && bq < J) nq[bq]++;
      __syncwarp();
    }
    if (lane == 0) {
      int c = 0;
      for (int q = 0; q < J; ++q) {
        first[q] = c;
        c += nq[q];
      }
      first[J] = c;
    }
  }
  __syncthreads();
  const int b0 = segs[0];
  for (int c = tid; c < G; c += blockDim.x) {
    int4 out = make_int4(b0, b0, 0, 0);
    if (c < first[J]) {
      int q = 0;
      while (first[q + 1] <= c) ++q;  // J is small
      const int n = nq[q], me = c - first[q];
      out = make_int4(segs[q] + (int)(((long long)L[q] * me) / n), segs[q] + (int)(((long long)L[q] * (me + 1)) / n), q, 0);
    }
    ranges[(size_t)j * G + c] = out;
  }
}
// Tiles of `tile` rows per (block, tuple) segment of a round: the per-step update kernels (TM) and the
// plan-order assignment (128)
__global__ void k_plan_tilecount(const int* __restrict__ seg_start, int S, int tile, int* __restrict__ tile_base) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= S; s += gridDim.x * blockDim.x) {
    int len = (s < S) ? seg_start[s + 1] - seg_start[s] : 0;
    tile_base[s] = (len + tile - 1) / tile;
  }
}
// the 128-row tiles of the segments of a round (the assignment step in plan order)
__global__ void k_plan_tilefill128(const int* __restrict__ seg_start, const int* __restrict__ tile_base, int S, int J,
                                   int* __restrict__ p0, int* __restrict__ len, int* __restrict__ tuple,
                                   int* __restrict__ blk) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const int a = seg_start[s], e = seg_start[s + 1];
    int i = tile_base[s];
    for (int p = a; p < e; p += 128, ++i) {
      p0[i] = p;
      len[i] = min(128, e - p);
      tuple[i] = s % J;
      blk[i] = s / J;
    }
  }
}

}  // namespace hb
namespace {

// The plan of a handle: two buffer sets (the running cluster_cpp call's, and the next call's prebuilt on a side stream)
// of `rounds` rounds each, laid out as DESIGN.md §3 describes.  Which buffers exist follows the kernel paths hb_setup
// chose (hb_setup runs once per handle); the build and plan_round0 test a buffer for the path it serves.
struct Plan {
  int rounds = 0, batch = 1;  // rounds per set; rounds sorted per launch (size of the histogram scratch)
  int nsub = 1;               // third sort key: block in the next round (nb values) or off (1)
  size_t pt_cap = 0;          // 128-row tiles of round 0 per set
  DevBuf<int> blk_of, order, next_at, prev_at, seg_start, tile_base, pt_p0, pt_len, pt_tuple, pt_blk, pt_base;
  DevBuf<int4> ranges;
  DevBuf<int> H;                          // histograms of the counting sort: [batch][nb][nsub][nchunks]
  DevBuf<unsigned long long> scan_state;  // state of the chained scans
  int nchunks = 0;                        // chunks: <= CHUNK consecutive cells of one tuple, + a trailing empty one
  DevBuf<int> chunk_start, chunk_q0, chunk_nq, tuple_chunk0;
  uint64_t round_counter = 0;  // native rounds run since the seed was set, plus any prebuilt (a round's key: seed, counter)
  int set = 0;                 // set of the running cluster_cpp call
  bool next_ready = false;     // the other set holds a prebuilt native plan of next_T rounds
  int next_T = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t done = nullptr;  // recorded on the main stream before a prebuild, then on the side stream after it
  Plan() {
    cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&done, cudaEventDisableTiming);
  }
  ~Plan() {
    cudaStreamSynchronize(stream);
    cudaEventDestroy(done);
    cudaStreamDestroy(stream);
  }
};

// Round 0 of one buffer set; the update kernels step through the rounds themselves.  Null: not on this path.
struct PlanRound0 {
  const int *order, *seg_start, *next_at, *prev_at, *tile_base;  // tile_base: per-step path (set 0)
  const int4* ranges;
  const int *tile_p0, *tile_len, *tile_tuple, *tile_blk, *tile_count;  // plan-order assignment: tiles, their count
};
PlanRound0 plan_round0(const hb_handle* h, int set) {
  const Plan& p = *h->plan;
  const size_t r0 = (size_t)set * p.rounds, n = (size_t)h->n, S1 = (size_t)h->nb * h->J + 1, t0 = set * p.pt_cap;
  auto at = [](const auto& buf, size_t off) { return buf.p ? buf.p + off : nullptr; };
  return {at(p.order, r0 * n),      at(p.seg_start, r0 * S1), at(p.next_at, r0 * n),  at(p.prev_at, r0 * n),
          p.tile_base.p,            at(p.ranges, r0 * h->nb * h->coop_grid),         at(p.pt_p0, t0),
          at(p.pt_len, t0),         at(p.pt_tuple, t0),       at(p.pt_blk, t0),       at(p.pt_base, set * S1 + S1 - 1)};
}

// Buffers of T rounds per set.  The sets start over: a prebuilt plan must have been discarded.
int plan_alloc_rounds(hb_handle* h, int T) {
  Plan& p = *h->plan;
  const size_t rn = 2 * (size_t)T * h->n;
  CK(p.blk_of.alloc(rn));
  CK(p.order.alloc(rn));
  if (h->paths.update != UpdatePath::PerStep) CK((h->paths.update == UpdatePath::SinglePass ? p.next_at : p.prev_at).alloc(rn));
  CK(p.seg_start.alloc(2 * (size_t)T * ((size_t)h->nb * h->J + 1)));
  if (h->paths.update != UpdatePath::PerStep && h->paths.tuple_ranges) CK(p.ranges.alloc(2 * (size_t)T * h->nb * h->coop_grid));
  p.rounds = T;
  p.set = 0;
  return 0;
}

// The chunk tables of the cells sorted by tuple (tuple q: cells [tstart[q], tstart[q + 1])) and the buffers that do
// not depend on the rounds of a call (the histogram scratch holds min(8, T) rounds).
int plan_setup(hb_handle* h, const std::vector<int64_t>& tstart, int T) {
  Plan& p = *h->plan;
  const int J = h->J, nb = h->nb;
  const int64_t n = h->n;
  const size_t S1 = (size_t)nb * J + 1;
  int CHUNK = 1024;  // ~2000 chunks per shard at most (the plan's scan is nb^2 x #chunks long)
  while (CHUNK < 16384 && n / CHUNK > 2048) CHUNK <<= 1;
  std::vector<int> c_start, t_chunk0(J, 0), c_q0, c_nq;
  for (int q = 0; q < J; ++q) {
    t_chunk0[q] = (int)c_start.size();
    for (int64_t s = tstart[q]; s < tstart[q + 1]; s += CHUNK) c_start.push_back((int)s);
    const int nq = (int)c_start.size() - t_chunk0[q];
    c_q0.insert(c_q0.end(), nq, t_chunk0[q]);
    c_nq.insert(c_nq.end(), nq, nq);
  }
  c_q0.push_back((int)c_start.size());  // the trailing empty chunk is a group of its own
  c_nq.push_back(1);
  c_start.insert(c_start.end(), 2, (int)n);  // start and end of the trailing empty chunk
  p.nchunks = (int)c_start.size() - 1;
  // tuples without local cells point at the first later chunk (their segments are empty)
  for (int q = J - 1; q >= 0; --q)
    if (tstart[q + 1] == tstart[q]) t_chunk0[q] = (q + 1 < J) ? t_chunk0[q + 1] : p.nchunks - 1;
  using Table = std::pair<DevBuf<int>*, const std::vector<int>*>;
  for (Table u : {Table{&p.chunk_start, &c_start}, Table{&p.chunk_q0, &c_q0}, Table{&p.chunk_nq, &c_nq}, Table{&p.tuple_chunk0, &t_chunk0}}) {
    CK(u.first->alloc(u.second->size()));
    CK(cudaMemcpyAsync(u.first->p, u.second->data(), sizeof(int) * u.second->size(), cudaMemcpyHostToDevice, h->stream));
  }
  const bool single_pass = h->paths.update == UpdatePath::SinglePass;
  p.nsub = (single_pass && nb <= 64) ? nb : 1;
  p.pt_cap = (size_t)n / TC_TM + (size_t)nb * J + 2;
  if (h->paths.mm.k1_stages && single_pass)
    for (DevBuf<int>* b : {&p.pt_p0, &p.pt_len, &p.pt_tuple, &p.pt_blk}) CK(b->alloc(2 * p.pt_cap));
  CK(p.pt_base.alloc(2 * S1));
  CK(p.tile_base.alloc(S1));
  const size_t per_round = (size_t)nb * p.nsub * p.nchunks;
  p.batch = (int)std::max<size_t>(1, std::min<size_t>({(size_t)8, (size_t)T, ((size_t)16 << 20) / std::max<size_t>(1, per_round)}));
  CK(p.H.alloc(per_round * p.batch));
  auto scan_words = [](size_t len, size_t nseg) { return nseg * ((len + SCAN_TILE - 1) / SCAN_TILE + 1); };
  CK(p.scan_state.alloc(std::max(scan_words(per_round, p.batch), scan_words(S1, 1))));
  return 0;
}

// exclusive scan in place of nseg int arrays of len elements, back to back
int plan_scan(hb_handle* h, int* data, int64_t len, int nseg, cudaStream_t st) {
  const int tiles = (int)((len + SCAN_TILE - 1) / SCAN_TILE);
  CK(cudaMemsetAsync(h->plan->scan_state.p, 0, sizeof(unsigned long long) * (size_t)nseg * (tiles + 1), st));
  k_scan_chained<<<dim3(tiles, nseg), 1024, 0, st>>>(data, len, h->plan->scan_state.p, tiles);
  CKL();
  return 0;
}
// Counting sort of rounds [t, t + nt) of a set (nt <= batch: the histogram scratch holds that many rounds) and the
// derived tables; round t + nt - 1 has a next round iff last_has_next.
int plan_sort(hb_handle* h, int t, int nt, bool last_has_next, int set, cudaStream_t st) {
  Plan& p = *h->plan;
  const int nb = h->nb, J = h->J, nc = p.nchunks, nsub = p.nsub, S = nb * J;
  const int64_t n = h->n;
  const size_t r = (size_t)set * p.rounds + t;
  const int* blk_of = p.blk_of.p + r * n;
  int* seg_start = p.seg_start.p + r * (S + 1);
  const size_t per_warp = sizeof(int) * (size_t)nb * nsub;
  const int wpb = (int)std::max<size_t>(1, std::min<size_t>(8, (48 * 1024) / per_warp));  // warps per block
  const size_t sm = per_warp * wpb;
  const int with_next = last_has_next ? nt : nt - 1;
  k_plan_hist<<<dim3((nc + wpb - 1) / wpb, nt), wpb * 32, sm, st>>>(blk_of, p.chunk_start.p, p.chunk_q0.p, p.chunk_nq.p, nc,
                                                                   nb, nsub, p.H.p, h->err_flag.p, n, with_next);
  CKL();
  // offsets of the counting sort: multi-CTA scan of the nt histograms (a single CTA per round took ~145 us)
  TRY(plan_scan(h, p.H.p, (int64_t)nb * nsub * nc, nt, st));
  k_plan_scatter<<<dim3((nc + wpb - 1) / wpb, nt), wpb * 32, sm, st>>>(
      blk_of, p.chunk_start.p, p.chunk_q0.p, p.chunk_nq.p, nc, nb, nsub, p.H.p, p.order.p + r * n,
      p.prev_at.p ? p.prev_at.p + r * n : nullptr, p.next_at.p ? p.next_at.p + r * n : nullptr, n, with_next, t > 0);
  CKL();
  k_plan_segments<<<dim3(grid_for(S + 1, 256, 64), nt), 256, 0, st>>>(p.H.p, p.tuple_chunk0.p, nc, nb, nsub, J, (int)n,
                                                                       seg_start);
  CKL();
  if (p.ranges.p) {
    k_plan_ranges<<<dim3(nb, nt), 256, 0, st>>>(seg_start, nb, J, h->coop_grid, p.ranges.p + r * nb * h->coop_grid);
    CKL();
  }
  return 0;
}
// T rounds into a set (orders_d: device, T x N_global, or null for the native orders), and the tiles of round 0: the
// per-step kernels' (step: one round into set 0, the per-step update path) or the plan-order assignment's.
int build_plans(hb_handle* h, int T, const int64_t* orders_d, int set, cudaStream_t st, bool step = false) {
  if (T <= 0) return 0;
  RegionScope rs(h, "plan");
  Plan& p = *h->plan;
  const int64_t n = h->n;
  const int S = h->nb * h->J;
  // the block of every local cell in every round (harmony.cpp:272-291: position in the shuffled order / cells per block)
  int* blk_of = p.blk_of.p + (size_t)set * p.rounds * n;
  if (orders_d) {
    CK(cudaMemsetAsync(blk_of, 0xff, sizeof(int) * (size_t)n * T, st));
    k_plan_block_injected<<<dim3(grid_for(h->N_global, 256, h->num_sms * 8), T), 256, 0, st>>>(
        orders_d, h->N_global, h->cell_offset, n, h->inv_sort.p, h->cpb, h->nb, blk_of, h->err_flag.p);
  } else {
    k_plan_block_native<<<dim3(grid_for(n, 256, h->num_sms * 8), T), 256, 0, st>>>(
        h->N_global, h->cell_offset, n, h->sort_perm.p, h->cpb, h->nb, h->half_bits, h->seed, p.round_counter, blk_of);
  }
  CKL();
  if (!orders_d) p.round_counter += (uint64_t)T;  // injected orders take no native rounds
  for (int t = 0; t < T; t += p.batch) TRY(plan_sort(h, t, std::min(p.batch, T - t), t + p.batch < T, set, st));
  const PlanRound0 r = plan_round0(h, set);
  int* base = step ? p.tile_base.p : p.pt_base.p + (size_t)set * (S + 1);
  if (!step && !p.pt_p0.p) return 0;
  k_plan_tilecount<<<grid_for(S + 1, 256, 64), 256, 0, st>>>(r.seg_start, S, step ? TM : 128, base);
  CKL();
  TRY(plan_scan(h, base, (int64_t)S + 1, 1, st));  // base[S]: the number of tiles
  if (!step) {  // 128-row tiles, one (block, tuple) segment at a time: the cold-start assignment runs in this order
    k_plan_tilefill128<<<grid_for(S, 128, 64), 128, 0, st>>>(r.seg_start, base, S, h->J, p.pt_p0.p + set * p.pt_cap,
                                                             p.pt_len.p + set * p.pt_cap, p.pt_tuple.p + set * p.pt_cap,
                                                             p.pt_blk.p + set * p.pt_cap);
    CKL();
  }
  return 0;
}

// ---- the next-call protocol ----------------------------------------------------------------------------------
// Drop a prebuilt plan: its rounds were never run, so the next native plan draws them again.
int plan_discard(hb_handle* h) {
  Plan& p = *h->plan;
  if (!p.next_ready) return 0;
  CK(cudaStreamWaitEvent(h->stream, p.done, 0));  // the main stream's next plan build reuses the scan scratch
  p.round_counter -= (uint64_t)p.next_T;
  p.next_ready = false;
  return 0;
}
// This T-round call's plan (persistent update paths): the prebuilt one if it holds native orders of >= T rounds,
// else a new one in the current set.
int plan_acquire(hb_handle* h, int T, const int64_t* orders_d) {
  Plan& p = *h->plan;
  if (p.next_ready && !orders_d && p.next_T >= T) {
    CK(cudaStreamWaitEvent(h->stream, p.done, 0));
    p.set ^= 1;
    p.next_ready = false;
    return 0;
  }
  TRY(plan_discard(h));
  return build_plans(h, T, orders_d, p.set, h->stream);
}
// The native plan of a next T-round call, into the other set on the side stream once this call's own plan build and
// update kernel (main stream) are done with the shared scan scratch.
int plan_prebuild(hb_handle* h, int T) {
  Plan& p = *h->plan;
  CK(cudaEventRecord(p.done, h->stream));
  CK(cudaStreamWaitEvent(p.stream, p.done, 0));
  TRY(build_plans(h, T, nullptr, p.set ^ 1, p.stream));
  CK(cudaEventRecord(p.done, p.stream));
  p.next_ready = true;
  p.next_T = T;
  return 0;
}

}  // namespace
