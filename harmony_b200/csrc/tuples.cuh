// tuples.cuh — the covariate-tuple index of setup (and of hb_silhouette's (group, label) pairs), built on the device:
// each cell's key (the mixed-radix number of its C levels, covariate 0 most significant), the level counts, the
// dictionary of the distinct keys (tuple ids 0..J-1 in ascending key order), each cell's tuple id, and the stable sort
// of the cells by tuple id (sort_perm, inv_sort, tstart).  The kernels and the host code that drives them; the scan of
// the dictionary and the sort are sort.cuh's.  Included by harmony_b200.cu after sort.cuh.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int TI_HASH_LOG2 = 21;                      // 2^21 = 2,097,152 hash slots: load <= 0.48 at the 1e6 tuple limit
constexpr uint32_t TI_SLOTS = 1u << TI_HASH_LOG2;
constexpr int TI_MAX_PROBE = 512;                     // a longer probe sequence counts as a full table
constexpr unsigned long long TI_EMPTY = ~0ull;        // no key reaches it (the level product is <= 9e18)
constexpr int TI_SMEM_LEVELS = 8192;                  // level counts in shared memory up to this many levels

__device__ __forceinline__ uint32_t ti_home(uint64_t key) { return (uint32_t)(hb_mix64(key) >> (64 - TI_HASH_LOG2)); }

// Open addressing with linear probing.  A slot goes from TI_EMPTY to a key once, so a key read is final and a stale
// TI_EMPTY only costs the CAS.  false: no slot within TI_MAX_PROBE.
__device__ __forceinline__ bool ti_insert(unsigned long long* slots, unsigned long long key) {
  uint32_t s = ti_home(key);
  for (int p = 0; p < TI_MAX_PROBE; ++p, s = (s + 1) & (TI_SLOTS - 1)) {
    unsigned long long cur = slots[s];
    if (cur == TI_EMPTY) cur = atomicCAS(slots + s, TI_EMPTY, key);
    if (cur == TI_EMPTY || cur == key) return true;
  }
  return false;
}
// Slot of a key inserted by an earlier launch, -1 if absent
__device__ __forceinline__ int ti_find(const unsigned long long* __restrict__ slots, unsigned long long key) {
  uint32_t s = ti_home(key);
  for (int p = 0; p < TI_MAX_PROBE; ++p, s = (s + 1) & (TI_SLOTS - 1)) {
    const unsigned long long cur = slots[s];
    if (cur == key) return (int)s;
    if (cur == TI_EMPTY) return -1;
  }
  return -1;
}

struct TupleKeyArgs {
  const int* phi;                   // [n][C] global level of each (cell, covariate)
  int64_t n;
  int C, B;
  const int* base;                  // [C] first level of covariate c
  const int* nlev;                  // [C] its number of levels
  const unsigned long long* radix;  // [C] weight of covariate c in the key
  unsigned long long* key;          // [n]
  unsigned long long* count;        // [B] cells per level (added to)
  unsigned long long* bad;          // smallest i C + c whose level lies outside covariate c (TI_EMPTY: none)
  int* table;                       // direct dictionary: table[key] = 1 (key spaces <= 2^22), or null
  unsigned long long* slots;        // hash dictionary (TI_SLOTS keys), or null
  int* full;                        // set when a key found no hash slot
};
// One pass over phi: validation, level counts, keys, and every key entered in the dictionary.
__global__ void __launch_bounds__(256) k_tuple_keys(TupleKeyArgs a) {
  __shared__ unsigned int cnt[TI_SMEM_LEVELS];
  const bool shared_counts = a.B <= TI_SMEM_LEVELS;
  if (shared_counts)
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) cnt[b] = 0;
  __syncthreads();
  bool lost = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long key = 0;
    bool ok = true;
    for (int c = 0; c < a.C; ++c) {
      const int b = a.phi[i * a.C + c];
      const int64_t l = (int64_t)b - a.base[c];
      if (l < 0 || l >= a.nlev[c]) {  // the cell's first bad covariate is its smallest i C + c
        atomicMin(a.bad, (unsigned long long)(i * a.C + c));
        ok = false;
        break;
      }
      if (shared_counts)
        atomicAdd(cnt + b, 1u);
      else
        atomicAdd(a.count + b, 1ull);
      key += (unsigned long long)l * a.radix[c];
    }
    if (!ok) continue;
    a.key[i] = key;
    if (a.table)
      a.table[key] = 1;
    else if (!ti_insert(a.slots, key))
      lost = true;
  }
  if (lost) atomicExch(a.full, 1);
  if (!shared_counts) return;
  __syncthreads();
  for (int b = threadIdx.x; b < a.B; b += blockDim.x)
    if (cnt[b]) atomicAdd(a.count + b, (unsigned long long)cnt[b]);
}
// Direct dictionary after the exclusive scan of its marks (space + 1 words): key k is present iff table[k + 1] >
// table[k], and table[k] is then its tuple id.  uniq[table[k]] = k.
__global__ void k_table_keys(const int* __restrict__ table, int64_t space, unsigned long long* __restrict__ uniq) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < space; k += (int64_t)gridDim.x * blockDim.x)
    if (table[k + 1] != table[k]) uniq[table[k]] = (unsigned long long)k;
}
// Occupied hash slots -> keys[0..*count) (in no particular order; the host sorts them)
__global__ void k_hash_compact(const unsigned long long* __restrict__ slots, unsigned long long* __restrict__ keys,
                               int* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  for (uint32_t s0 = blockIdx.x * blockDim.x; s0 < TI_SLOTS; s0 += gridDim.x * blockDim.x) {
    const uint32_t s = s0 + threadIdx.x;
    const unsigned long long k = s < TI_SLOTS ? slots[s] : TI_EMPTY;
    const unsigned m = __ballot_sync(0xffffffffu, k != TI_EMPTY);
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(count, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (k != TI_EMPTY) keys[base + __popc(m & ((1u << lane) - 1u))] = k;
  }
}
// Tuple ids of the ascending keys uniq[0..J): into the direct table, or beside the keys' hash slots.  Keys without a
// local cell (the union of a sharded index) are skipped on the hash path and land in unused table entries.
__global__ void k_tuple_ids(const unsigned long long* __restrict__ uniq, int J, int* __restrict__ table,
                            const unsigned long long* __restrict__ slots, int* __restrict__ slot_id) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < J; q += gridDim.x * blockDim.x) {
    if (table) {
      table[uniq[q]] = q;
    } else {
      const int s = ti_find(slots, uniq[q]);
      if (s >= 0) slot_id[s] = q;
    }
  }
}
// Tuple id of every cell
__global__ void k_tuple_of(const unsigned long long* __restrict__ key, int64_t n, const int* __restrict__ table,
                           const unsigned long long* __restrict__ slots, const int* __restrict__ slot_id,
                           int* __restrict__ tuple_of) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    tuple_of[i] = table ? table[key[i]] : slot_id[ti_find(slots, key[i])];
}

}  // namespace hb
namespace {

// What setup keeps of the index besides sort_perm / inv_sort (which it writes in place): the ascending keys of the
// J tuples, the level counts (summed over the ranks of a sharded handle) and the tuple starts in sorted order.
struct TupleIndex {
  std::vector<uint64_t> uniq;
  std::vector<int64_t> lvl_count;
  std::vector<int64_t> tstart;
};

constexpr size_t TI_MAX_TUPLES = 1000000;
int too_many_tuples(hb_handle* h) { return fail(h, 2, "more than 1e6 distinct covariate tuples are not supported"); }

// The key layout of C covariates of nlev[c] levels: covariate c's first global level (base), its weight in the key
// (radix; covariate 0 most significant) and the number of keys.  Status 2 when the level product overflows 64 bits.
struct TupleKeys {
  std::vector<int> nlev, base;
  std::vector<uint64_t> radix;
  uint64_t key_space = 1;
  int B = 0;  // levels in all
};
int tuple_keys(hb_handle* h, const std::vector<int>& nlev, TupleKeys& k) {
  const int C = (int)nlev.size();
  k.nlev = nlev;
  k.radix.assign(C, 0);
  k.base.assign(C, 0);
  k.key_space = 1;
  long double prod = 1;
  for (int c = 0; c < C; ++c) prod *= (long double)nlev[c];
  if (prod > 9e18L) return fail(h, 2, "covariate level product overflows 64 bits");
  for (int c = C - 1; c >= 0; --c) {
    k.radix[c] = k.key_space;
    k.key_space *= (uint64_t)nlev[c];
  }
  for (int c = 1; c < C; ++c) k.base[c] = k.base[c - 1] + nlev[c - 1];
  k.B = std::accumulate(nlev.begin(), nlev.end(), 0);
  return 0;
}

// The index of the N cells whose levels phi_d (device, [N][C]) holds, read on the library stream.  global: the
// dictionary and the level counts are the union / sum over the ranks of h's communicator (setup of a sharded handle);
// else the cells are all there is.  Writes sort_perm / inv_sort (allocated here) and `out`; every other buffer is freed
// before it returns.  A level outside its covariate is refused with status 2, naming the cell; `names` (C names, or
// null for setup's message) name the covariates and report the caller's code (phi minus the covariate's base).
int build_tuple_index(hb_handle* h, const int* phi_d, int64_t N, const TupleKeys& keys, bool global,
                      DevBuf<int>& sort_perm, DevBuf<int>& inv_sort, TupleIndex& out, const char* const* names = nullptr) {
  const int C = (int)keys.nlev.size(), B = keys.B;
  const std::vector<int>& base = keys.base;
  const std::vector<uint64_t>& radix = keys.radix;
  const uint64_t key_space = keys.key_space;
  const int world = global ? h->world : 1;
  const bool direct = key_space <= (1ull << 22);  // the usual case: a table over the whole key space
  const cudaStream_t st = h->stream;
  const int grid = grid_for(N, 256, h->num_sms * 8);
  // ---- keys, validation, level counts and the dictionary in one pass
  DevBuf<unsigned long long> key, count, small, slots, uniq_d;
  DevBuf<int> geom, table, slot_id, flags;  // flags: {hash slots used, table full}
  SortScratch srt;
  CK(key.alloc(N));
  CK(count.alloc(B));
  CK(small.alloc(1 + (size_t)C));
  CK(geom.alloc(2 * (size_t)C));
  CK(flags.alloc(2));
  {
    std::vector<unsigned long long> sm(1 + C, TI_EMPTY);
    std::vector<int> g(2 * C);
    for (int c = 0; c < C; ++c) {
      sm[1 + c] = radix[c];
      g[c] = base[c];
      g[C + c] = keys.nlev[c];
    }
    CK(cudaMemcpyAsync(small.p, sm.data(), sizeof(unsigned long long) * sm.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(geom.p, g.data(), sizeof(int) * g.size(), cudaMemcpyHostToDevice, st));
  }
  CK(cudaMemsetAsync(count.p, 0, sizeof(unsigned long long) * B, st));
  CK(cudaMemsetAsync(flags.p, 0, 2 * sizeof(int), st));
  if (direct) {
    CK(table.alloc(key_space + 1));
    CK(cudaMemsetAsync(table.p, 0, sizeof(int) * (key_space + 1), st));
  } else {
    CK(slots.alloc(TI_SLOTS));
    CK(slot_id.alloc(TI_SLOTS));
    CK(cudaMemsetAsync(slots.p, 0xff, sizeof(unsigned long long) * TI_SLOTS, st));
  }
  TupleKeyArgs a{phi_d, N, C, B, geom.p, geom.p + C, small.p + 1, key.p, count.p, small.p,
                 direct ? table.p : nullptr, direct ? nullptr : slots.p, flags.p + 1};
  k_tuple_keys<<<grid, 256, 0, st>>>(a);
  CKL();
  unsigned long long bad = 0;
  CK(cudaMemcpyAsync(&bad, small.p, sizeof(bad), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad != TI_EMPTY) {
    int b = 0;
    CK(cudaMemcpyAsync(&b, phi_d + bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const int c = (int)(bad % C);
    if (names) return fail(h, 2, "%s of cell %lld is not a code in 0..%d", names[c], (long long)(bad / C), keys.nlev[c] - 1);
    return fail(h, 2, "phi row index %d of cell %lld is not a level of covariate %d", b, (long long)(bad / C), c);
  }
  // ---- the local dictionary: its keys on the device (uniq_d, J_local of them, ascending on the direct path)
  int J_local = 0, hash_full = 0;
  if (direct) {
    TRY(chained_scan(h, st, table.p, (int64_t)key_space + 1, 1, srt.scan));
    CK(cudaMemcpyAsync(&J_local, table.p + key_space, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(uniq_d.alloc(J_local));
    k_table_keys<<<grid_for((int64_t)key_space, 256, h->num_sms * 8), 256, 0, st>>>(table.p, (int64_t)key_space, uniq_d.p);
    CKL();
  } else {
    CK(uniq_d.alloc(TI_SLOTS));
    k_hash_compact<<<grid_for(TI_SLOTS, 256, h->num_sms * 8), 256, 0, st>>>(slots.p, uniq_d.p, flags.p);
    CKL();
    int f[2];
    CK(cudaMemcpyAsync(f, flags.p, sizeof(f), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    J_local = f[0];
    hash_full = f[1];
  }
  // a full hash table holds more than TI_SLOTS / 2 > 1e6 keys (or a probe sequence ran out): over the limit either way
  const bool over = hash_full || (size_t)J_local > TI_MAX_TUPLES;
  if (world == 1 && over) return too_many_tuples(h);
  out.lvl_count.assign(B, 0);
  if (world == 1) {
    out.uniq.resize(J_local);
    CK(cudaMemcpyAsync(out.uniq.data(), uniq_d.p, sizeof(uint64_t) * J_local, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(out.lvl_count.data(), count.p, sizeof(int64_t) * B, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (!direct) std::sort(out.uniq.begin(), out.uniq.end());
  } else {
    // global tuple dictionary = union over ranks; level counts summed over ranks.  Every rank learns the largest
    // local dictionary first, so that all of them stop together when one is over the limit.
    long long cnt = over ? (long long)TI_MAX_TUPLES + 1 : J_local, maxcnt = 0;
    DevBuf<long long> dcnt;
    CK(dcnt.alloc(1));
    CK(cudaMemcpyAsync(dcnt.p, &cnt, sizeof(cnt), cudaMemcpyHostToDevice, st));
    CKN(g_nccl.AllReduce(dcnt.p, dcnt.p, 1, ncclInt64, ncclMax, h->comm, st));
    CK(cudaMemcpyAsync(&maxcnt, dcnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if ((size_t)maxcnt > TI_MAX_TUPLES) return too_many_tuples(h);
    std::vector<uint64_t> recvbuf((size_t)maxcnt * h->world);
    DevBuf<uint64_t> ds, dr;
    CK(ds.alloc((size_t)maxcnt));
    CK(dr.alloc((size_t)maxcnt * h->world));
    CK(cudaMemsetAsync(ds.p, 0xff, sizeof(uint64_t) * (size_t)maxcnt, st));
    CK(cudaMemcpyAsync(ds.p, uniq_d.p, sizeof(uint64_t) * J_local, cudaMemcpyDeviceToDevice, st));
    CKN(g_nccl.AllGather(ds.p, dr.p, (size_t)maxcnt, ncclUint64, h->comm, st));
    CK(cudaMemcpyAsync(recvbuf.data(), dr.p, sizeof(uint64_t) * recvbuf.size(), cudaMemcpyDeviceToHost, st));
    CKN(g_nccl.AllReduce(count.p, count.p, B, ncclUint64, ncclSum, h->comm, st));
    CK(cudaMemcpyAsync(out.lvl_count.data(), count.p, sizeof(int64_t) * B, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    out.uniq.assign(recvbuf.begin(), recvbuf.end());
    std::sort(out.uniq.begin(), out.uniq.end());
    out.uniq.erase(std::unique(out.uniq.begin(), out.uniq.end()), out.uniq.end());
    if (!out.uniq.empty() && out.uniq.back() == ~0ull) out.uniq.pop_back();
  }
  if (out.uniq.size() > TI_MAX_TUPLES) return too_many_tuples(h);
  const int J = (int)out.uniq.size();
  // ---- tuple ids of the keys (the direct table of a single handle already holds them), then of the cells
  if (!direct || world > 1) {
    DevBuf<unsigned long long> ud;
    CK(ud.alloc(J));
    CK(cudaMemcpyAsync(ud.p, out.uniq.data(), sizeof(uint64_t) * J, cudaMemcpyHostToDevice, st));
    k_tuple_ids<<<grid_for(J, 256, h->num_sms * 4), 256, 0, st>>>(ud.p, J, direct ? table.p : nullptr, slots.p, slot_id.p);
    CKL();
    CK(cudaStreamSynchronize(st));
  }
  uniq_d.release();
  DevBuf<int> tid;
  CK(tid.alloc(N));
  k_tuple_of<<<grid, 256, 0, st>>>(key.p, N, direct ? table.p : nullptr, slots.p, slot_id.p, tid.p);
  CKL();
  key.release();
  table.release();
  slots.release();
  slot_id.release();
  srt.scan.release();
  // ---- stable sort by tuple id, and the tuple starts
  CK(sort_perm.reserve(N));
  CK(inv_sort.reserve(N));
  DevBuf<int> ts;
  CK(ts.alloc((size_t)J + 1));
  TRY(sort_by_code(h, srt, tid.p, N, J, nullptr, sort_perm.p, inv_sort.p, ts.p));
  std::vector<int> ts_h((size_t)J + 1);
  CK(cudaMemcpyAsync(ts_h.data(), ts.p, sizeof(int) * ts_h.size(), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  out.tstart.assign(ts_h.begin(), ts_h.end());
  return 0;
}

}  // namespace
