// update_single_pass.cuh — harmony::update_R (harmony.cpp:269-342) as one persistent kernel that reads every U row
// from HBM exactly ONCE per clustering round.  It runs whenever every CTA's slice of a block can lie inside one
// covariate tuple (2 J <= #SMs), K <= 256 and n KS < 2^32.
//
// The reference walks the blocks of a random partition sequentially (Gauss-Seidel on the K x B tables O, E):
//     O -= colsum(R_blk);  P = ((2E+1)/(O+E+1))^theta;  R_blk = L1norm(exp(U_blk) * P[level]);  O += colsum(R_blk)
// The removal term of a block, rem_{t,j} = sum of the CURRENT R over the cells of block j of round t, is the sum of
// rows that were last written in round t-1.  All T update orders of a cluster_cpp call are known before the first
// step runs, so the round that produces a row also files it under the block that will remove it: while round t
// updates a cell it adds the new row to add_{t,j} (its own block) and to remT[block of the cell in round t+1].
// Nothing is ever re-read: no look-ahead pass, no second (L2) touch, no saved penalty tables.  Round 0 takes its
// removal sums from k_rem_sums (one gather pass over the R of the assignment step / of the user), or from the
// assignment step itself when that runs in the plan's order.
//
// Accumulator slots and the table derivation are those of update_slots.cuh.  remT[parity][nb][J][KS] collects the
// next round's removal sums per (block, tuple); the first CTAs to arrive in a new round fold it into the rem halves
// of that round's slots (one extra grid-wide counter per round).
//
// How the rows reach the arithmetic: EVERY warp is a consumer that prefetches its own rows:
//   * a warp owns a contiguous run of its CTA's rows of every step and a private ring of DG row groups in shared
//     memory; lane l copies exactly the 16-byte pieces it will later read (cp.async.cg, one commit group per row
//     group), so completion is cp.async.wait_group — no mbarriers, no cross-lane visibility, no hand-shake words;
//   * the prefetch cursor runs DG groups ahead of the arithmetic in the warp's flat row stream and crosses block
//     steps: while the CTA waits for the step counter, the rows of the next step are already landing;
//   * plan entries (cell, next-round block) are fetched 32 rows at a time, one window ahead, and the CTA's range
//     records two steps ahead, so no load that feeds an address is waited for.
#pragma once
#include <type_traits>

#include "update_slots.cuh"

namespace hb {

constexpr int SP_MAXNV = 2;  // K <= 128 * SP_MAXNV (wider rows leave no room for the row rings)

struct SinglePassArgs {
  const float* U;        // [n][KS]
  float* R;              // [n][KS]
  const int* order;      // [T][n]  rows sorted by (block, tuple, block in the next round, cell)
  const int* next_at;    // [T][n]  block in round t+1 of the cell at each position of `order`
  const int4* ranges;    // [T*nb][grid] (lo, hi, tuple, 0): each CTA's slice of a block lies inside ONE tuple
  const int* tuple_levels;  // [J][C]
  const int* lvl_ptr;       // [B + 1]  CSR level -> tuples that contain it (ascending tuple order)
  const int* lvl_tup;       // [J C]
  const int* lvl_first1;    // [1] first level of covariate 1 (= B_vec[0])
  const float* sigma;    // [K]
  const float* theta;    // [B]
  const float* Pr_b;     // [B]
  float* ring;           // [2 parity][2 (O,E)][B][KS]
  float* acc;            // [(S+2)][SL]  slot(s) at (s+1)*SL: [add_O B*KS | add_rs KS | rem_O B*KS | rem_rs KS]
  float* remT;           // [2 parity][nb][J][KS]
  float* remS;           // [nb][J][KS]  sharded cells: sum of the ranks' remT of the round being folded
  float* OEend;          // [T][2][B][KS]  tables at the end of each round (for the objective)
  double* obj;           // [T][2]
  unsigned* bar;         // cntU[s + 1] for s = -1 .. S, then cntF[t] for t = 0 .. T
  int64_t n;
  int K, KS, C, J, B, nb, T;
  int s_begin, s_end;    // steps [s_begin, s_end) of this launch
  int write_from;        // rounds t >= write_from store R
  int has_next_from;     // rounds t < has_next_from file their rows under the next round's blocks
  int sigma_uniform;
  float sigma0;
  int ring_rows;         // rows of every warp's private ring (sp_ring_rows)
  int coop;              // 1: one launch covers many steps (counters + in-kernel fold); 0: single-step launch
};
struct SinglePassLaunch {
  SinglePassArgs a;
  PeerXch x;
};

__device__ __forceinline__ void sp_red_add_f4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__host__ __device__ inline int sp_nv(int KS) {
  int nv = 1;
  while (128 * nv < KS) nv <<= 1;
  return nv;
}

// Removal sums of a round from R in memory (round 0 of every cluster_cpp call: the R of the assignment step, or
// the R the user wrote): slot(t0 nb + j).rem += column sums of the rows of block j, per level.
//   grid = (G, nb): CTA (x, j) reduces range x of block j of the plan (the ranges of the update kernel).
__global__ void __launch_bounds__(256) k_rem_sums(const float* __restrict__ R, const int* __restrict__ order,
                                                  const int4* __restrict__ ranges, const int* __restrict__ tuple_levels,
                                                  float* __restrict__ acc, int s0, int G, int K, int KS, int C, int B) {
  extern __shared__ __align__(16) float sm_part[];  // [8][KS]
  const int j = blockIdx.y, x = blockIdx.x;
  const int4 rg = ranges[(size_t)j * G + x];
  const int lo = rg.x, hi = rg.y, q = rg.z;
  if (hi <= lo) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS4 = KS >> 2;
  const int BK = B * KS, SL = 2 * (BK + KS);
  for (int c4 = lane; c4 < KS4; c4 += 32) {
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = lo + warp; r < hi; r += 8) {
      const float4 v = ld_stream4(reinterpret_cast<const float4*>(R + (size_t)__ldg(order + r) * KS) + c4);
      s4.x += v.x;
      s4.y += v.y;
      s4.z += v.z;
      s4.w += v.w;
    }
    *reinterpret_cast<float4*>(sm_part + (size_t)warp * KS + 4 * c4) = s4;
  }
  __syncthreads();
  float* slot = acc + (size_t)(s0 + j + 1) * SL;
  float* rem_O = slot + BK + KS;
  float* rem_rs = rem_O + BK;
  for (int k = tid; k < K; k += 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sm_part[(size_t)w * KS + k];
    atomicAdd(rem_rs + k, t);
    for (int c = 0; c < C; ++c) atomicAdd(rem_O + (size_t)tuple_levels[q * C + c] * KS + k, t);
  }
}

// Fold of remT (the next round's removal sums per (block, tuple), filed during round t - 1) into the rem halves of
// round t's accumulator slots, one (block j, cluster k) column per call: rem_O[b][k] = sum over the tuples that
// contain level b, in ascending tuple order (the same order on every rank and in every launch mode); the row sum is
// the sum over the levels of covariate 0 (every tuple has exactly one).  Plain stores: the column has one owner.
// `table`: the [nb][J][KS] sums of round t — this rank's remT parity, or (sharded cells) the rank-ordered sum of all
// ranks' tables that gather_remT left in a.remS.
__device__ __forceinline__ void sp_fold_column(const SinglePassArgs& a, const float* table, int t, int j, int k) {
  const int KS = a.KS, J = a.J, nb = a.nb, B = a.B;
  const int BK = B * KS, SL = 2 * (BK + KS);
  const size_t joff = (size_t)j * J * KS + k;  // within `table` = the [nb][J][KS] sums of round t
  float* Tz = a.remT + (size_t)((t + 1) & 1) * nb * J * KS + (size_t)j * J * KS + k;
  float* slot = a.acc + (size_t)(t * nb + j + 1) * SL;
  float* rem_O = slot + BK + KS;
  float* rem_rs = rem_O + BK;
  auto val = [&](int q) -> float { return __ldcg(table + joff + (size_t)q * KS); };
  const int B0 = (a.C > 1) ? __ldg(a.lvl_first1) : B;  // levels of covariate 0 come first
  float rs = 0.f;
  for (int b0 = 0; b0 < B; b0 += 4) {  // four levels at a time: their loads are in flight together
    float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int b = b0 + i;
      if (b < B)
        for (int e = __ldg(a.lvl_ptr + b); e < __ldg(a.lvl_ptr + b + 1); ++e) o[i] += val(__ldg(a.lvl_tup + e));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int b = b0 + i;
      if (b < B) {
        rem_O[(size_t)b * KS + k] = o[i];
        if (b < B0) rs += o[i];
      }
    }
  }
  rem_rs[k] = rs;
  for (int q = 0; q < J; ++q) Tz[(size_t)q * KS] = 0.f;  // the other parity collects round t + 1's sums
}
// Stand-alone fold (per-step launches: sharded cells without the peer exchange, where remT is all-reduced by the
// host in between).  Same arithmetic as the in-kernel fold.
__global__ void k_fold_round(SinglePassArgs a, int t) {
  const float* table = a.remT + (size_t)(t & 1) * a.nb * a.J * a.KS;
  for (int item = blockIdx.x * blockDim.x + threadIdx.x; item < a.nb * a.K; item += gridDim.x * blockDim.x)
    sp_fold_column(a, table, t, item / a.K, item % a.K);
}

// After the last executed step S: O = O_S, E = E_S into the handle's tables.
__global__ void k_single_pass_finalize(SinglePassArgs a, PeerXch x, int S, float* __restrict__ O, float* __restrict__ E) {
  const int KS = a.KS, BK = a.B * KS, SL = 2 * (BK + KS);
  const bool multi = x.world > 1;
  // sharded cells: xch_sum waits for the other ranks' last add halves (their kernels may still be running)
  const float* ringO = a.ring + (size_t)((S - 1) & 1) * 2 * BK;
  const float* ringE = ringO + BK;
  const float* prev = a.acc + (size_t)(S)*SL;
  const float* cur = a.acc + (size_t)(S + 1) * SL;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < BK; idx += gridDim.x * blockDim.x) {
    const int b = idx / KS, k = idx - b * KS;
    float o = 0.f, e = 0.f;
    if (k < a.K) {
      // same arithmetic as derive() without the removal of step S (which never runs)
      const float prb = a.Pr_b[b];
      const float* prev_rem_O = prev + BK + KS;
      const float* prev_rem_rs = prev_rem_O + BK;
      const float add_o = multi ? (S >= 1 ? xch_sum(x, S + 1, idx) : 0.f) : cur[idx];
      const float add_rs = multi ? (S >= 1 ? xch_sum(x, S + 1, BK + k) : 0.f) : cur[BK + k];
      o = (ringO[idx] - prev_rem_O[idx]) + add_o;
      e = (ringE[idx] - prev_rem_rs[k] * prb) + add_rs * prb;
    }
    O[idx] = o;
    E[idx] = e;
  }
}



constexpr int SP_THREADS = 512;
constexpr int SP_NW = SP_THREADS / 32;

// shared-memory carve-up: tab[2 KP4] | sig[KP4] | part[NW][KP4] | ring[NW][D][KS] | meta[NW][2 D] (int2: cell, next block)
__host__ __device__ inline size_t sp_smem_bytes(int NV, int D, int KS) {
  return sizeof(float) * ((size_t)128 * NV * (3 + SP_NW) + (size_t)SP_NW * D * KS) + sizeof(int) * (size_t)SP_NW * 4 * D;
}
__host__ __device__ inline int sp_ru(int NV) { return NV == 1 ? 4 : 2; }  // rows per group (one warp iteration)
// rows per warp ring: the largest of 8 / 4 / 2 groups that fits (0: the kernel cannot run this row width)
inline int sp_ring_rows(int KS, size_t limit) {
  const int nv = sp_nv(KS);
  if (nv > SP_MAXNV) return 0;
  const int ru = sp_ru(nv);
  for (int dg : {8, 4, 2}) {
    const int D = dg * ru;
    if (sp_smem_bytes(nv, D, KS) <= limit) return D;
  }
  return 0;
}

template <int N>
__device__ __forceinline__ void sp_wait_group() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void sp_wait_pending(int dg) {  // at most dg - 1 groups still in flight
  if (dg == 8)
    sp_wait_group<7>();
  else if (dg == 4)
    sp_wait_group<3>();
  else
    sp_wait_group<1>();
}
// Row totals of RU rows at once: s[i] = this lane's partial of row i; on return every lane holds all RU totals.
// The butterfly halves the number of live values at every step (RU = 4: 10 shuffles instead of 20).
template <int RU>
__device__ __forceinline__ void sp_row_totals(float (&s)[RU], int lane) {
  static_assert(RU == 2 || RU == 4, "RU");
  float c;
  if (RU == 4) {
    const bool h16 = (lane & 16) != 0, h8 = (lane & 8) != 0;
    float a0 = h16 ? s[2] : s[0], a1 = h16 ? s[3] : s[1];
    const float b0 = h16 ? s[0] : s[2], b1 = h16 ? s[1] : s[3];
    a0 += __shfl_xor_sync(0xffffffffu, b0, 16);
    a1 += __shfl_xor_sync(0xffffffffu, b1, 16);
    c = h8 ? a1 : a0;
    const float d = h8 ? a0 : a1;
    c += __shfl_xor_sync(0xffffffffu, d, 8);  // lanes 8r .. 8r+7 hold row r
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = __shfl_sync(0xffffffffu, c, 8 * i);
  } else {
    const bool h16 = (lane & 16) != 0;
    c = h16 ? s[1] : s[0];
    const float d = h16 ? s[0] : s[1];
    c += __shfl_xor_sync(0xffffffffu, d, 16);  // lanes 16r .. 16r+15 hold row r
    c += __shfl_xor_sync(0xffffffffu, c, 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
#pragma unroll
    for (int i = 0; i < 2; ++i) s[i] = __shfl_sync(0xffffffffu, c, 16 * i);
  }
}

template <int NV, bool SIGU>
__global__ void __launch_bounds__(SP_THREADS, 1) k_update_single_pass(SinglePassLaunch lp) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const SinglePassArgs& a = lp.a;
  const PeerXch& x = lp.x;
  const bool multi = x.world > 1;
  constexpr int KP4 = 128 * NV;
  constexpr int RU = (NV == 1) ? 4 : 2;  // rows per group (in flight per warp iteration)
  const int K = a.K, KS = a.KS, C = a.C, J = a.J, B = a.B, nb = a.nb;
  const int KS4 = KS >> 2;
  const int BK = B * KS;
  const int SL = 2 * (BK + KS);
  const int D = a.ring_rows, DG = D / RU;  // DG: a power of two
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, grid = gridDim.x;

  float* tab = reinterpret_cast<float*>(smem_raw);  // log2 Psum of the CTA's tuple (second half unused)
  float* sig = tab + 2 * KP4;
  float* part = sig + KP4;                           // [NW][KP4]
  float* ringbuf = part + (size_t)SP_NW * KP4;       // [NW][D][KS]
  int2* meta = reinterpret_cast<int2*>(ringbuf + (size_t)SP_NW * D * KS);  // [NW][2 D] (cell, next block)
  int2* wmeta = meta + (size_t)warp * 2 * D;
  __shared__ double sh_obj[2];
  __shared__ int sh_last;

  // stale ring rows are read (with weight 0) by the tail of a row group: they must be finite
  for (float* q = ringbuf + tid; q < ringbuf + (size_t)SP_NW * D * KS; q += SP_THREADS) *q = 0.f;
  for (int i = tid; i < KP4; i += SP_THREADS) sig[i] = (i < K) ? a.sigma[i] : 0.f;
  for (int i = tid; i < 2 * KP4; i += SP_THREADS) tab[i] = -1.0e30f;  // padding columns: exp2 -> 0
  if (tid == 0) {
    sh_obj[0] = 0.0;
    sh_obj[1] = 0.0;
  }
  __syncthreads();

  bool lane_ok[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) lane_ok[v] = (lane + 32 * v) < KS4;
  // this lane's first 16-byte piece of ring row 0 of the warp (shared window address) and of a global row
  // lanes beyond the row (32 NV > KS / 4) read the row's last piece instead: their table entries make it weigh 0
  const int lane_c = (lane < KS4) ? lane : KS4 - 1;
  const unsigned ring_l = (unsigned)__cvta_generic_to_shared(ringbuf + (size_t)warp * D * KS + 4 * lane_c);
  const unsigned row_b = (unsigned)KS * 4u, grp_b = (unsigned)(RU * KS) * 4u, ring_b = (unsigned)(D * KS) * 4u;
  const float* U_l = a.U + 4 * lane_c;
  float* R_l = a.R + 4 * lane_c;
  const unsigned KSu = (unsigned)KS;  // n KS < 2^32 (checked by the host): 32-bit element offsets

  // ------------------------------------------------------------------------------------------------
  // the warp's flat row stream: for every step a run of whole groups of the CTA's range
  // ------------------------------------------------------------------------------------------------
  const int4 rg_none = make_int4(0, 0, 0, 0);
  auto ldrange = [&](int s) -> int4 { return (s < a.s_end) ? __ldg(a.ranges + (size_t)s * grid + cta) : rg_none; };
  // groups of RU rows are dealt out evenly: warp w takes groups [g0, g0 + cnt) of the ceil(n / RU) groups
  auto chunk_of = [&](const int4& rg, int& r0) -> int {  // returns the rows of the warp's run, r0 = its first row
    const int n = rg.y > rg.x ? rg.y - rg.x : 0;
    const int G = (n + RU - 1) / RU;
    const int gpw = G / SP_NW, rem = G - gpw * SP_NW;
    const int g0 = warp * gpw + (warp < rem ? warp : rem);
    const int cnt = gpw + (warp < rem ? 1 : 0);
    r0 = g0 * RU;
    const int r1 = (g0 + cnt) * RU;
    const int rows = (r1 < n ? r1 : n) - r0;
    return rows > 0 ? rows : 0;  // warps beyond the last group: r0 may exceed n
  };
  auto chunk_rows = [&](const int4& rg) {
    int r0;
    return chunk_of(rg, r0);
  };

  // prefetch cursor
  int ps = a.s_begin;             // step of the cursor
  int4 rg_cur = ldrange(ps), rg1 = ldrange(ps + 1), rg2 = ldrange(ps + 2);
  int p_rows = chunk_rows(rg_cur), p_off = 0;  // rows of the cursor's chunk / next row to issue
  int w_base = 0;                 // the current window holds rows [w_base, w_base + 32) of the chunk
  int wc = 0, wn = 0;             // this lane's entries of the current window
  int nw_step = a.s_end, nw_base = 0, nwc = 0, nwn = 0;  // the window after it
  int4 nw_rg = rg_none;
  int issued = 0;                 // groups issued so far
  unsigned issue_off = 0;         // byte offset of the next group's slot in the warp's ring
  auto load_window = [&](int s, const int4& rg, int base, int& c_out, int& n_out) {
    int r0;
    const int rows = chunk_of(rg, r0);
    c_out = 0;
    n_out = 0;
    if (base + lane < rows) {
      const size_t p = (size_t)(s / nb) * (size_t)a.n + (size_t)rg.x + (size_t)(r0 + base + lane);
      c_out = __ldg(a.order + p);
      n_out = __ldg(a.next_at + p);
    }
  };
  // identity + entries of the window that follows (ps, w_base)
  auto fetch_next_window = [&]() {
    if (w_base + 32 < p_rows) {
      nw_step = ps;
      nw_base = w_base + 32;
      nw_rg = rg_cur;
    } else {
      int S = ps + 1;
      int4 r = rg1;
      while (S < a.s_end && chunk_rows(r) == 0) {
        ++S;
        r = (S == ps + 2) ? rg2 : ldrange(S);
      }
      nw_step = S;
      nw_base = 0;
      nw_rg = r;
    }
    if (nw_step < a.s_end) load_window(nw_step, nw_rg, nw_base, nwc, nwn);
  };
  auto adopt_next_window = [&]() {
    if (nw_step != ps) {
      if (nw_step == ps + 1) {
        rg1 = rg2;
      } else {
        rg1 = ldrange(nw_step + 1);
      }
      rg2 = ldrange(nw_step + 2);
      ps = nw_step;
      rg_cur = nw_rg;
      p_rows = (ps < a.s_end) ? chunk_rows(rg_cur) : 0;
    }
    w_base = nw_base;
    p_off = nw_base;
    wc = nwc;
    wn = nwn;
    if (ps < a.s_end) fetch_next_window();
  };
  // first window: the first non-empty chunk at or after s_begin
  {
    while (ps < a.s_end && p_rows == 0) {
      ++ps;
      rg_cur = rg1;
      rg1 = rg2;
      rg2 = ldrange(ps + 2);
      p_rows = (ps < a.s_end) ? chunk_rows(rg_cur) : 0;
    }
    if (ps < a.s_end) {
      load_window(ps, rg_cur, 0, wc, wn);
      fetch_next_window();
    }
  }
  // one group (RU rows) of the stream -> the next ring slot; always commits (an empty group keeps the count)
  auto issue_group = [&]() {
    if (ps < a.s_end) {
      const int j0 = p_off - w_base;  // window row of the group's first row (a multiple of RU, <= 32 - RU)
      const int left = p_rows - p_off;  // > 0
      unsigned dst = ring_l + issue_off;
#pragma unroll
      for (int i = 0; i < RU; ++i) {
        const int cell = __shfl_sync(0xffffffffu, wc, j0 + i);
        if (i < left) {
          const float* src = U_l + (size_t)((unsigned)cell * KSu);
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (lane_ok[v])
              asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 512u * v), "l"(src + 128 * v) : "memory");
        }
        dst += row_b;
      }
      // the lanes that hold the group's plan entries file them for the arithmetic (cell < 0: no such row)
      const int li = lane - j0;
      if ((unsigned)li < (unsigned)RU) wmeta[(issued & (2 * DG - 1)) * RU + li] = make_int2(li < left ? wc : -1, wn);
      p_off += RU;
      if (p_off >= p_rows || p_off - w_base >= 32) adopt_next_window();
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    ++issued;
    issue_off += grp_b;
    if (issue_off == ring_b) issue_off = 0;
  };
  for (int g = 0; g < DG; ++g) issue_group();

  // ------------------------------------------------------------------------------------------------
  // step protocol (update_slots.cuh)
  // ------------------------------------------------------------------------------------------------
  const int S_total = a.T * nb;
  unsigned* cntU = a.bar + 1;              // cntU[s], s >= -1
  unsigned* cntF = a.bar + (S_total + 2);  // cntF[t]
  auto signal = [&](unsigned* c, int sl) {
    __syncthreads();
    if (!multi || sl < 0) {
      if (tid == 0) {
        __threadfence();
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(c) : "memory");
      }
      return;
    }
    if (tid == 0) {
      __threadfence();
      const unsigned old = atomicAdd(c, 1u);
      __threadfence();
      sh_last = (old == (unsigned)grid - 1u) ? 1 : 0;
    }
    __syncthreads();
    if (sh_last) {
      const float* src = a.acc + (size_t)sl * SL;  // complete: every CTA's atomics preceded its count
      const size_t entry = (size_t)sl * x.world + x.rank;
      for (int i = 2 * tid; i < x.XH; i += 2 * SP_THREADS) {  // XH is a multiple of 4: entries are 16-byte aligned
        const float2 v = __ldcg(reinterpret_cast<const float2*>(src + i));
        for (int r = 0; r < x.world; ++r) xch_st2(x.peer_inbox[r] + entry * x.XH + i, v.x, v.y, x.epoch);
      }
    }
  };
  auto wait_for = [&](const unsigned* c) {
    if (tid == 0) {
      while (ld_acquire_u32(c) < (unsigned)grid) __nanosleep(20);
      __threadfence();
    }
    __syncthreads();
  };
  auto tables_for = [&](int s) {
    SlotTables tv;
    const int par = (s - 1) & 1;
    tv.ringO = a.ring + (size_t)par * 2 * BK;
    tv.ringE = tv.ringO + BK;
    tv.prev = a.acc + (size_t)(s)*SL;       // slot(s-1)
    tv.cur = a.acc + (size_t)(s + 1) * SL;  // slot(s)
    tv.BK = BK;
    tv.KS = KS;
    return tv;
  };
  unsigned* cntG = cntF + (a.T + 1);        // cntG[t]: the ranks' removal sums of round t are gathered
  // sharded cells: the add half of slot index sl has started to arrive from every rank, i.e. every rank has finished
  // the step that produced it (its last CTA pushes after all of the rank's CTAs counted)
  auto wait_ranks = [&](int sl) {
    if (tid < x.world) {
      const uint2* w = x.inbox + ((size_t)sl * x.world + tid) * x.XH;
      while (xch_ld(w).y != x.epoch) __nanosleep(40);
    }
    __syncthreads();
  };
  // sharded cells: remS = sum over the ranks' remT tables of round t in rank order, 16 bytes per load (the peers'
  // tables are read over NVLink: 4-byte loads per (tuple, cluster) swamp the fabric at 8 ranks)
  auto gather_remT = [&](int t) {
    const size_t par_off = (size_t)(t & 1) * nb * J * KS;
    const int n4 = (nb * J * KS) >> 2;
    for (int i = cta * SP_THREADS + tid; i < n4; i += grid * SP_THREADS) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int r = 0; r < x.world; ++r) {
        const float4 p = __ldcg(reinterpret_cast<const float4*>(x.peer_remT[r] + par_off) + i);
        v.x += p.x;
        v.y += p.y;
        v.z += p.z;
        v.w += p.w;
      }
      reinterpret_cast<float4*>(a.remS)[i] = v;
    }
  };
  auto fold_round = [&](int t) {
    const float* table = multi ? a.remS : a.remT + (size_t)(t & 1) * nb * J * KS;
    for (int item = cta * SP_THREADS + tid; item < nb * K; item += grid * SP_THREADS)
      sp_fold_column(a, table, t, item / K, item % K);
  };

  // objective partial sums of this lane.  Scalar sigma: accA = sum_rows (1/s) sum_k e u, accB = sum_rows (1/s) sum_k e log Psum
  // (this lane's columns), accL = sum_rows log2 s (the same value in every lane); per-cluster sigma: okd / oent directly.
  float okd = 0.f, oent = 0.f, accA = 0.f, accB = 0.f, accL = 0.f;
  auto flush_objective = [&](int t) {
    if (SIGU) {
      // sum_k R dist = -sigma sum R u ;  sum_k sigma R log R = sigma (sum R (u + log Psum) - log s)
      const float sA = warp_sum(accA), sB = warp_sum(accB);
      okd = -a.sigma0 * sA;
      oent = a.sigma0 * (sA + (sB - accL) * 0.6931471805599453f);  // accB, accL in log2 units
    } else {
      okd = warp_sum(okd);
      oent = warp_sum(oent);
    }
    if (lane == 0) {
      atomicAdd(&sh_obj[0], (double)okd);
      atomicAdd(&sh_obj[1], (double)oent);
    }
    __syncthreads();
    if (tid == 0) {
      atomicAdd(a.obj + 2 * t + 0, sh_obj[0]);
      atomicAdd(a.obj + 2 * t + 1, sh_obj[1]);
      sh_obj[0] = 0.0;
      sh_obj[1] = 0.0;
    }
    __syncthreads();
    okd = oent = accA = accB = accL = 0.f;
  };

  int consumed = 0;       // groups consumed so far (same sequence as `issued`)
  unsigned cons_off = 0;  // byte offset of the next group's slot in the warp's ring
  for (int s = a.s_begin; s < a.s_end; ++s) {
    const int4 rg = ldrange(s);
    const int n = rg.y > rg.x ? rg.y - rg.x : 0;
    const int q = rg.z;
    const int my_rows = chunk_rows(rg);
    const int t = s / nb, j = s - t * nb;
    const bool writeR = t >= a.write_from;
    const bool has_next = t < a.has_next_from;
    if (a.coop) {
      if (s > a.s_begin) wait_for(cntU + s - 1);  // add_{s-1}, ring(s-1); at j == 0 also: round t-1 is complete
      if (j == 0 && t > 0) {
        if (multi) {
          wait_ranks(s + 1);  // add_{s-1} lives in slot index s + 1: every rank has finished round t - 1, its remT is final
          gather_remT(t);
          signal(cntG + t, -1);
          wait_for(cntG + t);
        }
        fold_round(t);
        signal(cntF + t, -1);
        wait_for(cntF + t);
      }
    }
    const PeerXch* xp = multi ? &x : nullptr;
    const int xs = (s >= 1) ? s + 1 : -1;
    // ---- tables of the step: the penalty row of this CTA's tuple, and this CTA's share of O_s, E_s ----
    {
      const SlotTables tv = tables_for(s);
      if (n > 0) {
        for (int k = tid; k < K; k += SP_THREADS) {
          float v = 0.f;
          for (int c = 0; c < C; ++c) {
            float o, e, pp;
            derive(tv, a.Pr_b, a.theta, __ldg(a.tuple_levels + q * C + c), k, o, e, pp, xp, xs);
            v += pp;
          }
          float l2;
          asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l2) : "f"(v));
          tab[k] = fmaxf(l2, -1.0e30f);  // log2 Psum (Psum = 0: exp2 -> 0 and 0 * -1e30 = 0 in the objective sums)
        }
      }
      float* outO = a.ring + (size_t)(s & 1) * 2 * BK;
      float* outE = outO + BK;
      for (int idx = cta + grid * (SP_THREADS - 1 - tid); idx < BK; idx += grid * SP_THREADS) {  // the last threads first: they idle above
        const int b = idx / KS, k = idx - b * KS;
        float o = 0.f, e = 0.f, pp = 0.f;
        if (k < K) derive(tv, a.Pr_b, a.theta, b, k, o, e, pp, xp, xs);
        outO[idx] = o;
        outE[idx] = e;
        if (j == 0 && t > 0) {
          float* oe = a.OEend + (size_t)(t - 1) * 2 * BK;
          oe[idx] = o;
          oe[BK + idx] = e;
        }
      }
    }
    __syncthreads();
    if (n > 0) {
      float4 pL[NV], sg[NV];  // log2 Psum of this lane's columns, sigma
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        pL[v] = *reinterpret_cast<const float4*>(tab + 4 * (lane + 32 * v));
        sg[v] = *reinterpret_cast<const float4*>(sig + 4 * (lane + 32 * v));
      }
      float4 cs[NV], cs2[NV];  // column sums of the step / of the rows filed under next-round block cur_nb
      bool st_ok[NV];
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        cs[v] = cs2[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        st_ok[v] = writeR && lane_ok[v];
      }
      int cur_nb = -1;
      float* remT_l = a.remT + (size_t)((t + 1) & 1) * nb * J * KS + (size_t)q * KS + 4 * lane;
      const unsigned nb_stride = (unsigned)(J * KS);
      auto flush_next = [&]() {
        if (cur_nb >= 0) {
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            if (has_next && lane_ok[v]) sp_red_add_f4(remT_l + (size_t)((unsigned)cur_nb * nb_stride) + 128 * v, cs2[v]);
            cs[v].x += cs2[v].x;
            cs[v].y += cs2[v].y;
            cs[v].z += cs2[v].z;
            cs[v].w += cs2[v].w;
            cs2[v] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      };
      constexpr float L2E = 1.4426950408889634f;
      const int ngroups = (my_rows + RU - 1) / RU;
      for (int gi = 0; gi < ngroups; ++gi) {
        sp_wait_pending(DG);
        __syncwarp();  // the plan entries of this group were filed DG iterations ago by other lanes
        const int2* mt = wmeta + (consumed & (2 * DG - 1)) * RU;
        const unsigned rd = ring_l + cons_off;
        float4 e[RU][NV];
        float ssum[RU], Aacc[RU], Bacc[RU], Sacc[RU];
        int cellr[RU], nbr[RU];
#pragma unroll
        for (int i = 0; i < RU; ++i) {
          const int2 m2 = mt[i];
          cellr[i] = m2.x;
          nbr[i] = m2.y;
        }
#pragma unroll
        for (int i = 0; i < RU; ++i) {
          ssum[i] = Aacc[i] = Bacc[i] = Sacc[i] = 0.f;
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            float4 u4;
            asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];"
                         : "=f"(u4.x), "=f"(u4.y), "=f"(u4.z), "=f"(u4.w)
                         : "r"(rd + (unsigned)i * row_b + 512u * v));
            const float uu[4] = {u4.x, u4.y, u4.z, u4.w};
            const float ll[4] = {pL[v].x, pL[v].y, pL[v].z, pL[v].w};
            const float ss[4] = {sg[v].x, sg[v].y, sg[v].z, sg[v].w};
            float ee[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              ee[c] = fast_exp2(fmaf(uu[c], L2E, ll[c]));  // exp(u) Psum: un-normalised R (exactly 0 in the padding columns)
              if (SIGU) {
                Aacc[i] = fmaf(ee[c], uu[c], Aacc[i]);
                Bacc[i] = fmaf(ee[c], ll[c], Bacc[i]);
              } else {
                const float tt = ss[c] * ee[c];
                Aacc[i] = fmaf(tt, uu[c], Aacc[i]);
                Bacc[i] = fmaf(tt, ll[c], Bacc[i]);
                Sacc[i] += tt;
              }
            }
            ssum[i] += (ee[0] + ee[1]) + (ee[2] + ee[3]);
            e[i][v] = make_float4(ee[0], ee[1], ee[2], ee[3]);
          }
        }
        sp_row_totals<RU>(ssum, lane);
        // the rows of a CTA are sorted by next-round block: the group lies in one block iff its ends do
        if (nbr[0] != cur_nb) {  // warp-uniform
          flush_next();
          cur_nb = nbr[0];
        }
        auto finish_row = [&](int i, auto fast_tag) {
          constexpr bool FAST = decltype(fast_tag)::value;  // the row exists and belongs to block cur_nb
          const bool valid = FAST || cellr[i] >= 0;
          const float sdiv = (ssum[i] == 0.f) ? 1.f : ssum[i];  // arma::normalise(.., 1, 0): zero norm divides by 1
          float inv = fast_rcp(sdiv);
          if (!FAST) {
            if (!valid) inv = 0.f;
            if (valid && nbr[i] != cur_nb) {  // warp-uniform
              flush_next();
              cur_nb = nbr[i];
            }
          }
          float* rp = R_l + (size_t)((unsigned)cellr[i] * KSu);
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            float4 rr;
            rr.x = e[i][v].x * inv;
            rr.y = e[i][v].y * inv;
            rr.z = e[i][v].z * inv;
            rr.w = e[i][v].w * inv;
            cs2[v].x += rr.x;
            cs2[v].y += rr.y;
            cs2[v].z += rr.z;
            cs2[v].w += rr.w;
            if (st_ok[v] && valid) *reinterpret_cast<float4*>(rp + 128 * v) = rr;
          }
          float l2s;
          asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l2s) : "f"(sdiv));
          if (SIGU) {
            accA = fmaf(inv, Aacc[i], accA);
            accB = fmaf(inv, Bacc[i], accB);
            accL += valid ? l2s : 0.f;
          } else {
            // sum_k R dist = -sum sigma R U ;  sum_k sigma R log R = sum sigma R (U + log Psum - log s)
            okd = fmaf(-inv, Aacc[i], okd);
            oent = fmaf(inv, fmaf(0.6931471805599453f, Bacc[i] - l2s * Sacc[i], Aacc[i]), oent);
          }
        };
        if (cellr[RU - 1] >= 0 && nbr[RU - 1] == cur_nb) {
#pragma unroll
          for (int i = 0; i < RU; ++i) finish_row(i, std::true_type());
        } else {
#pragma unroll
          for (int i = 0; i < RU; ++i) finish_row(i, std::false_type());
        }
        ++consumed;
        cons_off += grp_b;
        if (cons_off == ring_b) cons_off = 0;
        issue_group();  // refill the slot just read (its values are in registers: the arithmetic above depends on them)
      }
      flush_next();
      // ---- add_s: this CTA's column sums -> slot(s+1) ----
#pragma unroll
      for (int v = 0; v < NV; ++v) *reinterpret_cast<float4*>(part + (size_t)warp * KP4 + 4 * (lane + 32 * v)) = cs[v];
      __syncthreads();
      float* nslot = a.acc + (size_t)(s + 2) * SL;
      for (int k = tid; k < K; k += SP_THREADS) {
        float tsum = 0.f;
#pragma unroll
        for (int w = 0; w < SP_NW; ++w) tsum += part[(size_t)w * KP4 + k];
        atomicAdd(nslot + BK + k, tsum);
        for (int c = 0; c < C; ++c) atomicAdd(nslot + (size_t)__ldg(a.tuple_levels + q * C + c) * KS + k, tsum);
      }
    }
    if ((s + 1) % nb == 0) flush_objective(t);
    if (a.coop) signal(cntU + s, s + 2);  // add_s lives in slot(s + 1) = index s + 2
  }
  if (a.s_end % nb != 0 && a.s_end > a.s_begin) flush_objective((a.s_end - 1) / nb);  // partial round
  asm volatile("cp.async.wait_all;" ::: "memory");
}

}  // namespace hb
