// apply_tc3.cuh — K5 on the tensor cores: the correction of harmony.cpp:347 + :615 for all clusters at once,
//   Zc_i = Zo_i - sum_k R_ik V_q[k][:]        (q = covariate tuple of cell i, V_q from k_ridge_solve)
// as D[cell][c] = sum_k A[cell][k] * B[c][k] per 64-cell tile, A = the tile of R (M = 64 cells, from registers),
// B = V_q^T (N = 64 or 128 embedding columns, shared memory, static while the tuple does not change), 3xTF32, fp32
// accumulators in registers.
//   * each tile's rows of R and of the minuend (Zo, or the partial Zc of an earlier cluster range) go into a ring of
//     NST raw stages with bulk asynchronous copies, issued by one warp, whose bytes complete on the stage's "full"
//     mbarrier.  A tile never crosses a tuple and cells are sorted by tuple, so the tile is one contiguous span of
//     each array (one copy each; a cluster range narrower than the row of R copies row by row).  The copies of the
//     next NST - 1 tiles stay in flight while a tile is multiplied: at K = 100, d = 50 a stage holds
//     64 x (100 + 52) x 4 B = 38.9 KB and four fit, up to 117-156 KB per SM in flight.
//   * two MMA warpgroups take alternate tiles.  Each thread loads its A fragments (rows 16 w + l / 4 (+ 8) of the
//     raw R rows, all AP_MAXK / 8 K steps at once, zero beyond Kp) from the stage, splits them into tf32 hi / lo in
//     registers, issues 3 x AP_MAXK / 8 wgmma (a K-step count known only at run time makes ptxas serialise the
//     wgmma), and subtracts the accumulator from the minuend rows IN the stage; the warpgroup then writes the
//     whole rows (padding columns d..DS-1 included, which hold the minuend's zeros) back with one bulk store, and
//     once the store has read the stage its first warp refills it with tile it + NST.  NST is even (2 or 4), so
//     every stage belongs to one warpgroup and the refill needs no "empty" barrier.
//   * B = V_q^T is rebuilt by both warpgroups together (named barrier) when the tuple changes; both walk every tile
//     of the CTA's range in order, so they meet at the same rebuild points.
// Warp roles (256 threads): 0-3 MMA warpgroup of the even tiles, 4-7 of the odd tiles.  No separate copy warp: a
// ninth warp would put three warps on one SM sub-partition and cap the registers at 168, too few for the A
// fragments of 14 K steps next to 64 accumulators (NH = 2 needs 203).
// Shared memory: B hi/lo 2 x NB x AP_MAXK floats ([AP_MAXK/4][NB][4], K-major, NB = 64 NH), then NST raw stages of
// 64 x (RS + DS) floats (RS = floats of R per row in this launch), then the barriers.
// Limits per launch: d <= 128 and <= AP_MAXK clusters with at least two raw stages; more clusters run as several
// launches over cluster ranges, each subtracting its share from the partial result (the first from Zo).
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int AP_TN = 64;         // cells per tile (= wgmma M), equals the static tile size TM
constexpr int AP_THREADS = 256;   // two MMA warpgroups
constexpr int AP_MAXK = 112;      // clusters per launch: 14 K steps of A fragments in registers
constexpr int AP_NKS = AP_MAXK / 8;
constexpr int AP_MAXST = 4;       // raw stages

struct ApplyTcArgs {
  const float* R;   // [n][KS]
  const float* V;   // [J][K][d]
  float* Zc;        // [n][DS]
  const int* tile_cell0;
  const int* tile_len;
  const int* tile_tuple;
  int ntiles, d, K, KS, DS;
  int k_off, Kp, KD;  // this launch: clusters [k_off, k_off + Kp) (k_off a multiple of 8), KD = Kp rounded up to 8
  const float* minuend;  // Zo for the first cluster range, Zc (the partial result) for the following ones
  int tiles_per_cta;
  int c_off, DC;  // k_apply_tc_cols: embedding columns [c_off, c_off + DC) (multiples of 4; the last range ends at DS)
};

// k_apply_tc takes all of d in one launch up to d = 128 (NH = 2)
inline bool apply_tc_fits(int d) { return d <= 128; }
__host__ __device__ inline int apply_tc_nb(int d) { return d <= 64 ? 64 : 128; }
// floats of R per row of a raw stage: the launch's cluster range (the rest of the row when it is the last range)
__host__ __device__ inline int apply_tc_rs(int KD, int KS, int k_off) { return KS - k_off < KD ? KS - k_off : KD; }
__host__ __device__ inline size_t apply_tc_stage_bytes(int RS, int DS) { return sizeof(float) * (size_t)AP_TN * (RS + DS); }
__host__ __device__ inline size_t apply_tc_fixed_bytes(int d) {
  return sizeof(float) * 2 * (size_t)apply_tc_nb(d) * AP_MAXK + AP_MAXST * sizeof(uint64_t);
}
__host__ __device__ inline int apply_tc_stages(int RS, int d, int DS) {
  const size_t fixed = apply_tc_fixed_bytes(d), st = apply_tc_stage_bytes(RS, DS);
  const int n = fixed < SMEM_LIMIT ? (int)((SMEM_LIMIT - fixed) / st) : 0;
  // even, so that stage it % NST always serves warpgroup it % 2: that warpgroup refills the stage only after using
  // it, and a waiter can never find the stage's barrier a phase behind (with an odd count the other warpgroup's next
  // tile in the stage could pass the wait on the previous phase's parity before this tile's bytes have landed).
  // The host splits the clusters until this is >= 2.
  return (n < AP_MAXST ? n : AP_MAXST) & ~1;
}
__host__ __device__ inline size_t apply_tc_smem_bytes(int RS, int d, int DS) {
  return apply_tc_fixed_bytes(d) + apply_tc_stages(RS, d, DS) * apply_tc_stage_bytes(RS, DS);
}

// Column ranges (d > 256, or K x d beyond the FFMA apply): one launch per <= 128 embedding columns [c_off, c_off + DC)
// and cluster range, B = 128 columns of V_q^T.  A stage's minuend rows are the range's DC floats of each row (row-by-row
// bulk copies in and out, as the R rows of a narrow cluster range); the first cluster range of each column range
// subtracts from Zo.  Bytes per cell over the whole grid: 4 KS per column range (R) + 8 DS per cluster range (minuend
// in, Zc out).
__host__ __device__ inline size_t apply_cols_fixed_bytes() { return sizeof(float) * 2 * (size_t)128 * AP_MAXK + AP_MAXST * sizeof(uint64_t); }
__host__ __device__ inline int apply_cols_stages(int RS, int DC) {
  const size_t fixed = apply_cols_fixed_bytes(), st = apply_tc_stage_bytes(RS, DC);
  const int n = fixed < SMEM_LIMIT ? (int)((SMEM_LIMIT - fixed) / st) : 0;
  return (n < AP_MAXST ? n : AP_MAXST) & ~1;  // even: see apply_tc_stages
}
__host__ __device__ inline size_t apply_cols_smem_bytes(int RS, int DC) {
  return apply_cols_fixed_bytes() + apply_cols_stages(RS, DC) * apply_tc_stage_bytes(RS, DC);
}

// NH: 64-column halves of B = embedding columns (1: d <= 64, 2: d <= 128), fixed at compile time so that the
// accumulators stay in registers.  CR: one column range of the embedding per launch (NH = 2).
template <int NH, bool CR>
__device__ __forceinline__ void apply_tc_body(const ApplyTcArgs& a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int NB = 64 * NH;
  const int KD = a.KD, K = a.K, KS = a.KS, Kp = a.Kp;
  const int d = CR ? (a.d - a.c_off < a.DC ? a.d - a.c_off : a.DC) : a.d;  // columns of this launch
  const int DS = CR ? a.DC : a.DS;                                          // floats of a minuend row in a stage
  const int RS = apply_tc_rs(KD, KS, a.k_off);
  const int NST = CR ? apply_cols_stages(RS, DS) : apply_tc_stages(RS, d, DS);
  const int SST = AP_TN * (RS + DS);                 // floats per raw stage: R rows [64][RS], then minuend rows [64][DS]
  float* Bhi = reinterpret_cast<float*>(smem_raw);   // [AP_MAXK/4][NB][4]  V_q^T
  float* Blo = Bhi + (size_t)NB * AP_MAXK;
  float* raw = Blo + (size_t)NB * AP_MAXK;
  uint64_t* full = reinterpret_cast<uint64_t*>(raw + (size_t)NST * SST);  // [NST]  the stage's bytes have landed
  // the warp index through a shuffle: ptxas sees the role branches as warp-uniform and does not serialise the wgmma
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;

  const int t_begin = blockIdx.x * a.tiles_per_cta;
  const int t_end = (t_begin + a.tiles_per_cta < a.ntiles) ? t_begin + a.tiles_per_cta : a.ntiles;
  // tile `it` of the range -> stage it % NST; called by one whole warp
  auto load = [&](int it) {
    const int tile = t_begin + it, s = it % NST;
    const int cell0 = __ldg(a.tile_cell0 + tile), len = __ldg(a.tile_len + tile);
    float* rR = raw + (size_t)s * SST;
    float* rZ = rR + AP_TN * RS;
    if (lane == 0) {
      umma::mbar_arrive_expect_tx(full + s, (uint32_t)(sizeof(float) * len * (RS + DS)));
      if constexpr (!CR) umma::bulk_g2s(rZ, a.minuend + (size_t)cell0 * DS, (uint32_t)(sizeof(float) * len * DS), full + s);
      if (RS == KS) umma::bulk_g2s(rR, a.R + (size_t)cell0 * KS, (uint32_t)(sizeof(float) * len * KS), full + s);
    }
    if (RS != KS) {  // a cluster range narrower than the row: row by row
      __syncwarp();  // the expected bytes are registered before any row completes
      for (int j = lane; j < len; j += 32)
        umma::bulk_g2s(rR + (size_t)j * RS, a.R + (size_t)(cell0 + j) * KS + a.k_off, (uint32_t)(sizeof(float) * RS), full + s);
    }
    if constexpr (CR) {  // the column range of each minuend row
      __syncwarp();
      for (int j = lane; j < len; j += 32)
        umma::bulk_g2s(rZ + (size_t)j * DS, a.minuend + (size_t)(cell0 + j) * a.DS + a.c_off, (uint32_t)(sizeof(float) * DS), full + s);
    }
  };

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) umma::mbar_init(full + i, 1);
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (warp == 0)
    for (int it = 0; it < NST && t_begin + it < t_end; ++it) load(it);

  // =============================== MMA warpgroups + epilogue ===============================
  const int e = warp >> 2;   // tiles t_begin + e, + e + 2, ..
  const int w = warp & 3;    // warp of the warpgroup
  const int wt = tid & 127;  // thread of the warpgroup
  const uint32_t lboB = NB * 16, sbo = 128;
  const uint32_t bH = umma::smem_u32(Bhi), bL = umma::smem_u32(Blo);
  int cur_q = -1;
  for (int tile = t_begin, it = 0; tile < t_end; ++tile, ++it) {
    const int q = __ldg(a.tile_tuple + tile);
    if (q != cur_q) {
      // new tuple: B = V_q^T (k contiguous per embedding column c), tf32 hi/lo — after both warpgroups' MMAs
      umma::named_sync(1, 256);
      const float* Vq = a.V + ((size_t)q * K + a.k_off) * a.d + (CR ? a.c_off : 0);
      for (int idx = tid; idx < NB * AP_MAXK; idx += 256) {
        const int k = idx / NB, c = idx - k * NB;
        const float v = (k < Kp && c < d) ? Vq[(size_t)k * a.d + c] : 0.f;
        float hi, lo;
        umma::split_tf32(v, hi, lo);
        const int off = ((k >> 2) * NB + c) * 4 + (k & 3);
        Bhi[off] = hi;
        Blo[off] = lo;
      }
      umma::fence_proxy_async();
      umma::named_sync(1, 256);
      cur_q = q;
    }
    if ((it & 1) != e) continue;
    const int s = it % NST;
    const int cell0 = __ldg(a.tile_cell0 + tile), len = __ldg(a.tile_len + tile);
    float* rR = raw + (size_t)s * SST;
    float* rZ = rR + AP_TN * RS;
    umma::mbar_wait(full + s, (it / NST) & 1);

    // A fragments of all K steps: hi = the raw value (the tensor core reads its upper 19 bits), lo = the remainder
    // z - trunc_tf32(z), exact in fp32 and truncated by the tensor core in turn (relative error of the pair
    // <= 2^-20).  Clusters >= Kp are zero.  Rows beyond the tile hold stale values; their rows of D are not read.
    uint32_t ah[AP_NKS][4], al[AP_NKS][4];
    {
      const int r0 = 16 * w + (lane >> 2), k0 = lane & 3;
#pragma unroll
      for (int ks = 0; ks < AP_NKS; ++ks) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = r0 + 8 * (j & 1), k = 8 * ks + k0 + 4 * (j >> 1);
          const float z = k < Kp ? rR[r * RS + k] : 0.f;
          ah[ks][j] = __float_as_uint(z);
          al[ks][j] = __float_as_uint(umma::tf32_rem(z));
        }
      }
    }
    float acc[NB / 2];  // overwritten by the first MMA (accumulate = 0)
    umma::fence();
#pragma unroll
    for (int ks = 0; ks < AP_NKS; ++ks) {
      {
        const uint32_t bo = ks * 2 * lboB;
        const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
        const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
        if constexpr (NH == 1) {
          umma::mma_rs_n64(acc, ah[ks], bl, ks > 0);
          umma::mma_rs_n64(acc, al[ks], bh, 1);
          umma::mma_rs_n64(acc, ah[ks], bh, 1);
        } else {
          umma::mma_rs_n128(acc, ah[ks], bl, ks > 0);
          umma::mma_rs_n128(acc, al[ks], bh, 1);
          umma::mma_rs_n128(acc, ah[ks], bh, 1);
        }
      }
    }
    umma::commit();
    umma::wait0();
    // Zc[cell][c] = minuend[cell][c] - D[cell][c], in the stage
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) {
      const int j = umma::frag_row(i, w, lane), c = umma::frag_col(i, lane);
      if (c < d && j < len) rZ[j * DS + c] = rZ[j * DS + c] - acc[i];
    }
    umma::fence_proxy_async();  // the rows written above -> the bulk store
    umma::named_sync(2 + e, 128);
    if (w == 0) {
      if constexpr (CR) {
        for (int j = lane; j < len; j += 32)
          umma::bulk_s2g(a.Zc + (size_t)(cell0 + j) * a.DS + a.c_off, rZ + (size_t)j * DS, (uint32_t)(sizeof(float) * DS));
        umma::bulk_wait_read0();
      } else if (lane == 0) {
        umma::bulk_s2g(a.Zc + (size_t)cell0 * DS, rZ, (uint32_t)(sizeof(float) * len * DS));
        umma::bulk_wait_read0();
      }
      __syncwarp();
      if (tile + NST < t_end) load(it + NST);  // the stage is free: refill it
    }
  }
  if (CR ? w == 0 : wt == 0) umma::bulk_wait0();
}

template <int NH>
__global__ void __launch_bounds__(AP_THREADS, 1) k_apply_tc(ApplyTcArgs a) {
  apply_tc_body<NH, false>(a);
}
__global__ void __launch_bounds__(AP_THREADS, 1) k_apply_tc_cols(ApplyTcArgs a) { apply_tc_body<2, true>(a); }

}  // namespace hb
