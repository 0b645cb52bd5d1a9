// stats_tc3.cuh — K3 on the tensor cores: the ridge sufficient statistics of harmony.cpp:561-567 / 592-609 for
// all clusters at once,
//   S[q][k][c] = sum_{cells i of tuple q} R[i][k] * Z1[i][c],   Z1 = [Zo | 1]   (column d carries sum_i R_ik)
// as D[clusters x columns] += A * B^T with the CELLS as the reduction dimension, per launch 128 clusters x NB = 64 NH
// columns of [Zo | 1].  A = R^T comes from registers, B = Z1^T from shared memory, 3xTF32, fp32 accumulators in
// registers across the tiles of one covariate tuple, flushed with atomics when the tuple changes.
//   * each tile's rows of R (this launch's clusters) and of Zo (this launch's columns) go into a ring of NST raw
//     stages with bulk asynchronous copies, issued by one warp, whose bytes complete on the stage's "full" mbarrier.
//     A tile never crosses a tuple and cells are sorted by tuple, so when a launch covers whole rows the tile is one
//     contiguous span of each array (one copy each; narrower ranges copy row by row).  The copies of the next
//     NST - 1 tiles stay in flight while a tile is converted and multiplied: at K = 100, d = 50 a stage holds
//     64 x (100 + 52) x 4 B = 38.9 KB and four fit, up to 117-156 KB per SM in flight.
//   * all 256 threads turn the tile's Zo rows into the K-major B operand (cells contiguous per column: the
//     transpose), tf32 hi / lo, with the ones column and zeros beyond the tile; then each MMA warpgroup loads its
//     A fragments (64 clusters x 8 cells per K step, zero beyond the tile and beyond the launch's clusters)
//     straight from the raw R rows, splits them in registers and issues 3 x 8 wgmma, and completes them only after
//     the next tile's B is written (two B buffers for NB = 64; NB = 128 has room for one and waits first).  When
//     both warpgroups have read the stage, warp 0 refills it with tile it + NST.
// Warp roles (256 threads): warpgroup e = 0, 1 owns clusters k_off + 64 e .. + 63 of every tile.
// Shared memory: NBB B buffers of hi/lo 2 x NB x 64 floats ([16][NB][4]), then NST raw stages of 64 x (RK + RC)
// floats (RK, RC = floats of R and of Zo per row in this launch), then the barriers.
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int ST_TN = 64;        // cells per tile = reduction length per tile (8 wgmma K-steps)
constexpr int ST_THREADS = 256;  // two MMA warpgroups
constexpr int ST_MAXST = 4;      // raw stages

struct StatsTcArgs {
  const float* R;   // [n][KS]
  const float* Zo;  // [n][DS]
  const int* tile_cell0;
  const int* tile_len;
  const int* tile_tuple;
  float* S;         // [J][K][d+1]
  int ntiles, d, K, KS, DS, tiles_per_cta;
  int k_off, c_off;  // this launch: clusters [k_off, k_off + 128) x columns [c_off, c_off + NB) of [Zo | 1]
};

// floats per row of a raw stage: this launch's clusters of R, and its columns of Zo (none when it covers only the
// ones column)
__host__ __device__ inline int stats_tc_rk(int KS, int k_off) { return KS - k_off < 128 ? KS - k_off : 128; }
__host__ __device__ inline int stats_tc_rc(int DS, int c_off, int nb) {
  return DS - c_off < nb ? (DS - c_off > 0 ? DS - c_off : 0) : nb;
}
// B hi/lo buffers: two (the conversion of a tile overlaps the MMAs of the previous one) where shared memory allows
__host__ __device__ constexpr int stats_tc_bbufs(int nb) { return nb == 64 ? 2 : 1; }
__host__ __device__ inline size_t stats_tc_fixed_bytes(int nb) {
  return sizeof(float) * 2 * stats_tc_bbufs(nb) * (size_t)nb * ST_TN + ST_MAXST * sizeof(uint64_t);
}
__host__ __device__ inline int stats_tc_stages(int RK, int RC, int nb) {
  const size_t fixed = stats_tc_fixed_bytes(nb);
  const int n = (int)((SMEM_LIMIT - fixed) / (sizeof(float) * (size_t)ST_TN * (RK + RC)));  // >= 2: RK, RC <= 128
  return n < ST_MAXST ? n : ST_MAXST;
}
__host__ __device__ inline size_t stats_tc_smem_bytes(int RK, int RC, int nb) {
  return stats_tc_fixed_bytes(nb) + stats_tc_stages(RK, RC, nb) * sizeof(float) * (size_t)ST_TN * (RK + RC);
}

// NH: 64-column halves of B (1: launches of 64 columns, 2: of 128), fixed at compile time so that the accumulators
// stay in registers
template <int NH>
__global__ void __launch_bounds__(ST_THREADS, 1) k_stats_tc(StatsTcArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int NB = 64 * NH, NBB = stats_tc_bbufs(NB);
  const int K = a.K, d = a.d, KS = a.KS, DS = a.DS, D1 = d + 1;
  const int RK = stats_tc_rk(KS, a.k_off), RC = stats_tc_rc(DS, a.c_off, NB);
  const int Kp = K - a.k_off;                        // clusters of this launch (>= 128: all 128 rows of A)
  const int NST = stats_tc_stages(RK, RC, NB);
  const int SST = ST_TN * (RK + RC);                 // floats per raw stage: R rows [64][RK], then Zo rows [64][RC]
  float* Bhi = reinterpret_cast<float*>(smem_raw);   // [NBB][hi, lo][16 cell chunks][NB columns][4 cells]
  float* raw = Bhi + NBB * 2 * NB * ST_TN;
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
    float* rZ = rR + ST_TN * RK;
    if (lane == 0) {
      umma::mbar_arrive_expect_tx(full + s, (uint32_t)(sizeof(float) * len * (RK + RC)));
      if (RK == KS) umma::bulk_g2s(rR, a.R + (size_t)cell0 * KS, (uint32_t)(sizeof(float) * len * KS), full + s);
      if (RC == DS) umma::bulk_g2s(rZ, a.Zo + (size_t)cell0 * DS, (uint32_t)(sizeof(float) * len * DS), full + s);
    }
    if (RK != KS || (RC != DS && RC > 0)) {  // ranges narrower than the rows: row by row
      __syncwarp();  // the expected bytes are registered before any row completes
      for (int j = lane; j < len; j += 32) {
        if (RK != KS)
          umma::bulk_g2s(rR + (size_t)j * RK, a.R + (size_t)(cell0 + j) * KS + a.k_off, (uint32_t)(sizeof(float) * RK), full + s);
        if (RC != DS && RC > 0)
          umma::bulk_g2s(rZ + (size_t)j * RC, a.Zo + (size_t)(cell0 + j) * DS + a.c_off, (uint32_t)(sizeof(float) * RC), full + s);
      }
    }
  };

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) umma::mbar_init(full + i, 1);
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (warp == 0)
    for (int it = 0; it < NST && t_begin + it < t_end; ++it) load(it);

  const int e = warp >> 2;   // clusters k_off + 64 e ..
  const int w = warp & 3;    // warp of the warpgroup
  const uint32_t lboB = NB * 16, sbo = 128;
  float acc[NB / 2];  // clusters 64 e + frag_row, columns frag_col
  int run_acc = 0;    // 0: the first MMA of the tile starts the tuple's sums (overwrites the accumulator)
  int q_prev = -1;
  // completes the MMAs of the previous tile and flushes the accumulator when that tile ended its tuple's run
  auto retire = [&](bool last_of_run) {
    umma::wait0();
    if (last_of_run) {
#pragma unroll
      for (int i = 0; i < NB / 2; ++i) {
        const int k = a.k_off + 64 * e + umma::frag_row(i, w, lane), c = a.c_off + umma::frag_col(i, lane);
        if (k < K && c < D1) atomicAdd(a.S + ((size_t)q_prev * K + k) * D1 + c, acc[i]);
      }
    }
  };
  for (int tile = t_begin, it = 0; tile < t_end; ++tile, ++it) {
    const int s = it % NST;
    const int len = __ldg(a.tile_len + tile), q = __ldg(a.tile_tuple + tile);
    const float* rR = raw + (size_t)s * SST;
    const float* rZ = rR + ST_TN * RK;
    float* bh_t = Bhi + (NBB == 2 ? (it & 1) * 2 * NB * ST_TN : 0);
    float* bl_t = bh_t + NB * ST_TN;
    if (NBB == 1 && it > 0) {  // one B buffer: both warpgroups finish the previous tile's MMAs before it is rewritten
      retire(q != q_prev);
      umma::named_sync(1, ST_THREADS);
    }
    umma::mbar_wait(full + s, (it / NST) & 1);

    // B = Z1^T of the tile: column c of [Zo | 1] for 4 cells per float4; zero beyond the tile (stale rows) and
    // beyond column d.  hi = the value itself (the tensor core reads its upper 19 bits), lo = the remainder
    // v - trunc_tf32(v), exact in fp32 and truncated by the tensor core in turn (relative error of the pair
    // <= 2^-20).  With two B buffers this overlaps the previous tile's MMAs.
    for (int idx = tid; idx < NB * (ST_TN / 4); idx += ST_THREADS) {
      const int c = idx % NB, ch = idx / NB, cg = a.c_off + c;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int cell = 4 * ch + j;
        v[j] = cell < len ? (cg < d ? rZ[cell * RC + c] : (cg == d ? 1.f : 0.f)) : 0.f;
      }
      float4 hi, lo;
      hi = make_float4(v[0], v[1], v[2], v[3]);
      lo = make_float4(umma::tf32_rem(v[0]), umma::tf32_rem(v[1]), umma::tf32_rem(v[2]), umma::tf32_rem(v[3]));
      *reinterpret_cast<float4*>(bh_t + (ch * NB + c) * 4) = hi;
      *reinterpret_cast<float4*>(bl_t + (ch * NB + c) * 4) = lo;
    }
    // two B buffers: the previous tile's MMAs end before the barrier, so the buffer written at tile it + 1 is free
    if (NBB == 2 && it > 0) retire(q != q_prev);
    umma::fence_proxy_async();
    umma::named_sync(1, ST_THREADS);  // B is written; the stage of the previous tile has been read by everyone
    if (warp == 0 && it > 0 && tile - 1 + NST < t_end) load(it - 1 + NST);
    run_acc = (it > 0 && q == q_prev) ? 1 : 0;
    q_prev = q;

    // A fragments: A[m][kk] = R[cell 8 ks + kk][cluster 64 e + m], split like B
    uint32_t ah[ST_TN / 8][4], al[ST_TN / 8][4];
    {
      const int m0 = 64 * e + 16 * w + (lane >> 2), kk0 = lane & 3;
#pragma unroll
      for (int ks = 0; ks < ST_TN / 8; ++ks)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int m = m0 + 8 * (j & 1), cell = 8 * ks + kk0 + 4 * (j >> 1);
          const float z = (cell < len && m < Kp) ? rR[cell * RK + m] : 0.f;
          ah[ks][j] = __float_as_uint(z);
          al[ks][j] = __float_as_uint(umma::tf32_rem(z));
        }
    }
    const uint32_t bH = umma::smem_u32(bh_t), bL = umma::smem_u32(bl_t);
    umma::fence();
#pragma unroll
    for (int ks = 0; ks < ST_TN / 8; ++ks) {
      const uint32_t bo = ks * 2 * lboB;
      const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
      const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
      if constexpr (NH == 1) {
        umma::mma_rs_n64(acc, al[ks], bh, run_acc | (ks > 0));
        umma::mma_rs_n64(acc, ah[ks], bl, 1);
        umma::mma_rs_n64(acc, ah[ks], bh, 1);
      } else {
        umma::mma_rs_n128(acc, al[ks], bh, run_acc | (ks > 0));
        umma::mma_rs_n128(acc, ah[ks], bl, 1);
        umma::mma_rs_n128(acc, ah[ks], bh, 1);
      }
    }
    umma::commit();
  }
  retire(t_begin < t_end);  // unconditional wait: a conditional one makes ptxas add its own at the loop exit
}

}  // namespace hb
