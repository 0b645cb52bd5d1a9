// stats_tc3.cuh — K3 on the tensor cores: the ridge sufficient statistics of harmony.cpp:561-567 / 592-609 for
// all clusters at once,
//   S[q][k][c] = sum_{cells i of tuple q} R[i][k] * Z1[i][c],   Z1 = [Zo | 1]   (column d carries sum_i R_ik)
// as D[128 clusters x 64 columns] += A * B^T with the CELLS as the reduction dimension.  The operands are K-major
// with K = cells (wgmma takes tf32 operands K-major only), i.e. the TRANSPOSE of the row-major tiles in memory, so
// the converter threads transpose while they split into tf32 hi / lo.
// Second generation.  The first one staged raw tiles in shared memory (bulk copies) and converted them into ONE
// operand stage: 2.9 us per 64-cell tile in a chain load -> convert -> MMA -> convert.  Here the converter threads
// read their values straight from global memory (lanes along the cluster / column index: 128-byte segments of a
// row), one tile AHEAD in registers, and the freed shared memory holds TWO operand stages: the conversion of tile
// t + 1 overlaps the MMAs of tile t.  Persistent CTA per SM over a contiguous range of 64-cell tiles; the
// accumulator stays in the registers of the MMA warpgroup across the tiles of one covariate tuple and is flushed
// with atomics when the tuple changes.
//   warps 0-3  MMA warpgroup : 2 halves x 3 x 8 wgmma (M=64, N=64, K=8 cells) per tile, 64 accumulators per thread
//   warps 4-11 convert       : global -> registers (next tile) -> K-major tf32 hi/lo stages
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int ST_TN = 64;        // cells per tile = reduction length per stage (8 wgmma K-steps)
constexpr int ST_THREADS = 384;  // warps 0-3 MMA warpgroup, warps 4-11 converters
constexpr int ST_CONV = 256;     // converter threads

struct StatsTcArgs {
  const float* R;   // [n][KS]
  const float* Zo;  // [n][DS]
  const int* tile_cell0;
  const int* tile_len;
  const int* tile_tuple;
  float* S;         // [J][K][d+1]
  int ntiles, d, K, KS, DS, tiles_per_cta;
  int k_off, c_off;  // this launch: clusters [k_off, k_off + 128) x columns [c_off, c_off + 64) of [Zo | 1] (wider shapes: several launches)
};

__host__ __device__ inline size_t stats_tc_smem_bytes(int KS, int DS) {
  // two operand stages: A hi/lo 2 x 128 x 64, B hi/lo 2 x 64 x 64 floats each
  (void)KS;
  (void)DS;
  return sizeof(float) * 2 * (2 * 128 * ST_TN + 2 * 64 * ST_TN) + 1024;
}

__global__ void __launch_bounds__(ST_THREADS, 1) k_stats_tc(StatsTcArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int K = a.K, d = a.d, KS = a.KS, DS = a.DS, D1 = d + 1;
  constexpr int A_ST = 128 * ST_TN, B_ST = 64 * ST_TN;      // floats per operand tile
  float* Ahi = reinterpret_cast<float*>(smem_raw);          // [2][16 cell chunks][128 clusters][4 cells]
  float* Alo = Ahi + 2 * A_ST;
  float* Bhi = Alo + 2 * A_ST;                              // [2][16][64 columns][4]
  float* Blo = Bhi + 2 * B_ST;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Blo + 2 * B_ST);
  uint64_t* ab_full = bars + 0;     // [2]  converters (256): stage written
  uint64_t* ab_empty = bars + 2;    // [2]  MMA warpgroup (128): stage consumed
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      umma::mbar_init(ab_full + i, ST_CONV);
      umma::mbar_init(ab_empty + i, 128);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();

  const int t_begin = blockIdx.x * a.tiles_per_cta;
  const int t_end = (t_begin + a.tiles_per_cta < a.ntiles) ? t_begin + a.tiles_per_cta : a.ntiles;

  if (warp < 4) {
    // =============================== MMA warpgroup ===============================
    const uint32_t lboA = 128 * 16, lboB = 64 * 16, sbo = 128;
    float acc[2][32];  // clusters 64 g + frag_row, columns frag_col
    int run_acc = 0;   // 0: the first MMA of the tile starts the tuple's sums (overwrites the accumulator)
    int it = 0;
    for (int tile = t_begin; tile < t_end; ++tile, ++it) {
      const int s = it & 1;
      const int q = a.tile_tuple[tile];
      const bool last_of_run = (tile + 1 == t_end) || (a.tile_tuple[tile + 1] != q);
      umma::mbar_wait(ab_full + s, (it >> 1) & 1);
      const uint32_t aH = umma::smem_u32(Ahi + s * A_ST), aL = umma::smem_u32(Alo + s * A_ST);
      const uint32_t bH = umma::smem_u32(Bhi + s * B_ST), bL = umma::smem_u32(Blo + s * B_ST);
      umma::fence();
#pragma unroll
      for (int g = 0; g < 2; ++g)
        for (int ks = 0; ks < ST_TN / 8; ++ks) {
          const uint32_t ao = ks * 2 * lboA + g * 64 * 16, bo = ks * 2 * lboB;
          const uint64_t ah = umma::make_desc(aH + ao, lboA, sbo);
          const uint64_t al = umma::make_desc(aL + ao, lboA, sbo);
          const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
          const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
          umma::mma_n64(acc[g], al, bh, run_acc | (ks > 0));
          umma::mma_n64(acc[g], ah, bl, 1);
          umma::mma_n64(acc[g], ah, bh, 1);
        }
      umma::commit();
      umma::wait0();
      umma::mbar_arrive(ab_empty + s);
      run_acc = last_of_run ? 0 : 1;
      if (last_of_run) {
        // flush the accumulator of this tuple
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int k = a.k_off + 64 * g + umma::frag_row(i, warp, lane), c = a.c_off + umma::frag_col(i, lane);
            if (k < K && c < D1) atomicAdd(a.S + ((size_t)q * K + k) * D1 + c, acc[g][i]);
          }
      }
    }
  } else if (warp >= 4) {
    // =============================== converters ===============================
    const int ct = tid - 128;          // 0..255
    const int kA = ct & 127, ccA = ct >> 7;   // A: cluster kA, cell chunks ccA + 2 i (i < 8)
    const int cB = ct & 63, ccB = ct >> 6;    // B: column cB,  cell chunks ccB + 4 i (i < 4)
    float vA[8][4], vB[4][4];
    // operand pair of a value: hi = the value itself (the tensor core reads its upper 19 bits), lo = the remainder
    // v - trunc_tf32(v), exact in fp32 and truncated by the tensor core in turn (relative error of the pair <= 2^-20)
    auto split = [](float v, float& hi, float& lo) {
      hi = v;
      lo = v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    };
    // tile records (first cell, cells, tuple) run two tiles ahead of the value loads, the value loads one tile ahead of
    // the conversion: no load that feeds an address or a branch is waited for
    auto meta = [&](int tile, int& cell0, int& len, int& q) {
      cell0 = 0;
      len = 0;
      q = -1;
      if (tile < t_end) {
        cell0 = __ldg(a.tile_cell0 + tile);
        len = __ldg(a.tile_len + tile);
        q = __ldg(a.tile_tuple + tile);
      }
    };
    auto fetch = [&](int cell0, int len) {  // this thread's values of a tile, straight from global memory
      const float* rR = a.R + (size_t)cell0 * KS + a.k_off + kA;
      const float* rZ = a.Zo + (size_t)cell0 * DS + a.c_off + cB;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cell = 4 * (ccA + 2 * i) + j;
          vA[i][j] = (cell < len && a.k_off + kA < K) ? ld_stream(rR + (size_t)cell * KS) : 0.f;
        }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cell = 4 * (ccB + 4 * i) + j;
          float v = 0.f;
          if (cell < len) v = (a.c_off + cB < d) ? ld_stream(rZ + (size_t)cell * DS) : (a.c_off + cB == d ? 1.f : 0.f);  // column d: the ones column
          vB[i][j] = v;
        }
    };
    int c0_0, len0, q0, c0_1, len1, q1, c0_2, len2, q2;
    meta(t_begin, c0_0, len0, q0);
    meta(t_begin + 1, c0_1, len1, q1);
    meta(t_begin + 2, c0_2, len2, q2);
    fetch(c0_0, len0);
    int it = 0;
    for (int tile = t_begin; tile < t_end; ++tile, ++it) {
      const int s = it & 1;
      if (it >= 2) umma::mbar_wait(ab_empty + s, ((it >> 1) - 1) & 1);  // MMAs of tile it - 2 are done with the stage
      float* ah = Ahi + s * A_ST;
      float* al = Alo + s * A_ST;
      float* bh = Bhi + s * B_ST;
      float* bl = Blo + s * B_ST;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float4 hi, lo;
        split(vA[i][0], hi.x, lo.x);
        split(vA[i][1], hi.y, lo.y);
        split(vA[i][2], hi.z, lo.z);
        split(vA[i][3], hi.w, lo.w);
        const int off = ((ccA + 2 * i) * 128 + kA) * 4;
        *reinterpret_cast<float4*>(ah + off) = hi;
        *reinterpret_cast<float4*>(al + off) = lo;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float4 hi, lo;
        split(vB[i][0], hi.x, lo.x);
        split(vB[i][1], hi.y, lo.y);
        split(vB[i][2], hi.z, lo.z);
        split(vB[i][3], hi.w, lo.w);
        const int off = ((ccB + 4 * i) * 64 + cB) * 4;
        *reinterpret_cast<float4*>(bh + off) = hi;
        *reinterpret_cast<float4*>(bl + off) = lo;
      }
      umma::fence_proxy_async();
      umma::mbar_arrive(ab_full + s);
      fetch(c0_1, len1);  // the next tile's values travel while this one is multiplied
      c0_0 = c0_1, len0 = len1, q0 = q1;
      c0_1 = c0_2, len1 = len2, q1 = q2;
      meta(tile + 3, c0_2, len2, q2);
    }
  }
}

}  // namespace hb
