// apply_tc3.cuh — K5 on the tensor cores: the correction of harmony.cpp:347 + :615 for all clusters at once,
//   Zc_i = Zo_i - sum_k R_ik V_q[k][:]        (q = covariate tuple of cell i, V_q from k_ridge_solve)
// computed transposed so that the per-tile operand is the small one:
//   D'[c][cell] = sum_k A[c][k] * B[cell][k],   A = V_q^T (static while the tuple does not change, M = 64 rows per
//   wgmma, one or two halves for d <= 64 / d <= 128),  B = a 64-cell tile of R (N = 64),  3xTF32, fp32 accumulators
//   in registers.
//   * a loader thread owns half a row of the tile: it copies its 16-byte pieces with cp.async straight into the
//     canonical K-major operand layout (the raw fp32 tile IS the `hi` operand: the tensor core reads the upper 19
//     bits), waits for its OWN copies (cp.async.wait_group, no mbarrier between loading and converting), and writes
//     the `lo` pieces; two or three operand stages, so the rows of tile t + 1 land while tile t is multiplied;
//   * A = V_q^T is rebuilt by the same threads when the tuple changes (after the MMAs of the previous tiles);
//   * two MMA warpgroups take alternate tiles and subtract their accumulators straight from registers
//     (Zc[cell][c] = minuend[cell][c] - D'[c][cell], 32-byte pieces of a row per quad of lanes): the MMAs of one
//     tile overlap the stores of the other.
// Warp roles (384 threads): 0-3 loaders / converters; 4-7 MMA warpgroup of the even tiles, 8-11 of the odd tiles.
// Limits per launch: d <= 128 and <= 112 clusters (shared memory); more clusters run as several launches over
// cluster ranges, each subtracting its share from the partial result (the first from Zo).
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int AP_TN = 64;         // cells per tile (= wgmma N), equals the static tile size TM
constexpr int AP_THREADS = 384;   // 12 warps
constexpr int AP_LOAD = 128;      // loader / converter threads (warps 0-3)
constexpr int AP_MAXK = 112;      // clusters per launch: (2 x 128 + 4 x 64) x KD floats of operands must fit 227 KB

struct ApplyTcArgs {
  const float* R;   // [n][KS]
  const float* Zo;  // [n][DS]
  const float* V;   // [J][K][d]
  float* Zc;        // [n][DS]
  const int* tile_cell0;
  const int* tile_len;
  const int* tile_tuple;
  int ntiles, d, K, KS, DS;
  int k_off, Kp, KD;  // this launch: clusters [k_off, k_off + Kp) (k_off a multiple of 4), KD = Kp rounded up to 8
  const float* minuend;  // Zo for the first cluster range, Zc (the partial result) for the following ones
  int tiles_per_cta;
  // Always null (no caller records stamps): the never-taken stamp branches below stay because they shape ptxas'
  // schedule of k_apply_tc<2>; without them the d > 64 variant runs about 3 % slower (H100 SXM, 400 W).
  long long* dbg;
};

// A = V_q^T is stored with AROWS = 64 rows per 16-byte K chunk when d <= 64 (one wgmma M = 64 half; descriptor
// LBO = 64 x 16 bytes), 128 rows (two halves) otherwise.  The freed 53 KB buy a third operand stage.
__host__ __device__ inline int apply_tc_arows(int d) { return d <= 64 ? 64 : 128; }
__host__ __device__ inline size_t apply_tc_smem_bytes_n(int KD, int d, int nst) {
  // A hi/lo: 2 x AROWS x KD (+ one chunk plane of slack for the aliased rows of the last chunk); B hi/lo: nst x 2 x 64 x KD
  return sizeof(float) * (2 * (size_t)apply_tc_arows(d) * KD + 2 * (size_t)nst * AP_TN * KD) + 1024;
}
__host__ __device__ inline int apply_tc_stages(int KD, int d) {
  return apply_tc_smem_bytes_n(KD, d, 3) <= SMEM_LIMIT ? 3 : 2;
}
__host__ __device__ inline size_t apply_tc_smem_bytes(int KD, int d) { return apply_tc_smem_bytes_n(KD, d, apply_tc_stages(KD, d)); }

// NH: 64-row halves of A = embedding columns (1: d <= 64, 2: d <= 128), fixed at compile time so that the
// accumulators and minuends stay in registers
template <int NH>
__global__ void __launch_bounds__(AP_THREADS, 1) k_apply_tc(ApplyTcArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int KD = a.KD, K = a.K, d = a.d, KS = a.KS, DS = a.DS, Kp = a.Kp;
  const int AR = apply_tc_arows(d);       // rows of A per K chunk
  const int NST = apply_tc_stages(KD, d);  // operand stages of B
  const int BST = AP_TN * KD;              // floats per B tile
  float* Ahi = reinterpret_cast<float*>(smem_raw);  // [KD/4][AR][4]   V_q^T
  float* Alo = Ahi + (size_t)AR * KD;
  float* Bhi = Alo + (size_t)AR * KD;                // [NST][KD/4][64][4]  raw R rows = hi operand
  float* Blo = Bhi + (size_t)NST * BST;              // [NST][KD/4][64][4]
  uint64_t* bars = reinterpret_cast<uint64_t*>(Blo + (size_t)NST * BST);
  uint64_t* lo_full = bars + 0;    // [3]  loaders (128): operands of the stage complete
  uint64_t* st_empty = bars + 3;   // [3]  MMA warpgroup (128): operands consumed
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R4 = ((KS - a.k_off < KD ? KS - a.k_off : KD)) >> 2;   // 16-byte chunks of this launch's cluster range in a row of R

  // the padding chunks of B (k >= KS) are never written by the loaders and must be zero (0 x NaN would poison D')
  for (int i = tid; i < 2 * NST * BST; i += AP_THREADS) Bhi[i] = 0.f;
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) {
      umma::mbar_init(lo_full + i, AP_LOAD);
      umma::mbar_init(st_empty + i, 128);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();

  const int t_begin = blockIdx.x * a.tiles_per_cta;
  const int t_end = (t_begin + a.tiles_per_cta < a.ntiles) ? t_begin + a.tiles_per_cta : a.ntiles;
  auto stamp = [&](int it, int slot) {
    if (a.dbg && blockIdx.x == 0 && it < 32) {
      long long tns;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tns));
      a.dbg[it * 16 + slot] = tns;
    }
  };

  if (warp < 4) {
    // =============================== loaders / converters ===============================
    const int lt = tid;                  // 0..127
    const int cell = lt & (AP_TN - 1);   // row of the tile
    const int half = lt >> 6;            // which half of the row's 16-byte pieces
    const int hsplit = (R4 + 1) >> 1;
    const int c_lo = half ? hsplit : 0, c_hi = half ? R4 : hsplit;
    auto meta = [&](int it, int& cell0, int& len, int& q) {
      const int tile = t_begin + it;
      cell0 = 0;
      len = 0;
      q = -1;
      if (tile < t_end) {
        cell0 = __ldg(a.tile_cell0 + tile);
        len = __ldg(a.tile_len + tile);
        q = __ldg(a.tile_tuple + tile);
      }
    };
    auto issue_row = [&](int it, int cell0, int len) {  // tile `it` -> stage it % NST; always commits
      if (cell < len) {
        const float* src = a.R + (size_t)(cell0 + cell) * KS + a.k_off;
        const unsigned dst = umma::smem_u32(Bhi + (size_t)(it % NST) * BST + (size_t)cell * 4);
        for (int c = c_lo; c < c_hi; ++c)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (unsigned)c * (AP_TN * 16u)), "l"(src + 4 * c) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    auto wait_mma = [&](int t) { umma::mbar_wait(st_empty + (t % NST), (t / NST) & 1); };  // MMAs of tile t are done
    // tile records run NST tiles ahead of the conversion: m[j] = record of tile it + j
    int mc[4], ml[4], mq[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) meta(j, mc[j], ml[j], mq[j]);
    issue_row(0, mc[0], ml[0]);  // prologue: NST - 1 tiles in flight
    if (NST == 3) issue_row(1, mc[1], ml[1]);
    int cur_q = -1;
    int it = 0;
    for (int tile = t_begin; tile < t_end; ++tile, ++it) {
      const int s = it % NST;
      if (lt == 0) stamp(it, 0);
      if (NST == 3)
        asm volatile("cp.async.wait_group 1;" ::: "memory");  // this tile's pieces have landed (tile it + 1 may be in flight)
      else
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      if (lt == 0) stamp(it, 1);
      if (mq[0] != cur_q) {
        // new tuple: A = V_q^T (k contiguous per embedding column c), tf32 hi/lo — after the MMAs of the previous
        // tiles (the two warpgroups finish theirs in either order)
        if (it >= 1) wait_mma(it - 1);
        if (it >= 2) wait_mma(it - 2);
        const float* Vq = a.V + ((size_t)mq[0] * K + a.k_off) * d;
        for (int idx = lt; idx < AR * KD; idx += AP_LOAD) {
          const int k = idx / AR, c = idx - k * AR;
          const float v = (k < Kp && c < d) ? Vq[(size_t)k * d + c] : 0.f;
          float hi, lo;
          umma::split_tf32(v, hi, lo);
          const int off = ((k >> 2) * AR + c) * 4 + (k & 3);
          Ahi[off] = hi;
          Alo[off] = lo;
        }
        cur_q = mq[0];
      }
      // `lo` pieces of this thread's half row: the remainder z - trunc_tf32(z) is exact in fp32; the tensor core
      // truncates it to tf32 like it truncates z itself (relative error of the pair <= 2^-20).  Rows beyond the
      // tile keep whatever the stage holds: their columns of D' are not read.
      {
        const float* hi = Bhi + (size_t)s * BST + (size_t)cell * 4;
        float* lo = Blo + (size_t)s * BST + (size_t)cell * 4;
        if (cell < ml[0]) {
          for (int c = c_lo; c < c_hi; ++c) {
            const float4 z = *reinterpret_cast<const float4*>(hi + (size_t)c * AP_TN * 4);
            float4 l4;
            l4.x = z.x - __uint_as_float(__float_as_uint(z.x) & 0xffffe000u);
            l4.y = z.y - __uint_as_float(__float_as_uint(z.y) & 0xffffe000u);
            l4.z = z.z - __uint_as_float(__float_as_uint(z.z) & 0xffffe000u);
            l4.w = z.w - __uint_as_float(__float_as_uint(z.w) & 0xffffe000u);
            *reinterpret_cast<float4*>(lo + (size_t)c * AP_TN * 4) = l4;
          }
        }
      }
      umma::fence_proxy_async();  // this thread's cp.async pieces (observed above), `lo` and A writes -> tensor core
      umma::mbar_arrive(lo_full + s);
      if (lt == 0) stamp(it, 2);
      // tile it + NST - 1 goes into the stage tile it - 1 used: after that tile's MMAs
      if (tile + NST - 1 < t_end && it >= 1) wait_mma(it - 1);
      issue_row(it + NST - 1, NST == 3 ? mc[2] : mc[1], NST == 3 ? ml[2] : ml[1]);
      if (lt == 0) stamp(it, 3);
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        mc[j] = mc[j + 1];
        ml[j] = ml[j + 1];
        mq[j] = mq[j + 1];
      }
      meta(it + 4, mc[3], ml[3], mq[3]);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // =============================== MMA warpgroups + epilogue ===============================
    const int e = (warp >> 2) - 1;   // tiles t_begin + e, + e + 2, ..
    const int w = warp & 3;          // warp of the warpgroup
    const uint32_t lboA = (uint32_t)AR * 16, lboB = AP_TN * 16, sbo = 128;
    const uint32_t aH = umma::smem_u32(Ahi), aL = umma::smem_u32(Alo);
    for (int tile = t_begin + e; tile < t_end; tile += 2) {
      const int it = tile - t_begin, s = it % NST;
      const int cell0 = __ldg(a.tile_cell0 + tile), len = __ldg(a.tile_len + tile);
      // the minuend of this thread's accumulator elements travels while the operands are prepared and multiplied
      float zo[NH][32];
#pragma unroll
      for (int g = 0; g < NH; ++g)
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int c = 64 * g + umma::frag_row(i, w, lane), j = umma::frag_col(i, lane);
          zo[g][i] = (c < d && j < len) ? ld_stream(a.minuend + (size_t)(cell0 + j) * DS + c) : 0.f;
        }
      umma::mbar_wait(lo_full + s, (it / NST) & 1);
      if (lane == 0 && w == 0) stamp(it, 5);
      float acc[NH][32];  // overwritten by the first MMA of each half (accumulate = 0)
      const uint32_t bH = umma::smem_u32(Bhi + (size_t)s * BST), bL = umma::smem_u32(Blo + (size_t)s * BST);
      umma::fence();
#pragma unroll
      for (int g = 0; g < NH; ++g) {
        {
          for (int ks = 0; ks < KD / 8; ++ks) {
            const uint32_t ao = ks * 2 * lboA + g * 64 * 16, bo = ks * 2 * lboB;
            const uint64_t ah = umma::make_desc(aH + ao, lboA, sbo);
            const uint64_t al = umma::make_desc(aL + ao, lboA, sbo);
            const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
            const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
            umma::mma_n64(acc[g], al, bh, ks > 0);
            umma::mma_n64(acc[g], ah, bl, 1);
            umma::mma_n64(acc[g], ah, bh, 1);
          }
        }
      }
      umma::commit();
      umma::wait0();
      umma::mbar_arrive(st_empty + s);  // operands consumed -> the loaders may refill the stage
      if (lane == 0 && w == 0) stamp(it, 7);
#pragma unroll
      for (int g = 0; g < NH; ++g)
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int c = 64 * g + umma::frag_row(i, w, lane), j = umma::frag_col(i, lane);
          if (c < d && j < len) a.Zc[(size_t)(cell0 + j) * DS + c] = zo[g][i] - acc[g][i];
        }
      if (lane == 0 && w == 0) stamp(it, 9);
    }
  }
}

}  // namespace hb
