// assign_tc3.cuh — K1, the assignment step of harmony.cpp:141-150 (init) / :220-227 (cold start), third generation:
//   cos = z . y_k / |z|,  dist = 2 (1 - cos),  U = -dist / sigma,  R = softmax_k(U),  column sums of R per level
// for tiles of 128 cells, the K x d contraction as wgmma (tf32) in 3xTF32 form, fp32 accumulators in registers.
//
// What changed against k_assign_tc / k_assign_tc2 (both deleted):
//   * the rows of a tile are GATHERED (an index per row) with 16-byte cp.async straight into the canonical K-major
//     wgmma operand layout: the raw fp32 tile IS the `hi` operand (the tensor core reads the upper 19 bits of every
//     word), CUDA cores only produce the `lo` tile (z - trunc_tf32(z), rounded to tf32) and the row norms; the
//     L2 normalisation moves behind the contraction (cos = (z . y) / |z|), so nothing is normalised, split or
//     written back before the MMAs can start.
//   * tiles can follow the update plan of the coming cluster_cpp call (rows of one (block, tuple) segment of round
//     0): the column sums of a tile are then exactly a share of that block's removal sums (harmony.cpp:312-313)
//     and go straight into the update kernel's accumulator slots — R is not stored at all (the update kernel writes
//     it in its last round) and no separate pass over R is needed.  Natural-order mode (init_cluster_cpp, the
//     per-round compatibility paths) stores R and accumulates O / row sums as before.
//   * U rows leave through a shared-memory stage and coalesced row stores (a thread-per-row store of 16-byte pieces
//     costs 32 LSU wavefronts per instruction: 3200 per tile and matrix); exp() is evaluated once per element,
//     the column sums come out of registers through a shuffle butterfly.
// Warp roles (384 threads): 0-3 row gather + `lo` converters (row per thread), then the MMA warpgroup (two 64-row
// halves, m64n32k8 per 32 clusters + m64n16k8 for a 16-cluster tail), which leaves the accumulator columns < KS in
// the U stage (padding clusters have zero centroids: their dot products are 0); 4-11 epilogue (row quarter x
// column half).  Two operand stages: the rows of tile t + 1 land while tile t is multiplied; the epilogue of tile t
// overlaps the conversion and the MMAs of tile t + 1.
// Limits: K <= 128 (NP), d <= 64 (KD); other shapes run the FFMA kernel k_assign.
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int A3_THREADS = 384;
constexpr int A3_NS = 2;          // operand stages (1 when two do not fit shared memory)
constexpr int A3_RING_N = 4;      // row-norm ring (tiles): written by the converters, read at the start of the epilogue
constexpr int A3_RING_C = 8;      // row -> cell ring (tiles): written by the producer, read until the rows have left

struct Assign3Args {
  const float* Zc;          // [n][DS]
  const float* Y;           // [K][d]
  const float* sigma;       // [K]
  float* U;                 // [n][KS]
  float* R;                 // [n][KS]   (natural mode only)
  const int* row_index;     // plan mode: position -> cell (order[] of round 0); null: rows are cells
  const int* tile_p0;       // first position / cell of every tile
  const int* tile_len;
  const int* tile_tuple;
  const int* tile_blk;      // plan mode: block of the tile
  const int* tuple_levels;  // [J][C]
  float* O_acc;             // natural mode: [B][KS] column sums per level, [KS] row sums
  float* rs_acc;
  float* acc;               // plan mode: accumulator slots of the update kernel, slot(j) at (j + 1) * SL
  double* obj_acc;          // [2] (init only)
  float* Zc_out;            // natural mode + normalise: the normalised rows are stored here (null: not stored)
  const int* ntiles_ptr;    // plan mode: tile count on the device (the plan is built without a host round trip)
  int ntiles, d, K, C, B, DS, KS;
  int KD;         // reduction length padded to a multiple of 8
  int NP;         // clusters padded to a multiple of 16
  int SS;         // row stride of the U stage in floats ((SS / 4) odd: conflict-free row-per-thread stores)
  int ns;         // operand stages (1 or 2)
  int normalise;  // divide by the row norm (cold start; init runs on rows that setup normalised)
  int want_obj;   // objective partial sums (init)
};

__host__ __device__ inline int assign3_stage_stride(int KS) { return ((KS >> 2) | 1) << 2; }
__host__ __device__ inline size_t assign3_smem_bytes(int ns, int KD, int NP, int KS) {
  // A hi (raw) + lo per stage, B hi/lo, U stage, per-column constants, metadata rings, row-sum / column-sum scratch
  return sizeof(float) * ((size_t)ns * 2 * TC_TM * KD + 2 * (size_t)NP * KD + (size_t)TC_TM * assign3_stage_stride(KS) +
                          3 * (size_t)NP + (size_t)(A3_RING_N + A3_RING_C) * TC_TM + 2 * (size_t)TC_TM + 4 * (size_t)NP) + 256;
}

template <bool OBJ>
__global__ void __launch_bounds__(A3_THREADS, 1) k_assign_tc3(Assign3Args a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int KD = a.KD, NP = a.NP, KS = a.KS, K = a.K, d = a.d, DS = a.DS, SS = a.SS;
  const int KD4 = KD >> 2, DS4 = DS >> 2, KS4 = KS >> 2;
  const int NS = a.ns;
  float* Ahi = reinterpret_cast<float*>(smem_raw);               // [NS][KD/4][128][4]  raw rows = hi operand
  float* Alo = Ahi + (size_t)NS * TC_TM * KD;                    // [NS][KD/4][128][4]
  float* Bhi = Alo + (size_t)NS * TC_TM * KD;                    // [KD/4][NP][4]
  float* Blo = Bhi + (size_t)NP * KD;
  float* Ust = Blo + (size_t)NP * KD;                            // [128][SS]  accumulator, then U
  float* ca = Ust + (size_t)TC_TM * SS;                          // [NP]  2 / sigma          (1e30 in padding columns)
  float* ca2 = ca + NP;                                          // [NP]  2 log2(e) / sigma
  float* sig = ca2 + NP;                                         // [NP]
  float* rnorm = sig + NP;                                       // [RING_N][128]  1 / |z|
  int* rowcell = reinterpret_cast<int*>(rnorm + (size_t)A3_RING_N * TC_TM);  // [RING_C][128]
  float* rs_part = reinterpret_cast<float*>(rowcell + (size_t)A3_RING_C * TC_TM);  // [2][128]
  float* cs_part = rs_part + 2 * TC_TM;                          // [4][NP]
  uint64_t* bars = reinterpret_cast<uint64_t*>(cs_part + 4 * (size_t)NP);
  uint64_t* t_full = bars;                        // MMA warpgroup (128): accumulator in the U stage
  uint64_t* t_empty = bars + 1;                   // epilogue (256): U stage drained

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr float L2E = 1.4426950408889634f;

  // ---- one-time setup ----
  for (int i = tid; i < NP * KD; i += A3_THREADS) {
    const int n = i / KD, k = i - n * KD;
    const float y = (n < K && k < d) ? a.Y[(size_t)n * d + k] : 0.f;
    float hi, lo;
    umma::split_tf32(y, hi, lo);
    const int off = ((k >> 2) * NP + n) * 4 + (k & 3);
    Bhi[off] = hi;
    Blo[off] = lo;
  }
  for (int k = tid; k < NP; k += A3_THREADS) {
    const float s = (k < K) ? a.sigma[k] : 1.f;
    sig[k] = (k < K) ? s : 0.f;
    ca[k] = (k < K) ? 2.f / s : 1.0e30f;          // padding columns: cos = 0 -> u = -1e30 = U_PAD -> exp = 0
    ca2[k] = (k < K) ? 2.f * L2E / s : 1.0e30f;
  }
  // the hi stages: padding chunks (columns >= DS) and rows beyond short tiles must hold finite values
  for (int i = tid; i < NS * TC_TM * KD; i += A3_THREADS) Ahi[i] = 0.f;
  if (tid == 0) {
    umma::mbar_init(t_full, 128);
    umma::mbar_init(t_empty, 256);
    umma::fence_barrier_init();
  }
  __syncthreads();

  const int my_first = blockIdx.x, stride = gridDim.x;
  if (a.ntiles_ptr) a.ntiles = __ldg(a.ntiles_ptr);

  if (warp < 4) {
    // ============== row loaders + converters (one row of the tile per thread), then the MMA warpgroup ==============
    // Thread r copies ITS row of the next tile with 16-byte cp.async straight into the canonical K-major operand
    // layout (consecutive lanes -> consecutive 16-byte slots of a chunk plane: conflict-free; one warp-wide gather
    // instruction with scattered destinations costs ~290 cycles of a single producer warp, measured), waits for its
    // own copies of the current tile (cp.async.wait_group: no mbarrier between loading and converting), produces the
    // `lo` operand and the row norm; after a warpgroup barrier the same threads multiply the stage.  Plan entries run
    // two tiles ahead.
    const int r = tid;  // row of the tile
    const int nfull = NP >> 5;          // 32-cluster chunks (wgmma N = 32)
    const bool tail = (NP & 16) != 0;   // one 16-cluster chunk after them (wgmma N = 16)
    const uint32_t lboA = TC_TM * 16, lboB = NP * 16, sbo = 128;
    const uint32_t bH = umma::smem_u32(Bhi), bL = umma::smem_u32(Blo);
    auto tile_of = [&](int it) { return my_first + it * stride; };
    auto ld_meta = [&](int it, int& p0, int& len) {
      const int tile = tile_of(it);
      p0 = 0;
      len = 0;
      if (tile < a.ntiles) {
        p0 = __ldg(a.tile_p0 + tile);
        len = __ldg(a.tile_len + tile);
      }
    };
    auto ld_cell = [&](int p0, int len) { return (r < len) ? (a.row_index ? __ldg(a.row_index + p0 + r) : p0 + r) : -1; };
    auto issue_row = [&](int it, int cell) {  // tile `it` -> stage it % NS; always commits
      if (cell >= 0) {
        const int s = it % NS;
        const float* src = a.Zc + (size_t)cell * DS;
        const unsigned dst = umma::smem_u32(Ahi + (size_t)s * TC_TM * KD + (size_t)r * 4);
        for (int c = 0; c < DS4; ++c)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (unsigned)c * (TC_TM * 16u)), "l"(src + 4 * c) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    int p0_0, len0, p0_1, len1, p0_2, len2;
    ld_meta(0, p0_0, len0);
    ld_meta(1, p0_1, len1);
    ld_meta(2, p0_2, len2);
    int cell0 = ld_cell(p0_0, len0), cell1 = ld_cell(p0_1, len1);
    issue_row(0, cell0);
    int it = 0;
    for (int tile = my_first; tile < a.ntiles; tile += stride, ++it) {
      const int s = it % NS;
      // next tile -> the other stage (with one stage: after this tile's MMAs, below); the MMAs of tile it - 1, which
      // used that stage, are complete (this warpgroup waited for them)
      if (NS == 2) {
        issue_row(it + 1, cell1);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      rowcell[(size_t)(it % A3_RING_C) * TC_TM + r] = cell0 >= 0 ? cell0 : 0;
      // plan entries two / three tiles ahead
      const int cell2 = ld_cell(p0_2, len2);
      int p0_3, len3;
      ld_meta(it + 3, p0_3, len3);
      const float* hi = Ahi + (size_t)s * TC_TM * KD;
      float* lo = Alo + (size_t)s * TC_TM * KD;
      float ss = 0.f;
      const bool live = cell0 >= 0;
      for (int c = 0; c < KD4; ++c) {
        float4 z = make_float4(0.f, 0.f, 0.f, 0.f), l4 = z;
        if (live && c < DS4) {
          z = *reinterpret_cast<const float4*>(hi + ((size_t)c * TC_TM + r) * 4);
          ss += (z.x * z.x + z.y * z.y) + (z.z * z.z + z.w * z.w);
          l4 = umma::tf32_lo(z);
        }
        *reinterpret_cast<float4*>(lo + ((size_t)c * TC_TM + r) * 4) = l4;
      }
      float rn = 1.f;
      if (a.normalise) {
        float nrm = (norm_sq_ok(ss) || !live)
                        ? sqrtf(ss)
                        : norm_rescaled(4 * DS4, [&](int i) { return hi[((size_t)(i >> 2) * TC_TM + r) * 4 + (i & 3)]; });
        if (nrm == 0.f) nrm = 1.f;  // arma::normalise: zero norm divides by 1
        rn = 1.f / nrm;
      }
      rnorm[(size_t)(it % A3_RING_N) * TC_TM + r] = live ? rn : 0.f;  // rows beyond the tile: cos = 0, finite exp
      if (a.Zc_out && a.normalise && live) {  // compatibility paths read the normalised embedding back
        float4* zw = reinterpret_cast<float4*>(a.Zc_out + (size_t)cell0 * DS);
        for (int c = 0; c < DS4; ++c) {
          float4 z = *reinterpret_cast<const float4*>(hi + ((size_t)c * TC_TM + r) * 4);
          z.x *= rn;
          z.y *= rn;
          z.z *= rn;
          z.w *= rn;
          zw[c] = z;
        }
      }
      umma::fence_proxy_async();  // this thread's cp.async rows (observed above) and `lo` writes -> tensor core
      umma::named_sync(2, 128);
      {
        const uint32_t aH = umma::smem_u32(Ahi + (size_t)s * TC_TM * KD);
        const uint32_t aL = umma::smem_u32(Alo + (size_t)s * TC_TM * KD);
        for (int g = 0; g < 2; ++g) {  // rows 64 g .. 64 g + 63 of the tile
          float acc[4][16], tl[8];  // overwritten by the first MMA of each chunk (accumulate = 0)
          umma::fence();
          for (int ks = 0; ks < KD / 8; ++ks) {
            const uint32_t ao = ks * 2 * lboA + g * 64 * 16;
            const uint64_t ah = umma::make_desc(aH + ao, lboA, sbo);
            const uint64_t al = umma::make_desc(aL + ao, lboA, sbo);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (j < nfull) {
                const uint32_t bo = ks * 2 * lboB + j * 32 * 16;
                const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
                const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
                umma::mma_n32(acc[j], al, bh, ks > 0);
                umma::mma_n32(acc[j], ah, bl, 1);
                umma::mma_n32(acc[j], ah, bh, 1);
              }
            }
            if (tail) {
              const uint32_t bo = ks * 2 * lboB + nfull * 32 * 16;
              const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
              const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
              umma::mma_n16(tl, al, bh, ks > 0);
              umma::mma_n16(tl, ah, bl, 1);
              umma::mma_n16(tl, ah, bh, 1);
            }
          }
          umma::commit();
          umma::wait0();
          if (g == 0 && it >= 1) umma::mbar_wait(t_empty, (it - 1) & 1);  // the epilogue is done with the previous tile
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j < nfull) {
#pragma unroll
              for (int i = 0; i < 16; i += 2) {
                const int row = 64 * g + umma::frag_row(i, warp, lane), col = 32 * j + umma::frag_col(i, lane);
                if (col < KS) *reinterpret_cast<float2*>(Ust + (size_t)row * SS + col) = make_float2(acc[j][i], acc[j][i + 1]);
              }
            }
          }
          if (tail) {
#pragma unroll
            for (int i = 0; i < 8; i += 2) {
              const int row = 64 * g + umma::frag_row(i, warp, lane), col = 32 * nfull + umma::frag_col(i, lane);
              if (col < KS) *reinterpret_cast<float2*>(Ust + (size_t)row * SS + col) = make_float2(tl[i], tl[i + 1]);
            }
          }
        }
      }
      umma::mbar_arrive(t_full);
      if (NS == 1) issue_row(it + 1, cell1);  // single stage: the next tile's rows land once this tile's MMAs are done
      cell0 = cell1;
      cell1 = cell2;
      p0_2 = p0_3;
      len2 = len3;
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // =============================== epilogue ===============================
    const int ew = warp - 4;           // 0..7
    const int q = warp & 3;            // row quarter
    const int h = ew >> 2;             // column half
    const int r = q * 32 + lane;       // row of the tile
    const int et = ew * 32 + lane;     // 0..255
    const int C0 = NP > 64 ? 64 : NP;
    const int cb = h ? C0 : 0, ce = h ? NP : C0;  // this thread's columns (multiples of 16, at most 64)
    // column owned by this lane after the butterfly (bit i of the column = bit i + 1 of the lane)
    const int bcol = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    float okd = 0.f, oent = 0.f;
    int it = 0;
    // tile records one tile ahead: the loads overlap the previous tile's epilogue instead of opening every tile
    int len_n = 0, tq_n = 0, blk_n = 0;
    if (my_first < a.ntiles) {
      len_n = __ldg(a.tile_len + my_first);
      tq_n = __ldg(a.tile_tuple + my_first);
      blk_n = a.tile_blk ? __ldg(a.tile_blk + my_first) : 0;
    }
    for (int tile = my_first; tile < a.ntiles; tile += stride, ++it) {
      const int len = len_n, tq = tq_n, tblk = blk_n;
      if (tile + stride < a.ntiles) {
        len_n = __ldg(a.tile_len + tile + stride);
        tq_n = __ldg(a.tile_tuple + tile + stride);
        blk_n = a.tile_blk ? __ldg(a.tile_blk + tile + stride) : 0;
      }
      const bool live = r < len;
      umma::mbar_wait(t_full, it & 1);
      const float rn = rnorm[(size_t)(it % A3_RING_N) * TC_TM + r];
      float ev[64];                        // exp(u) of this thread's columns
      float ssum = 0.f, A1 = 0.f, S1 = 0.f;  // sum e, sum e*dist, sum sigma*e*u, sum sigma*e
      float* urow = Ust + (size_t)r * SS;
#pragma unroll
      for (int ci = 0; ci < 4; ++ci) {
        const int c = cb + ci * 16;
        if (c < ce) {
          float v[16];  // accumulator columns c .. c + 15 of this row (0 beyond KS); U overwrites them in place
#pragma unroll
          for (int i = 0; i < 16; i += 4) {
            const float4 v4 = (c + i < KS) ? *reinterpret_cast<const float4*>(urow + c + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            v[i] = v4.x;
            v[i + 1] = v4.y;
            v[i + 2] = v4.z;
            v[i + 3] = v4.w;
          }
          float uu[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float cosv = v[i] * rn;
            uu[i] = fmaf(cosv, ca[c + i], -ca[c + i]);                       // -dist / sigma
            const float e = fast_exp2(fmaf(cosv, ca2[c + i], -ca2[c + i]));  // exp(u)
            ev[ci * 16 + i] = e;
            ssum += e;
            if (OBJ) {
              const float se = sig[c + i] * e;
              A1 = fmaf(se, uu[i], A1);   // sum sigma e u = -sum e dist
              S1 += se;
            }
          }
#pragma unroll
          for (int i = 0; i < 16; i += 4)
            if (c + i < KS) *reinterpret_cast<float4*>(urow + c + i) = make_float4(uu[i], uu[i + 1], uu[i + 2], uu[i + 3]);
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i) ev[ci * 16 + i] = 0.f;
        }
      }
      rs_part[h * TC_TM + r] = ssum;
      umma::named_sync(1, 256);
      // R.each_row() /= sum(R, 0) (no zero guard in the reference); rows beyond the tile weigh 0
      const float tot = rs_part[r] + rs_part[TC_TM + r];
      const float inv = live ? 1.f / tot : 0.f;
      if (OBJ && live) {
        const float ls = __logf(tot);
        okd -= A1 * inv;                  // sum_k R dist (this thread's columns)
        oent += inv * (A1 - ls * S1);     // sum_k sigma R log R,  log R = u - log(sum)
      }
      // column sums of the warp's 32 rows: butterfly; afterwards lane L holds column c + bcol(L)
#pragma unroll
      for (int ci = 0; ci < 4; ++ci) {
        const int c = cb + ci * 16;
        if (c < ce) {
          float rr[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) rr[i] = ev[ci * 16 + i] * inv;
          float w8[8], w4[4], w2[2];
          {
            const bool up = (lane & 16) != 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float send = up ? rr[j] : rr[j + 8];
              const float keep = up ? rr[j + 8] : rr[j];
              w8[j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
          }
          {
            const bool up = (lane & 8) != 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float send = up ? w8[j] : w8[j + 4];
              const float keep = up ? w8[j + 4] : w8[j];
              w4[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
          }
          {
            const bool up = (lane & 4) != 0;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const float send = up ? w4[j] : w4[j + 2];
              const float keep = up ? w4[j + 2] : w4[j];
              w2[j] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
          }
          float w1;
          {
            const bool up = (lane & 2) != 0;
            const float send = up ? w2[0] : w2[1];
            const float keep = up ? w2[1] : w2[0];
            w1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
          }
          w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
          if ((lane & 1) == 0) cs_part[q * NP + c + bcol] = w1;
        }
      }
      // rows out: the staged U tile (and, natural mode, R = exp(U) / row sum) with coalesced row stores
      {
        const int* rc = rowcell + (size_t)(it % A3_RING_C) * TC_TM;
        const bool one = KS4 <= 32;  // one 16-byte piece per lane and row: four rows in flight per warp
        if (one) {
          const bool on = lane < KS4;
          for (int rb = ew; rb < len; rb += 32) {
            int cellv[4];
            float4 u4[4];
            float invr[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int rr2 = rb + 8 * k;
              const int rq = rr2 < len ? rr2 : rb;
              cellv[k] = rc[rq];
              u4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (on) u4[k] = *reinterpret_cast<const float4*>(Ust + (size_t)rq * SS + 4 * lane);
              invr[k] = a.R ? 1.f / (rs_part[rq] + rs_part[TC_TM + rq]) : 0.f;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if (on && rb + 8 * k < len) {
                *reinterpret_cast<float4*>(a.U + (size_t)cellv[k] * KS + 4 * lane) = u4[k];
                if (a.R) {
                  float4 r4;
                  r4.x = fast_exp(u4[k].x) * invr[k];
                  r4.y = fast_exp(u4[k].y) * invr[k];
                  r4.z = fast_exp(u4[k].z) * invr[k];
                  r4.w = fast_exp(u4[k].w) * invr[k];
                  *reinterpret_cast<float4*>(a.R + (size_t)cellv[k] * KS + 4 * lane) = r4;
                }
              }
            }
          }
        } else {
          for (int rr2 = ew; rr2 < len; rr2 += 8) {
            const int cell = rc[rr2];
            const float* us = Ust + (size_t)rr2 * SS;
            float invr = 0.f;
            if (a.R) invr = 1.f / (rs_part[rr2] + rs_part[TC_TM + rr2]);
            for (int c4 = lane; c4 < KS4; c4 += 32) {
              const float4 u4 = *reinterpret_cast<const float4*>(us + 4 * c4);
              *reinterpret_cast<float4*>(a.U + (size_t)cell * KS + 4 * c4) = u4;
              if (a.R) {
                float4 r4;
                r4.x = fast_exp(u4.x) * invr;
                r4.y = fast_exp(u4.y) * invr;
                r4.z = fast_exp(u4.z) * invr;
                r4.w = fast_exp(u4.w) * invr;
                *reinterpret_cast<float4*>(a.R + (size_t)cell * KS + 4 * c4) = r4;
              }
            }
          }
        }
      }
      umma::mbar_arrive(t_empty);  // U stage drained -> the MMA warpgroup may leave the next accumulator there
      umma::named_sync(1, 256);
      // column sums of the tile -> the block's removal sums (plan mode) or O / row sums (natural mode)
      if (et < K) {
        const float t = (cs_part[et] + cs_part[NP + et]) + (cs_part[2 * NP + et] + cs_part[3 * NP + et]);
        float* dO;
        float* drs;
        if (a.tile_blk) {
          const size_t XH = (size_t)a.B * KS + KS;
          float* slot = a.acc + (size_t)(tblk + 1) * 2 * XH;
          dO = slot + XH;              // rem_O
          drs = dO + (size_t)a.B * KS;  // rem_rs
        } else {
          dO = a.O_acc;
          drs = a.rs_acc;
        }
        atomicAdd(drs + et, t);
        for (int c = 0; c < a.C; ++c) atomicAdd(dO + (size_t)__ldg(a.tuple_levels + tq * a.C + c) * KS + et, t);
      }
    }
    if (OBJ) {
      okd = warp_sum(okd);
      oent = warp_sum(oent);
      if (lane == 0) {
        atomicAdd(a.obj_acc + 0, (double)okd);
        atomicAdd(a.obj_acc + 1, (double)oent);
      }
    }
  }
}

}  // namespace hb
