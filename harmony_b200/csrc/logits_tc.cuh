// logits_tc.cuh — the cold-start logits of harmony.cpp:220-223 for shapes the fused assignment kernel
// (assign_tc3.cuh) cannot hold in shared memory (d > 64 or K > 128; BASELINE.json config 5: K = 200, d = 100):
//   U[i][k] = -dist_ik / sigma_k = (2 / sigma_k) (z_i . y_k / |z_i| - 1)        for clusters k in [n_off, n_off + 64)
// as one wgmma contraction per 128-cell tile and cluster range (3xTF32, fp32 accumulators in registers).  The softmax
// and the per-block column sums need the whole row, so they are NOT fused here: k_softmax_block_sums (below) makes one
// gather pass over U in the update plan's order — the update kernel recomputes R from U anyway.  The tf32 operand pair
// of all of Y (160 KB at K = 200, d = 100) does not fit beside a cell tile; 64 clusters per launch do (53 KB), at the
// price of re-reading Z once per range: 4 x 400 + 800 B per cell at config 5 against ~40 kflop of FFMA work.
// Same operand pipeline as assign_tc3.cuh: a loader thread copies ITS row with 16-byte cp.async into the canonical
// K-major layout (the raw fp32 tile is the `hi` operand), waits for its own copies, writes the `lo` pieces and the
// row norm; then the four loader warps, one warpgroup, multiply the tile (two 64-row halves, m64n64k8) and leave the
// accumulator in the U stage.  One operand stage (a second one does not fit at d = 100): the epilogue of tile t
// overlaps the load and the MMAs of tile t + 1.
// Warp roles (384 threads): 0-3 loaders / converters / MMA warpgroup (row per thread), 4-11 epilogue (row quarter x
// column half).  Limits: d <= 128.
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int LG_TM = 128;      // cells per tile (two wgmma M = 64 halves)
constexpr int LG_NP = 64;       // clusters per launch (= wgmma N)
constexpr int LG_THREADS = 384;
constexpr int LG_SS = 68;       // row stride of the U stage in floats ((SS / 4) odd: conflict-free row-per-thread stores)

struct LogitsArgs {
  const float* Zc;      // [n][DS]
  const float* Y;       // [K][d]
  const float* sigma;   // [K]
  float* U;             // [n][KS]
  int64_t n;
  int d, K, DS, KS, KD;  // KD = d rounded up to a multiple of 8
  int n_off;            // first cluster of this launch (a multiple of 4)
  int normalise;        // divide by the row norm (cold start)
};

__host__ __device__ inline size_t logits_smem_bytes(int KD) {
  // A hi (raw) + lo, B hi/lo, U stage, 2/sigma, row norms of two tiles
  return sizeof(float) * (2 * (size_t)LG_TM * KD + 2 * (size_t)LG_NP * KD + (size_t)LG_TM * LG_SS + LG_NP + 4 * (size_t)LG_TM) + 256;
}

__global__ void __launch_bounds__(LG_THREADS, 1) k_logits_tc(LogitsArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int KD = a.KD, KS = a.KS, K = a.K, d = a.d, DS = a.DS;
  const int KD4 = KD >> 2, DS4 = DS >> 2;
  float* Ahi = reinterpret_cast<float*>(smem_raw);   // [KD/4][128][4]  raw rows = hi operand
  float* Alo = Ahi + (size_t)LG_TM * KD;
  float* Bhi = Alo + (size_t)LG_TM * KD;             // [KD/4][64][4]
  float* Blo = Bhi + (size_t)LG_NP * KD;
  float* Ust = Blo + (size_t)LG_NP * KD;             // [128][SS]  accumulator, then U
  float* ca = Ust + (size_t)LG_TM * LG_SS;           // [64]  2 / sigma (1e30 in padding columns)
  float* rnorm = ca + LG_NP;                         // [4][128]  1 / |z|
  uint64_t* bars = reinterpret_cast<uint64_t*>(rnorm + 4 * LG_TM);
  uint64_t* t_full = bars;         // MMA warpgroup (128): accumulator in the U stage
  uint64_t* t_empty = bars + 1;    // epilogue (256): U stage drained
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int i = tid; i < LG_NP * KD; i += LG_THREADS) {
    const int n = i / KD, k = i - n * KD;
    const float y = (a.n_off + n < K && k < d) ? a.Y[(size_t)(a.n_off + n) * d + k] : 0.f;
    float hi, lo;
    umma::split_tf32(y, hi, lo);
    const int off = ((k >> 2) * LG_NP + n) * 4 + (k & 3);
    Bhi[off] = hi;
    Blo[off] = lo;
  }
  for (int k = tid; k < LG_NP; k += LG_THREADS) ca[k] = (a.n_off + k < K) ? 2.f / a.sigma[a.n_off + k] : 1.0e30f;  // padding: u = -1e30 = U_PAD
  for (int i = tid; i < LG_TM * KD; i += LG_THREADS) Ahi[i] = 0.f;  // padding chunks / rows beyond short tiles: finite
  if (tid == 0) {
    umma::mbar_init(t_full, 128);
    umma::mbar_init(t_empty, 256);
    umma::fence_barrier_init();
  }
  __syncthreads();

  const int64_t ntiles = (a.n + LG_TM - 1) / LG_TM;
  const int64_t my_first = blockIdx.x, stride = gridDim.x;

  if (warp < 4) {
    // ================= row loaders + converters (one row of the tile per thread), then the MMA warpgroup =================
    const int r = tid;
    const uint32_t lboA = LG_TM * 16, lboB = LG_NP * 16, sbo = 128;
    const uint32_t aH = umma::smem_u32(Ahi), aL = umma::smem_u32(Alo), bH = umma::smem_u32(Bhi), bL = umma::smem_u32(Blo);
    int it = 0;
    for (int64_t tile = my_first; tile < ntiles; tile += stride, ++it) {
      const int64_t cell = tile * LG_TM + r;
      const bool live = cell < a.n;
      // the stage is free: this warpgroup waited for the previous tile's MMAs
      if (live) {
        const float* src = a.Zc + (size_t)cell * DS;
        const unsigned dst = umma::smem_u32(Ahi + (size_t)r * 4);
        for (int c = 0; c < DS4; ++c)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (unsigned)c * (LG_TM * 16u)), "l"(src + 4 * c) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      float ss = 0.f;
      for (int c = 0; c < KD4; ++c) {
        float4 z = make_float4(0.f, 0.f, 0.f, 0.f), l4 = z;
        if (live && c < DS4) {
          z = *reinterpret_cast<const float4*>(Ahi + ((size_t)c * LG_TM + r) * 4);
          ss += (z.x * z.x + z.y * z.y) + (z.z * z.z + z.w * z.w);
          // the tensor core reads trunc_tf32(z); the remainder is exact in fp32 and is rounded to tf32 here
          l4.x = umma::round_tf32(z.x - __uint_as_float(__float_as_uint(z.x) & 0xffffe000u));
          l4.y = umma::round_tf32(z.y - __uint_as_float(__float_as_uint(z.y) & 0xffffe000u));
          l4.z = umma::round_tf32(z.z - __uint_as_float(__float_as_uint(z.z) & 0xffffe000u));
          l4.w = umma::round_tf32(z.w - __uint_as_float(__float_as_uint(z.w) & 0xffffe000u));
        }
        *reinterpret_cast<float4*>(Alo + ((size_t)c * LG_TM + r) * 4) = l4;
      }
      float rn = 1.f;
      if (a.normalise) {
        float nrm = (norm_sq_ok(ss) || !live)
                        ? sqrtf(ss)
                        : norm_rescaled(4 * DS4, [&](int i) { return Ahi[((size_t)(i >> 2) * LG_TM + r) * 4 + (i & 3)]; });
        if (nrm == 0.f) nrm = 1.f;  // arma::normalise: zero norm divides by 1
        rn = 1.f / nrm;
      }
      rnorm[(size_t)(it & 3) * LG_TM + r] = live ? rn : 0.f;
      umma::fence_proxy_async();  // this thread's cp.async rows (observed above) and `lo` writes -> tensor core
      umma::named_sync(2, 128);
      for (int g = 0; g < 2; ++g) {  // rows 64 g .. 64 g + 63 of the tile
        float acc[32];  // overwritten by the first MMA (accumulate = 0)
        umma::fence();
        for (int ks = 0; ks < KD / 8; ++ks) {
          const uint32_t ao = ks * 2 * lboA + g * 64 * 16, bo = ks * 2 * lboB;
          const uint64_t ah = umma::make_desc(aH + ao, lboA, sbo);
          const uint64_t al = umma::make_desc(aL + ao, lboA, sbo);
          const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo);
          const uint64_t bl = umma::make_desc(bL + bo, lboB, sbo);
          umma::mma_n64(acc, al, bh, ks > 0);
          umma::mma_n64(acc, ah, bl, 1);
          umma::mma_n64(acc, ah, bh, 1);
        }
        umma::commit();
        umma::wait0();
        if (g == 0 && it >= 1) umma::mbar_wait(t_empty, (it - 1) & 1);  // the epilogue is done with the previous tile
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int row = 64 * g + umma::frag_row(i, warp, lane), col = umma::frag_col(i, lane);
          *reinterpret_cast<float2*>(Ust + (size_t)row * LG_SS + col) = make_float2(acc[i], acc[i + 1]);
        }
      }
      umma::mbar_arrive(t_full);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // =============================== epilogue ===============================
    const int ew = warp - 4;           // 0..7
    const int q = warp & 3;            // row quarter
    const int h = ew >> 2;             // column half: clusters [32 h, 32 h + 32) of the range
    const int r = q * 32 + lane;       // row of the tile
    const int ncol4 = ((KS - a.n_off < LG_NP ? KS - a.n_off : LG_NP) + 3) >> 2;  // 16-byte pieces of the range inside a U row
    int it = 0;
    for (int64_t tile = my_first; tile < ntiles; tile += stride, ++it) {
      const int64_t cell0 = tile * LG_TM;
      const int len = (int)(a.n - cell0 < LG_TM ? a.n - cell0 : LG_TM);
      umma::mbar_wait(t_full, it & 1);
      const float rn = rnorm[(size_t)(it & 3) * LG_TM + r];
      float* urow = Ust + (size_t)r * LG_SS + 32 * h;
#pragma unroll
      for (int i = 0; i < 32; i += 4) {  // in place: accumulator -> U
        const float4 v = *reinterpret_cast<const float4*>(urow + i);
        const float* cc = ca + 32 * h + i;
        float4 u4;
        u4.x = fmaf(v.x * rn, cc[0], -cc[0]);  // -dist / sigma
        u4.y = fmaf(v.y * rn, cc[1], -cc[1]);
        u4.z = fmaf(v.z * rn, cc[2], -cc[2]);
        u4.w = fmaf(v.w * rn, cc[3], -cc[3]);
        *reinterpret_cast<float4*>(urow + i) = u4;
      }
      umma::named_sync(1, 256);  // the staged tile is complete
      // rows out: 16 lanes per row (64 clusters = 16 pieces of 16 bytes), two rows per warp instruction
      {
        const int sub = lane >> 4, c4 = lane & 15;
        for (int rr = 2 * ew + sub; rr < len; rr += 16) {
          if (c4 < ncol4) {
            const float4 u4 = *reinterpret_cast<const float4*>(Ust + (size_t)rr * LG_SS + 4 * c4);
            *reinterpret_cast<float4*>(a.U + (size_t)(cell0 + rr) * KS + a.n_off + 4 * c4) = u4;
          }
        }
      }
      umma::mbar_arrive(t_empty);  // stage drained -> the MMA warpgroup may leave the next accumulator there
    }
  }
}

// Softmax of the stored logits + column sums per block of an update round (harmony.cpp:224-227 and the removal sums
// of :312-313 for round 0), for launches of k_logits_tc that could not fuse them:
//   slot(j).rem += column sums of R = softmax(U) over the rows of block j, per level;   R itself is not stored.
// grid = (G, nb): CTA (x, j) walks range x of block j of the plan (the ranges of the update kernel; one tuple each).
// One warp per row (lane l owns the 16-byte pieces l, l + 32, ..), 8 warps per CTA.
template <int NV>
__global__ void __launch_bounds__(256) k_softmax_block_sums(const float* __restrict__ U, const int* __restrict__ order,
                                                            const int4* __restrict__ ranges, const int* __restrict__ tuple_levels,
                                                            float* __restrict__ acc, int G, int K, int KS, int C, int B) {
  extern __shared__ __align__(16) float sm_part[];  // [8][128 NV]
  constexpr int KP4 = 128 * NV;
  const int j = blockIdx.y, x = blockIdx.x;
  const int4 rg = ranges[(size_t)j * G + x];
  const int lo = rg.x, hi = rg.y, q = rg.z;
  if (hi <= lo) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS4 = KS >> 2;
  const int BK = B * KS, SL = 2 * (BK + KS);
  float4 cs[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) cs[v] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = lo + warp; r < hi; r += 8) {
    const float4* row = reinterpret_cast<const float4*>(U + (size_t)__ldg(order + r) * KS);
    float4 e[NV];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      e[v] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane + 32 * v < KS4) {
        const float4 u = ld_stream4(row + lane + 32 * v);
        e[v] = make_float4(fast_exp(u.x), fast_exp(u.y), fast_exp(u.z), fast_exp(u.w));  // padding columns: exp(-1e30) = 0
      }
      s += (e[v].x + e[v].y) + (e[v].z + e[v].w);
    }
    s = warp_sum(s);
    const float inv = 1.f / s;  // R.each_row() /= sum(R, 0): no zero guard in the reference
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      cs[v].x = fmaf(e[v].x, inv, cs[v].x);
      cs[v].y = fmaf(e[v].y, inv, cs[v].y);
      cs[v].z = fmaf(e[v].z, inv, cs[v].z);
      cs[v].w = fmaf(e[v].w, inv, cs[v].w);
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) *reinterpret_cast<float4*>(sm_part + (size_t)warp * KP4 + 4 * (lane + 32 * v)) = cs[v];
  __syncthreads();
  float* slot = acc + (size_t)(j + 1) * SL;
  float* rem_O = slot + BK + KS;
  float* rem_rs = rem_O + BK;
  for (int k = tid; k < K; k += 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sm_part[(size_t)w * KP4 + k];
    atomicAdd(rem_rs + k, t);
    for (int c = 0; c < C; ++c) atomicAdd(rem_O + (size_t)tuple_levels[q * C + c] * KS + k, t);
  }
}

}  // namespace hb
