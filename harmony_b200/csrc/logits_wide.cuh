// logits_wide.cuh — the logits of harmony.cpp:141-147 / :220-223 for embeddings too wide for k_logits_tc (d > 120:
// its A and B operands hold the whole row, 1.5 KB per column of d, and stop fitting shared memory at KD = 128):
//   U[i][k] = -dist_ik / sigma_k = (2 / sigma_k) (z_i . y_k / |z_i| - 1)        for clusters k in [n_off, n_off + 128)
// as one wgmma contraction per 128-cell tile and cluster range (3xTF32, fp32 accumulators in registers), with d streamed
// through a ring of two 32-column chunks: shared memory does not depend on d (2 x 64 KB stages), and any d runs.
//   * The four operand planes of a chunk (A = 128 rows of Z, B = 128 clusters of Y, raw `hi` values and `lo`
//     remainders, K-major canonical layout as in logits_tc.cuh) are filled with 16-byte cp.async by all 256 threads:
//     thread t copies pieces 4 (t / 128) .. + 3 of row t % 128 of both, waits for its own copies, writes their `lo`
//     planes and adds its pieces of Z to the row's sum of squares.  The copies of chunk c + 1 (possibly the first chunk
//     of the next tile) are in flight while chunk c is split and multiplied.
//   * Warpgroup e multiplies rows 64 e .. 64 e + 63 of the tile by the 128 clusters (m64n128k8, 64 accumulators per
//     thread), accumulating across the chunks of the row; after the last chunk it scales by 1 / |z| and 2 / sigma and
//     stores its fragments straight to U (each warp instruction writes 8 rows x 32 contiguous bytes: whole sectors).
//   * Y is read from a copy padded to 128-row and 32-column multiples (k_pad_rows), so every B piece is a 16-byte copy
//     and needs no bounds; Z pieces beyond the row (last chunk) or beyond the last cell are zero-filled by cp.async.
// Traffic: every cell's Z row is read once per cluster range, ceil(K / 128) times (K = 200: twice; K = 1024: 8 times),
// and its U row is written once.  N = 128 halves the re-reads of N = 64 for K > 64 and keeps the accumulators at 64
// registers per thread; N = 256 would need 128 accumulator registers per thread beside the split operands and saves
// a re-read only for K in (128, 256].  Y (at most 4 MB) is read from L2 once per tile and cluster range.
// Rows whose fp32 sum of squares under- or overflows take the rescaled norm of the global row (norm_sq_ok).
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int LW_TM = 128;       // cells per tile (two warpgroups of m64)
constexpr int LW_NP = 128;       // clusters per launch (= wgmma N)
constexpr int LW_DC = 32;        // embedding columns per chunk (four k8 steps)
constexpr int LW_THREADS = 256;
constexpr int LW_PLANE = LW_TM * LW_DC;  // floats of one operand plane (A and B both have 128 rows)

struct LogitsWideArgs {
  const float* Zc;     // [n][DS]
  const float* Ypad;   // [ceil(K / 128) 128][KDc]  Y, zero-padded
  const float* sigma;  // [K]
  float* U;            // [n][KS]
  int64_t n;
  int d, K, DS, KS, KDc;  // KDc = d rounded up to a multiple of LW_DC
  int n_off;              // first cluster of this launch (a multiple of 128)
  int normalise;          // divide by the row norm (cold start)
};

// two stages of four planes, 2 / sigma of the range, the two halves of the rows' sums of squares, 1 / |z|
__host__ __device__ inline size_t logits_wide_smem_bytes() {
  return sizeof(float) * (2 * 4 * (size_t)LW_PLANE + LW_NP + 3 * (size_t)LW_TM);
}

// Ypad[k][c] = Y[k][c] for k < K, c < d, else 0
__global__ void k_pad_rows(const float* __restrict__ Y, float* __restrict__ Ypad, int K, int d, int rows, int ld) {
  const int64_t total = (int64_t)rows * ld;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / ld), c = (int)(i - (int64_t)k * ld);
    Ypad[i] = (k < K && c < d) ? Y[(size_t)k * d + c] : 0.f;
  }
}

__device__ __forceinline__ void cp_async16_zfill(unsigned dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}

__global__ void __launch_bounds__(LW_THREADS, 1) k_logits_wide(LogitsWideArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* stage0 = reinterpret_cast<float*>(smem_raw);  // [2][Ahi | Alo | Bhi | Blo], each [LW_DC / 4][128][4]
  float* ca = stage0 + 2 * 4 * (size_t)LW_PLANE;       // [128]  2 / sigma (1e30 in padding columns)
  float* ssb = ca + LW_NP;                             // [2][128]  halves of the rows' sums of squares
  float* rnb = ssb + 2 * LW_TM;                        // [128]  1 / |z|
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int r = tid & 127, p0 = 4 * (tid >> 7);        // this thread's row and first 16-byte piece of a chunk
  const int KS = a.KS, DS4 = a.DS >> 2, nch = a.KDc / LW_DC;

  for (int k = tid; k < LW_NP; k += LW_THREADS) ca[k] = (a.n_off + k < a.K) ? 2.f / a.sigma[a.n_off + k] : 1.0e30f;  // padding: U_PAD

  const int64_t ntiles = (a.n + LW_TM - 1) / LW_TM;
  const int64_t nmine = ntiles > blockIdx.x ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  const int64_t nchunks = nmine * nch;  // the CTA's chunk stream: tile blockIdx.x + i gridDim.x, chunk c
  auto issue = [&](int64_t g) {
    const int64_t tile = blockIdx.x + (g / nch) * gridDim.x;
    const int c = (int)(g % nch);
    float* st = stage0 + (size_t)(g & 1) * 4 * LW_PLANE;
    const int64_t cell = tile * LW_TM + r;
    const bool live = cell < a.n;
    const float* zrow = a.Zc + (size_t)(live ? cell : 0) * a.DS;
    const float* yrow = a.Ypad + (size_t)(a.n_off + r) * a.KDc + c * LW_DC;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int p = p0 + j, zp = c * (LW_DC / 4) + p;
      const unsigned off = (unsigned)((p * LW_TM + r) * 16);
      const bool ok = live && zp < DS4;
      cp_async16_zfill(umma::smem_u32(st) + off, zrow + 4 * (ok ? zp : 0), ok);
      cp_async16_zfill(umma::smem_u32(st + 2 * LW_PLANE) + off, yrow + 4 * p, true);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  const int e = warp >> 2, w = warp & 3;  // MMA warpgroup e: rows 64 e .. 64 e + 63
  const uint32_t lbo = LW_TM * 16, sbo = 128;
  float acc[64];  // overwritten by the first MMA of a tile (accumulate = 0)
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  float ss = 0.f;
  if (nchunks > 0) issue(0);
  for (int64_t g = 0; g < nchunks; ++g) {
    const int c = (int)(g % nch);
    // the stage of chunk g + 1 was last read by the MMAs of chunk g - 1, which all warpgroups have waited for
    if (g + 1 < nchunks) issue(g + 1);
    else asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");  // this thread's copies of chunk g have landed
    float* st = stage0 + (size_t)(g & 1) * 4 * LW_PLANE;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t off = ((size_t)(p0 + j) * LW_TM + r) * 4;
      const float4 z = *reinterpret_cast<const float4*>(st + off);
      const float4 y = *reinterpret_cast<const float4*>(st + 2 * LW_PLANE + off);
      ss += (z.x * z.x + z.y * z.y) + (z.z * z.z + z.w * z.w);
      *reinterpret_cast<float4*>(st + LW_PLANE + off) = umma::tf32_lo(z);
      *reinterpret_cast<float4*>(st + 3 * LW_PLANE + off) = umma::tf32_lo(y);
    }
    umma::fence_proxy_async();  // this thread's cp.async pieces (observed above) and `lo` writes -> tensor core
    __syncthreads();
    {
      const uint32_t aH = umma::smem_u32(st), aL = aH + 4 * LW_PLANE, bH = aH + 8 * LW_PLANE, bL = aH + 12 * LW_PLANE;
      umma::fence();
#pragma unroll
      for (int ks = 0; ks < LW_DC / 8; ++ks) {
        const uint32_t ao = ks * 2 * lbo + e * 64 * 16, bo = ks * 2 * lbo;
        const uint64_t ah = umma::make_desc(aH + ao, lbo, sbo), al = umma::make_desc(aL + ao, lbo, sbo);
        const uint64_t bh = umma::make_desc(bH + bo, lbo, sbo), bl = umma::make_desc(bL + bo, lbo, sbo);
        umma::mma_n128(acc, al, bh, c > 0 || ks > 0);
        umma::mma_n128(acc, ah, bl, 1);
        umma::mma_n128(acc, ah, bh, 1);
      }
      umma::commit();
      umma::wait0();
    }
    if (c == nch - 1) {
      // ---- tile done: row norms, then U = (2 / sigma) (acc / |z| - 1) straight from the fragments
      const int64_t cell0 = (blockIdx.x + (g / nch) * gridDim.x) * LW_TM;
      ssb[(tid >> 7) * LW_TM + r] = ss;
      ss = 0.f;
      __syncthreads();
      if (tid < LW_TM) {
        float rn = 1.f;
        const int64_t cell = cell0 + r;
        if (a.normalise && cell < a.n) {
          const float s = ssb[r] + ssb[LW_TM + r];
          const float* zrow = a.Zc + (size_t)cell * a.DS;
          float nrm = norm_sq_ok(s) ? sqrtf(s) : norm_rescaled(a.d, [&](int i) { return zrow[i]; });
          if (nrm == 0.f) nrm = 1.f;  // arma::normalise: zero norm divides by 1
          rn = 1.f / nrm;
        }
        rnb[r] = rn;
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 64; i += 2) {
        const int row = 64 * e + umma::frag_row(i, w, lane), col = umma::frag_col(i, lane);
        if (cell0 + row < a.n && a.n_off + col < KS) {
          const float rn = rnb[row];
          *reinterpret_cast<float2*>(a.U + (size_t)(cell0 + row) * KS + a.n_off + col) =
              make_float2(fmaf(acc[i] * rn, ca[col], -ca[col]), fmaf(acc[i + 1] * rn, ca[col + 1], -ca[col + 1]));
        }
      }
    } else {
      __syncthreads();  // both warpgroups are done with the stage before chunk g + 2 refills it
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
}

// Natural-order assignment from stored logits (harmony.cpp:144-150 / :224-227) for shapes whose FFMA k_assign does not
// fit shared memory: R = softmax(U) stored, column sums per 64-row tile (one tuple) -> O_acc per level and rs_acc, and,
// with want_obj, the objective sums sum R dist and sum sigma R log R — what k_assign produces, with the same
// k_assign_finalize after it.  One warp per row (lane l owns the 16-byte pieces l, l + 32, .., KS <= 128 NV; the host
// takes NV = sp_nv(KS), 1 .. 8 for K <= 1024), 8 warps per CTA, the CTA walks tiles; padding columns of U hold U_PAD,
// so their R is 0.
template <int NV>
__global__ void __launch_bounds__(256) k_softmax_tiles(const float* __restrict__ U, float* __restrict__ R,
                                                       const float* __restrict__ sigma, const int* __restrict__ tile_cell0,
                                                       const int* __restrict__ tile_len, const int* __restrict__ tile_tuple,
                                                       const int* __restrict__ tuple_levels, float* __restrict__ O_acc,
                                                       float* __restrict__ rs_acc, double* __restrict__ obj_acc, int ntiles,
                                                       int K, int KS, int C, int want_obj) {
  extern __shared__ __align__(16) float sm_part[];  // [8][128 NV]
  constexpr int KP4 = 128 * NV;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS4 = KS >> 2;
  float4 sg[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int k = 4 * (lane + 32 * v);
    sg[v] = make_float4(k < K ? sigma[k] : 0.f, k + 1 < K ? sigma[k + 1] : 0.f, k + 2 < K ? sigma[k + 2] : 0.f,
                        k + 3 < K ? sigma[k + 3] : 0.f);
  }
  float okd = 0.f, oent = 0.f;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int cell0 = tile_cell0[tile], len = tile_len[tile], q = tile_tuple[tile];
    float4 cs[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) cs[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = warp; r < len; r += 8) {
      const size_t row = (size_t)(cell0 + r) * KS;
      float4 u[NV], ex[NV];
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        u[v] = make_float4(U_PAD, U_PAD, U_PAD, U_PAD);
        if (lane + 32 * v < KS4) u[v] = ld_stream4(reinterpret_cast<const float4*>(U + row) + lane + 32 * v);
        ex[v] = make_float4(expf(u[v].x), expf(u[v].y), expf(u[v].z), expf(u[v].w));
        s += (ex[v].x + ex[v].y) + (ex[v].z + ex[v].w);
      }
      s = warp_sum(s);
      const float ls = logf(s);
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        if (lane + 32 * v >= KS4) continue;
        // R.each_row() /= sum(R, 0): no zero guard in the reference
        const float4 rv = make_float4(ex[v].x / s, ex[v].y / s, ex[v].z / s, ex[v].w / s);
        *reinterpret_cast<float4*>(R + row + 4 * (lane + 32 * v)) = rv;
        cs[v].x += rv.x;
        cs[v].y += rv.y;
        cs[v].z += rv.z;
        cs[v].w += rv.w;
        if (want_obj) {
          const float rr[4] = {rv.x, rv.y, rv.z, rv.w}, uu[4] = {u[v].x, u[v].y, u[v].z, u[v].w};
          const float gg[4] = {sg[v].x, sg[v].y, sg[v].z, sg[v].w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (4 * (lane + 32 * v) + j < K) {
              okd += rr[j] * (-gg[j] * uu[j]);  // dist = -sigma U
              if (rr[j] > 0.f) oent += gg[j] * rr[j] * (uu[j] - ls);
            }
        }
      }
    }
#pragma unroll
    for (int v = 0; v < NV; ++v) *reinterpret_cast<float4*>(sm_part + (size_t)warp * KP4 + 4 * (lane + 32 * v)) = cs[v];
    __syncthreads();
    for (int k = tid; k < K; k += 256) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += sm_part[(size_t)w * KP4 + k];
      atomicAdd(rs_acc + k, t);
      for (int c = 0; c < C; ++c) atomicAdd(O_acc + (size_t)tuple_levels[q * C + c] * KS + k, t);
    }
    __syncthreads();  // the partials are read before the next tile overwrites them
  }
  if (want_obj) {
    okd = warp_sum(okd);
    oent = warp_sum(oent);
    if (lane == 0) {
      atomicAdd(obj_acc + 0, (double)okd);
      atomicAdd(obj_acc + 1, (double)oent);
    }
  }
}

}  // namespace hb
