// knn.cuh — exact k nearest rows of a reference X for every row of a query Q (DESIGN §9), sm_90a.
//   k_knn_colsum   column sums of the finite entries of X: the centre c both sides are shifted by (Euclidean only;
//                  distances do not change, and q.x - |x|^2 / 2 stops cancelling for data far from the origin)
//   k_knn_prepare  rows of any stride and dtype -> padded fp32 rows [n][KD] (centred, or normalised for cosine) and
//                  hx[j] = |x_j|^2 / 2 (0 for cosine): both metrics become "largest q.x - hx"
//   k_knn_tc       a CTA keeps TQ query rows as tf32 hi / lo operands in shared memory and streams its range of the
//                  reference past them once, KNN_TN = 64 rows per tile, wgmma m64n64k8 in 3xTF32.  The scores stay in the
//                  accumulator registers: a thread compares its fragment with its rows' thresholds (the k-th best so
//                  far); survivors go to a per-row candidate buffer which the row's warp folds into the row's sorted
//                  list.  A query row's fragments all lie in one warp (umma::frag_row), so lists need no CTA barrier.
//                  GROUPED (hb_kbet): a CTA takes its query rows [r0, r1) and its reference rows [g0, g1) from a tile
//                  record, one reference split, and every row number is a position in the caller's sorted order.
//   k_knn_merge    per query row: the direct fp32 distance of every listed candidate of every reference split, the k
//                  smallest in ascending order.
// Operand pipeline as in logits_tc.cuh: per-thread 16-byte cp.async into the canonical K-major layout, the raw tile is
// the `hi` operand, the `lo` pieces are written once the copies have landed.  k_silhouette_tc runs the same pipeline,
// written out in its kernel as here: taken out into a shared struct, it made ptxas serialise the wgmma (DESIGN §9).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "umma.cuh"

namespace hb {

constexpr int KNN_CAP = 16;          // candidate slots per query row; a fold is due above KNN_CAP - 8
constexpr int KNN_SS = 18;           // row stride of a warp's 16 x 16 score stage (even: 8-byte stores)
constexpr int KNN_TN = 64;           // reference rows per tile (= wgmma N)
constexpr int KNN_MAX_K = 64;       // hb_knn's k
constexpr int KNN_SWEEP_MAX_K = 128; // the sweep's: a list of 4 entries per lane (hb_lisi)
constexpr int KNN_MAX_D = 128;
constexpr int KNN_MERGE_MAX = 1024;  // candidates per query row in k_knn_merge (splits * k)
constexpr float KNN_INF = __builtin_huge_valf();

// Shared memory of the sweep's operand pipeline (k_knn_tc, k_silhouette_tc): Q hi / lo, reference stages + one lo
// tile, hx of two tiles
__host__ __device__ inline size_t sweep_smem_bytes(int tq, int stages, int KD) {
  return 4 * (2 * (size_t)tq * KD + (size_t)(stages + 1) * KNN_TN * KD + 2 * (size_t)KNN_TN) + 256;
}
// k_knn_tc's shared memory past the pipeline, per query row: threshold, count, list, candidate buffer and the row's
// share of its warp's score stage
__host__ __device__ inline size_t knn_row_bytes(int k) { return 4 * (2 + 2 * (size_t)k + 2 * KNN_CAP + KNN_SS); }

// ---- preparation ----------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_knn_colsum(const T* __restrict__ X, int64_t ld, int64_t n, int d, double* __restrict__ sum) {
  __shared__ double part[256];
  const int c = threadIdx.x % KNN_MAX_D, half = threadIdx.x / KNN_MAX_D;  // two rows in flight per CTA
  double s = 0.0;
  if (c < d)
    for (int64_t r = 2 * (int64_t)blockIdx.x + half; r < n; r += 2 * (int64_t)gridDim.x) {
      const double v = (double)X[r * ld + c];
      if (isfinite(v)) s += v;
    }
  part[threadIdx.x] = s;
  __syncthreads();
  if (half == 0 && c < d) atomicAdd(sum + c, part[c] + part[c + KNN_MAX_D]);
}

// One warp per row (d <= 128: four values per lane).  centre: column sums (divided by centre_n here) or null.
// GATHER: row r of dst and hx is row perm[r] of src (hb_silhouette's rows in sorted order).
template <typename T, bool GATHER = false>
__global__ void __launch_bounds__(256) k_knn_prepare(const T* __restrict__ src, int64_t ld, int64_t n, int d, int KD,
                                                     int cosine, const double* __restrict__ centre, double centre_n,
                                                     float* __restrict__ dst, float* __restrict__ hx,
                                                     const int* __restrict__ perm) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double c[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) c[i] = (centre && lane + 32 * i < d) ? centre[lane + 32 * i] / centre_n : 0.0;
  for (int64_t r = w; r < n; r += nw) {
    const int64_t sr = GATHER ? (int64_t)perm[r] : r;
    float v[4];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[i] = lane + 32 * i < d ? (float)((double)src[sr * ld + lane + 32 * i] - c[i]) : 0.f;
      ss = fmaf(v[i], v[i], ss);
    }
    ss = warp_sum(ss);
    if (cosine) {
      float nrm = sqrtf(ss);
      if (!norm_sq_ok(ss)) {  // the library's rule (common.cuh): measure again relative to the largest magnitude
        float m = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        nrm = m;
        if (m != 0.f && isfinite(m)) {
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) s = fmaf(v[i] / m, v[i] / m, s);
          nrm = m * sqrtf(warp_sum(s));
        }
      }
      if (nrm == 0.f) nrm = 1.f;  // a zero row divides by 1
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] /= nrm;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (lane + 32 * i < KD) dst[r * KD + lane + 32 * i] = v[i];
    if (hx && lane == 0) hx[r] = cosine ? 0.f : 0.5f * ss;
  }
}

// ---- the sweep ------------------------------------------------------------------------------------------------------
struct KnnArgs {
  const float* Qp;   // [Nq][KD]
  const float* Xp;   // [Nx][KD]
  const float* hx;   // [Nx]
  int* part_i;       // [Nq][splits][k] reference rows by descending score, -1: none
  int64_t Nq, Nx;
  int KD, k, stages, exclude_self;
  int64_t tiles_per_split;
};
// The grouped sweep's arguments: KnnArgs (Nq, Nx and tiles_per_split unused) and the tile records
struct KnnGroupArgs : KnnArgs {
  const int4* tiles;  // {first query row, end query row, first reference row, end reference row}
};

// (score, row) a before (score, row) b in a list: larger score, then smaller row
__device__ __forceinline__ bool knn_before(float sa, int ia, float sb, int ib) { return sa > sb || (sa == sb && ia < ib); }

// The warp folds the candidates of one query row into its list (k <= 32 E entries, best first; lane holds entries
// lane + 32 u) and returns the new threshold.
template <int E>
__device__ __noinline__ float knn_fold(float* ls, int* li, const float* bs, const int* bi, int nb, int k, int lane) {
  float s[E], cs = 0.f;
  int id[E], ci = 0, rank[E], crank = 0;
#pragma unroll
  for (int u = 0; u < E; ++u) {
    const int e = lane + 32 * u;
    if (e < k) {
      s[u] = ls[e];
      id[u] = li[e];
      int rk = e;  // the list is in order: only the candidates can move an entry down
      for (int b = 0; b < nb; ++b) rk += knn_before(bs[b], bi[b], s[u], id[u]);
      rank[u] = rk;
    }
  }
  if (lane < nb) {
    cs = bs[lane];
    ci = bi[lane];
    for (int e = 0; e < k; ++e) crank += !knn_before(cs, ci, ls[e], li[e]);
    for (int b = 0; b < nb; ++b) crank += knn_before(bs[b], bi[b], cs, ci);
  }
  __syncwarp();
#pragma unroll
  for (int u = 0; u < E; ++u)
    if (lane + 32 * u < k && rank[u] < k) {
      ls[rank[u]] = s[u];
      li[rank[u]] = id[u];
    }
  if (lane < nb && crank < k) {
    ls[crank] = cs;
    li[crank] = ci;
  }
  __syncwarp();
  return ls[k - 1];
}

// grid = (query tiles, reference splits), 2 TQ threads: warpgroup g multiplies query rows [64 g, 64 g + 64) of the tile.
// E: list entries per lane, k <= 32 E (2 for hb_knn's k <= 64, 4 up to KNN_SWEEP_MAX_K).  GROUPED: grid = tile records.
template <int TQ, int E, bool GROUPED = false>
__global__ void __launch_bounds__(2 * TQ, 1) k_knn_tc(std::conditional_t<GROUPED, KnnGroupArgs, KnnArgs> a) {
  constexpr int TN = KNN_TN;
  constexpr int THREADS = 2 * TQ, NACC = TN / 2, NG = TN / 8, NCH = TN / 16;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int KD = a.KD, KD4 = KD >> 2, k = a.k, S = a.stages;
  float* Qhi = reinterpret_cast<float*>(smem_raw);  // [KD/4][TQ][4]
  float* Qlo = Qhi + (size_t)TQ * KD;
  float* Braw = Qlo + (size_t)TQ * KD;              // [S][KD/4][TN][4]  raw rows = hi operand
  float* Blo = Braw + (size_t)S * TN * KD;
  float* hxs = Blo + (size_t)TN * KD;               // [2][TN]  hx of the tile, +inf past Nx
  float* thr = hxs + 2 * TN;                        // [TQ]  k-th best score so far
  int* cnt = reinterpret_cast<int*>(thr + TQ);      // [TQ]  filled candidate slots
  float* lst_s = reinterpret_cast<float*>(cnt + TQ);  // [TQ][k]
  int* lst_i = reinterpret_cast<int*>(lst_s + (size_t)TQ * k);
  float* buf_s = reinterpret_cast<float*>(lst_i + (size_t)TQ * k);  // [TQ][KNN_CAP]
  int* buf_i = reinterpret_cast<int*>(buf_s + (size_t)TQ * KNN_CAP);
  float* stage = reinterpret_cast<float*>(buf_i + (size_t)TQ * KNN_CAP);  // [warps][16][KNN_SS]  a chunk of scores
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, w4 = warp & 3;
  int64_t q0, q_end, x0, x_end;  // query rows [q0, q_end) of this CTA (q_end: a bound, not the tile's end) and the reference's
  if constexpr (GROUPED) {
    const int4 tile = a.tiles[blockIdx.x];
    q0 = tile.x, q_end = tile.y, x0 = tile.z, x_end = tile.w;
  } else {
    q0 = (int64_t)blockIdx.x * TQ, q_end = a.Nq, x0 = 0, x_end = a.Nx;
  }
  const int64_t xtiles = (x_end - x0 + TN - 1) / TN;
  const int64_t t_begin = GROUPED ? 0 : (int64_t)blockIdx.y * a.tiles_per_split;
  const int64_t t_end = GROUPED ? xtiles : t_begin + a.tiles_per_split < xtiles ? t_begin + a.tiles_per_split : xtiles;

  // reference tile t -> stage buffer (row per thread, one 16-byte piece per chunk) and its hx
  auto issue = [&](int64_t t) {
    float* dst = Braw + (size_t)(S == 2 ? (t & 1) : 0) * TN * KD;
    const int r = tid % TN;
    const int64_t j = x0 + t * TN + r;
    if (j < x_end) {
      const float* src = a.Xp + (size_t)j * KD;
      const unsigned d0 = umma::smem_u32(dst + (size_t)r * 4);
      for (int c = tid / TN; c < KD4; c += THREADS / TN)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d0 + (unsigned)c * (TN * 16u)), "l"(src + 4 * c) : "memory");
    }
    if (tid < TN) hxs[(t & 1) * TN + tid] = j < x_end ? a.hx[j] : KNN_INF;  // rows past the end score -inf (or NaN)
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (t_begin < t_end) issue(t_begin);

  for (int i = tid; i < TQ * KD4; i += THREADS) {
    const int r = i % TQ, c = i / TQ;
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < q_end) z = *reinterpret_cast<const float4*>(a.Qp + (size_t)(q0 + r) * KD + 4 * c);
    const float4 l4 = umma::tf32_lo(z);
    *reinterpret_cast<float4*>(Qhi + ((size_t)c * TQ + r) * 4) = z;
    *reinterpret_cast<float4*>(Qlo + ((size_t)c * TQ + r) * 4) = l4;
  }
  for (int i = tid; i < TQ; i += THREADS) {
    thr[i] = -KNN_INF;
    cnt[i] = 0;
  }
  for (int i = tid; i < TQ * k; i += THREADS) {
    lst_s[i] = -KNN_INF;
    lst_i[i] = -1;
  }
  __syncthreads();

  // this thread's two query rows of the tile (accumulator elements with bit 1 clear / set), and its warp's sixteen
  const int row0 = 64 * wg + 16 * w4 + (lane >> 2), row1 = row0 + 8, wrow = 64 * wg + 16 * w4;
  const uint32_t lboA = TQ * 16, lboB = TN * 16, sbo = 128;
  const uint32_t aH = umma::smem_u32(Qhi) + wg * 64 * 16, aL = umma::smem_u32(Qlo) + wg * 64 * 16;
  const uint32_t bL = umma::smem_u32(Blo);

  for (int64_t t = t_begin; t < t_end; ++t) {
    float* raw = Braw + (size_t)(S == 2 ? (t & 1) : 0) * TN * KD;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // tile t is in shared memory; the MMAs of tile t - 1 are complete in every warp
    if (S == 2 && t + 1 < t_end) issue(t + 1);
    for (int i = tid; i < TN * KD4; i += THREADS) {
      const float4 z = *reinterpret_cast<const float4*>(raw + (size_t)i * 4);
      *reinterpret_cast<float4*>(Blo + (size_t)i * 4) = umma::tf32_lo(z);
    }
    umma::fence_proxy_async();  // cp.async rows (observed above) and the `lo` writes -> tensor core
    __syncthreads();
    float acc[NACC];  // overwritten by the first MMA (accumulate = 0)
    {
      const uint32_t bH = umma::smem_u32(raw);
      umma::fence();
      for (int ks = 0; ks < KD / 8; ++ks) {
        const uint32_t ao = ks * 2 * lboA, bo = ks * 2 * lboB;
        const uint64_t ah = umma::make_desc(aH + ao, lboA, sbo), al = umma::make_desc(aL + ao, lboA, sbo);
        const uint64_t bh = umma::make_desc(bH + bo, lboB, sbo), bl = umma::make_desc(bL + bo, lboB, sbo);
        umma::mma_n64(acc, al, bh, ks > 0);
        umma::mma_n64(acc, ah, bl, 1);
        umma::mma_n64(acc, ah, bh, 1);
      }
      umma::commit();
      umma::wait0();
    }
    if (S == 1 && t + 1 < t_end) {
      __syncthreads();  // both warpgroups are done with the only stage
      issue(t + 1);
    }

    // ---- selection: score = q.x - hx against the rows' thresholds ----
    const int64_t j0 = x0 + t * TN;
    const float* hxt = hxs + (t & 1) * TN;
    const float t0 = thr[row0], t1 = thr[row1];
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const float2 h2 = *reinterpret_cast<const float2*>(hxt + 8 * g + 2 * (lane & 3));
      acc[4 * g] -= h2.x;
      acc[4 * g + 1] -= h2.y;
      acc[4 * g + 2] -= h2.x;
      acc[4 * g + 3] -= h2.y;
    }
    if (a.exclude_self && j0 < q0 + TQ && q0 < j0 + TN) {  // the tile holds some of this CTA's own rows
#pragma unroll
      for (int i = 0; i < NACC; ++i) {
        const int64_t j = j0 + umma::frag_col(i, lane);
        acc[i] = j == q0 + ((i & 2) ? row1 : row0) ? -KNN_INF : acc[i];
      }
    }
    // 16-column chunks of the tile with a score above a threshold of the tile's start (thresholds only rise).  The
    // accumulator is read in warp-uniform code only: the survivors of a chunk are found in a copy in shared memory.
    unsigned mine = 0;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const float c0 = fmaxf(fmaxf(acc[8 * c], acc[8 * c + 1]), fmaxf(acc[8 * c + 4], acc[8 * c + 5]));  // fmaxf drops NaN
      const float c1 = fmaxf(fmaxf(acc[8 * c + 2], acc[8 * c + 3]), fmaxf(acc[8 * c + 6], acc[8 * c + 7]));
      mine |= (c0 > t0 || c1 > t1) ? 1u << c : 0u;
    }
    unsigned mask = __reduce_or_sync(0xffffffffu, mine);
    while (mask) {
      const int c = __ffs(mask) - 1;
      mask &= mask - 1;
      float* st = stage + warp * (16 * KNN_SS);
#pragma unroll
      for (int cc = 0; cc < NCH; ++cc)
        if (cc == c) {
          float* s0 = st + (lane >> 2) * KNN_SS + 2 * (lane & 3);
          *reinterpret_cast<float2*>(s0) = make_float2(acc[8 * cc], acc[8 * cc + 1]);
          *reinterpret_cast<float2*>(s0 + 8) = make_float2(acc[8 * cc + 4], acc[8 * cc + 5]);
          *reinterpret_cast<float2*>(s0 + 8 * KNN_SS) = make_float2(acc[8 * cc + 2], acc[8 * cc + 3]);
          *reinterpret_cast<float2*>(s0 + 8 * KNN_SS + 8) = make_float2(acc[8 * cc + 6], acc[8 * cc + 7]);
        }
      __syncwarp();
      // two lanes per row, eight columns per step: a row gains at most 8 candidates between two fold checks
      const int r = wrow + (lane >> 1);
      for (int step = 0; step < 2; ++step) {
        const float tr = thr[r];
        for (int i = 0; i < 4; ++i) {
          const int col = 8 * step + 4 * (lane & 1) + i;
          const float v = st[(lane >> 1) * KNN_SS + col];
          if (v > tr) {
            const int pos = atomicAdd(cnt + r, 1);
            buf_s[r * KNN_CAP + pos] = v;
            buf_i[r * KNN_CAP + pos] = (int)(j0 + 16 * c + col);
          }
        }
        __syncwarp();
        if (__any_sync(0xffffffffu, cnt[r] > KNN_CAP - 8)) {
          for (int rr = wrow; rr < wrow + 16; ++rr) {
            // through a shuffle: ptxas sees the branch around the call as warp-uniform and does not serialise the wgmma
            const int nb = __shfl_sync(0xffffffffu, cnt[rr], 0);
            if (nb > KNN_CAP - 8) {
              const float nt = knn_fold<E>(lst_s + (size_t)rr * k, lst_i + (size_t)rr * k, buf_s + rr * KNN_CAP, buf_i + rr * KNN_CAP, nb, k, lane);
              if (lane == 0) {
                thr[rr] = nt;
                cnt[rr] = 0;
              }
            }
          }
          __syncwarp();
        }
      }
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");

  // the candidates still waiting, then this split's lists out
  __syncwarp();
  for (int r = wrow; r < wrow + 16; ++r) {
    const int nb = cnt[r];
    if (nb > 0) knn_fold<E>(lst_s + (size_t)r * k, lst_i + (size_t)r * k, buf_s + r * KNN_CAP, buf_i + r * KNN_CAP, nb, k, lane);
    __syncwarp();
    if (q0 + r < q_end) {
      const size_t o = ((size_t)(q0 + r) * gridDim.y + blockIdx.y) * k;
      for (int e = lane; e < k; e += 32) a.part_i[o + e] = lst_i[(size_t)r * k + e];
    }
  }
}

// ---- merge: direct distances of the listed candidates, the k smallest in order -----------------------------------
// One warp per query row, nc = splits * k <= KNN_MERGE_MAX candidates; a lane computes whole distances.  A candidate
// whose direct distance is NaN or +inf is dropped; missing neighbours are idx = -1, dist = +inf.
__global__ void __launch_bounds__(128, 4) k_knn_merge(const float* __restrict__ Qp, const float* __restrict__ Xp,
                                                   const int* __restrict__ part_i, int64_t Nq, int KD, int k, int nc,
                                                   int cosine, int32_t* __restrict__ idx, float* __restrict__ dist) {
  extern __shared__ __align__(16) unsigned char merge_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* cd = reinterpret_cast<float*>(merge_raw) + (size_t)warp * 2 * nc;
  int* ci = reinterpret_cast<int*>(cd + nc);
  const int64_t q = (int64_t)blockIdx.x * 4 + warp;
  if (q >= Nq) return;
  const float4* qr = reinterpret_cast<const float4*>(Qp + (size_t)q * KD);
  for (int c = lane; c < nc; c += 32) {
    int j = part_i[(size_t)q * nc + c];
    float dd = KNN_INF;
    if (j >= 0) {
      const float4* xr = reinterpret_cast<const float4*>(Xp + (size_t)j * KD);
      float s = 0.f;
      for (int u = 0; u < KD / 4; ++u) {
        const float4 x = __ldg(xr + u), z = __ldg(qr + u);
        if (cosine) {
          s = fmaf(z.x, x.x, s);
          s = fmaf(z.y, x.y, s);
          s = fmaf(z.z, x.z, s);
          s = fmaf(z.w, x.w, s);
        } else {
          const float e0 = z.x - x.x, e1 = z.y - x.y, e2 = z.z - x.z, e3 = z.w - x.w;
          s = fmaf(e0, e0, s);
          s = fmaf(e1, e1, s);
          s = fmaf(e2, e2, s);
          s = fmaf(e3, e3, s);
        }
      }
      dd = cosine ? 1.f - s : sqrtf(s);
      if (!(dd < KNN_INF)) {
        dd = KNN_INF;
        j = -1;
      }
    }
    cd[c] = dd;
    ci[c] = j;
  }
  __syncwarp();
  for (int c = lane; c < nc; c += 32) {
    const float dd = cd[c];
    const int j = ci[c];
    int rank = 0;
    for (int o = 0; o < nc; ++o) {
      const float od = cd[o];
      const int oj = ci[o];
      rank += od < dd || (od == dd && (oj < j || (oj == j && o < c)));
    }
    if (rank < k) {
      idx[(size_t)q * k + rank] = j;
      if (dist) dist[(size_t)q * k + rank] = dd;
    }
  }
}

}  // namespace hb
