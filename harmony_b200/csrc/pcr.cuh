// pcr.cuh — principal component regression of an embedding on its batches (DESIGN §14), sm_90a.  The rows are
// sorted by batch with setup's covariate-tuple index (tuples.cuh); everything here is fp64 and free of atomics, so two
// calls give bit-identical results.
//   k_pcr_sums     one warp per chunk of PCR_CHUNK sorted rows: the column sums and finite rows of each batch piece in
//                  the chunk (a batch inside the chunk is final; a batch that crosses a chunk edge leaves a head or
//                  tail piece), and the chunk's total
//   k_pcr_mean     one CTA per column: the chunk totals summed in a fixed tree -> the column mean m over finite rows
//   k_pcr_combine  one warp per batch: its pieces in chunk order -> S_b = sum (x - m) and n_b, written in place as the
//                  row T_b = S_b / sqrt(n_b), whose Gram is the between-batch scatter sum_b S_b S_b^T / n_b
//   k_pcr_gram     the Gram Y^T Y of centred rows on the fp64 tensor cores (mma m16n8k16 f64): each CTA a fixed
//                  contiguous range of rows in natural order, staged in shared memory as fp64 x - m (zero for a row
//                  with a non-finite value and for padding), the upper-triangle 16 x 8 tiles of the KD x KD result
//                  dealt to 8 warps, one partial per CTA
//   k_pcr_reduce   the partials summed in CTA order
#pragma once
#include "common.cuh"

namespace hb {

constexpr int PCR_CHUNK = 256;   // sorted rows per warp of k_pcr_sums
constexpr int PCR_WARPS = 4;     // warps per CTA of k_pcr_sums and k_pcr_combine
constexpr int PCR_GR = 64;       // rows per shared-memory stage of k_pcr_gram (4 k-steps of 16)
constexpr int PCR_GW = 8;        // warps of k_pcr_gram

struct PcrSumArgs {
  int64_t ld, N;
  int d, J;
  int64_t chunks;
  const int* sort_perm;  // sorted row -> caller's row
  const int* pstart;     // [J + 1] first sorted row of each batch
  double* sums;          // [J][d] raw column sums of the batches that lie inside one chunk
  int* count;            // [J] their finite rows
  double* edge;          // [3][chunks][d] head, tail and total piece of each chunk
  int* edge_n;           // [3][chunks] their finite rows
};

__device__ __forceinline__ int pcr_batch_of(const int* __restrict__ pstart, int J, int64_t p) {
  int lo = 0, hi = J - 1;  // the last batch starting at or before p
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(pstart + mid) <= p)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

template <typename T>
__global__ void __launch_bounds__(32 * PCR_WARPS) k_pcr_sums(PcrSumArgs a, const T* __restrict__ X) {
  const int lane = threadIdx.x & 31;
  const int64_t c = (int64_t)blockIdx.x * PCR_WARPS + (threadIdx.x >> 5);
  if (c >= a.chunks) return;
  const int64_t p0 = c * PCR_CHUNK, p1 = min(p0 + PCR_CHUNK, a.N);
  int q = pcr_batch_of(a.pstart, a.J, p0);
  int64_t qs = __ldg(a.pstart + q), qe = __ldg(a.pstart + q + 1);
  double s[4] = {0, 0, 0, 0}, t[4] = {0, 0, 0, 0};
  int n = 0, tn = 0;
  // the piece of batch q just ended at `end`: head (the batch began before the chunk), tail (it goes on after the
  // chunk) or the whole batch
  auto flush = [&](int64_t end) {
    double* dst;
    int* dn;
    if (qs < p0) {
      dst = a.edge + c * a.d, dn = a.edge_n + c;
    } else if (qe > end) {
      dst = a.edge + (a.chunks + c) * a.d, dn = a.edge_n + a.chunks + c;
    } else {
      dst = a.sums + (int64_t)q * a.d, dn = a.count + q;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int col = lane + 32 * u;
      if (col < a.d) dst[col] = s[u];
      t[u] += s[u];
      s[u] = 0.0;
    }
    if (lane == 0) *dn = n;
    tn += n;
    n = 0;
  };
  for (int64_t base = p0; base < p1; base += 32) {
    const int rows = (int)min((int64_t)32, p1 - base);
    const int mine = lane < rows ? __ldg(a.sort_perm + base + lane) : 0;
    for (int j0 = 0; j0 < rows; j0 += 8) {
      T v[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t r = __shfl_sync(0xffffffffu, mine, (j0 + j) & 31);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int col = lane + 32 * u;
          v[j][u] = j0 + j < rows && col < a.d ? X[r * a.ld + col] : T(0);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (j0 + j >= rows) break;
        const int64_t p = base + j0 + j;
        if (p == qe) {  // batches are never empty: one step reaches the next
          flush(p);
          ++q;
          qs = qe;
          qe = __ldg(a.pstart + q + 1);
        }
        bool fin = true;
#pragma unroll
        for (int u = 0; u < 4; ++u) fin &= isfinite((double)v[j][u]);
        if (__all_sync(0xffffffffu, fin)) {
#pragma unroll
          for (int u = 0; u < 4; ++u) s[u] += (double)v[j][u];
          ++n;
        }
      }
    }
  }
  flush(p1);
  double* tot = a.edge + (2 * a.chunks + c) * a.d;
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (lane + 32 * u < a.d) tot[lane + 32 * u] = t[u];
  if (lane == 0) a.edge_n[2 * a.chunks + c] = tn;
}

// CTA `col` (of d): the column's chunk totals and the finite rows in a fixed tree -> centre[col] = sum / n (0 when no
// row is finite); CTA 0 also writes n to *n_out
__global__ void __launch_bounds__(256) k_pcr_mean(const double* __restrict__ total, const int* __restrict__ total_n,
                                                  int64_t chunks, int d, double* __restrict__ centre,
                                                  double* __restrict__ n_out) {
  __shared__ double ss[256], sn[256];
  const int col = blockIdx.x, tid = threadIdx.x;
  double s = 0.0, n = 0.0;
  for (int64_t c = tid; c < chunks; c += 256) {
    s += total[c * d + col];
    n += (double)total_n[c];
  }
  ss[tid] = s;
  sn[tid] = n;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w) {
      ss[tid] += ss[tid + w];
      sn[tid] += sn[tid + w];
    }
    __syncthreads();
  }
  if (tid == 0) {
    centre[col] = sn[0] > 0 ? ss[0] / sn[0] : 0.0;
    if (col == 0) *n_out = sn[0];
  }
}

// Batch q's raw column sums into s (lane's columns lane + 32 u) and its finite rows, returned: the batch's own sums,
// or for a batch that crossed chunk edges the tail of its first chunk, then the heads of the following ones (the
// count is then also written to a.count[q])
__device__ __forceinline__ int pcr_batch_sum(const PcrSumArgs& a, int64_t q, int lane, double (&s)[4]) {
  const int64_t s0 = a.pstart[q], s1 = a.pstart[q + 1];
  const int64_t c0 = s0 / PCR_CHUNK, c1 = (s1 - 1) / PCR_CHUNK;
  const double* row = a.sums + q * a.d;
  int n;
  if (c0 == c1) {
#pragma unroll
    for (int u = 0; u < 4; ++u) s[u] = lane + 32 * u < a.d ? row[lane + 32 * u] : 0.0;
    n = a.count[q];
  } else {
    const double* tail = a.edge + (a.chunks + c0) * a.d;
#pragma unroll
    for (int u = 0; u < 4; ++u) s[u] = lane + 32 * u < a.d ? tail[lane + 32 * u] : 0.0;
    n = a.edge_n[a.chunks + c0];
    for (int64_t c = c0 + 1; c <= c1; ++c) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (lane + 32 * u < a.d) s[u] += a.edge[c * a.d + lane + 32 * u];
      n += a.edge_n[c];
    }
    if (lane == 0) a.count[q] = n;
  }
  return n;
}

// One warp per batch q: its raw sums -> T_q = (sums - n_q m) / sqrt(n_q), 0 for a batch without finite rows, in place
__global__ void __launch_bounds__(32 * PCR_WARPS) k_pcr_combine(PcrSumArgs a, const double* __restrict__ centre) {
  const int lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * PCR_WARPS + (threadIdx.x >> 5);
  if (q >= a.J) return;
  double* row = a.sums + q * a.d;
  double s[4];
  const int n = pcr_batch_sum(a, q, lane, s);
  const double r = n > 0 ? 1.0 / sqrt((double)n) : 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int col = lane + 32 * u;
    if (col < a.d) row[col] = n > 0 ? (s[u] - n * centre[col]) * r : 0.0;
  }
}

struct PcrGramArgs {
  int64_t ld, n, rows_per_cta;
  int d;
  const double* centre;  // [d] subtracted from every row, or null
  double* part;          // [gridDim.x][KD][KD], upper-triangle 16 x 8 tiles written
};

// D += A B on one 16 x 8 x 16 fp64 tile: a[v] = A(g + 8 (v & 1), t + 4 (v >> 1)), b[v] = B(t + 4 v, g),
// c[v] = D(g + 8 (v >> 1), 2 t + (v & 1)), with g = lane / 4 and t = lane % 4
__device__ __forceinline__ void mma_f64_16x8x16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
      "{%12, %13, %14, %15}, {%0, %1, %2, %3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// the upper-triangle tiles of a KD x KD Gram: row strip mi of 16 columns, column blocks nj >= 2 mi of 8
__host__ __device__ constexpr int pcr_tiles(int KD) { return (KD / 16) * (KD / 16) + KD / 16; }
constexpr size_t pcr_gram_smem(int KD) { return (size_t)PCR_GR * (KD + 4) * sizeof(double); }

template <typename T, int KD>
__global__ void __launch_bounds__(32 * PCR_GW, 2) k_pcr_gram(PcrGramArgs a, const T* __restrict__ X) {
  constexpr int NB = KD / 8, U = pcr_tiles(KD), PER = (U + PCR_GW - 1) / PCR_GW;
  constexpr int LD = KD + 4;   // a row stride of 8 words mod 32: a half-warp's fragment loads hit 16 distinct banks
  constexpr int CU = (KD + 31) / 32;
  constexpr int LG = KD > 96 ? 2 : 4;  // rows a lane loads at once: what the accumulators leave of 128 registers
  extern __shared__ double ys[];  // [PCR_GR][LD]
  __shared__ double cs[KD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  __shared__ int tile[PCR_GW * PER];  // strip mi << 8 | block nj of tile b (warp b / PER), -1: none; in shared
                                      // memory, so that the accumulators keep the registers
  for (int b = threadIdx.x; b < PCR_GW * PER; b += blockDim.x) {
    int r = b, m = 0;
    if (r < U) {
      while (r >= NB - 2 * m) r -= NB - 2 * m++;
      tile[b] = m << 8 | (2 * m + r);
    } else {
      tile[b] = -1;
    }
  }
  double acc[PER][4];
#pragma unroll
  for (int s = 0; s < PER; ++s) acc[s][0] = acc[s][1] = acc[s][2] = acc[s][3] = 0.0;
  for (int col = threadIdx.x; col < KD; col += blockDim.x) cs[col] = a.centre && col < a.d ? a.centre[col] : 0.0;
  __syncthreads();
  const int64_t r0 = blockIdx.x * a.rows_per_cta, r1 = min(r0 + a.rows_per_cta, a.n);
  for (int64_t base = r0; base < r1; base += PCR_GR) {
    // ---- stage: warp w takes rows w, w + 8, ..., LG at a time
#pragma unroll
    for (int i0 = 0; i0 < PCR_GR / PCR_GW; i0 += LG) {
      T v[LG][CU];
#pragma unroll
      for (int i = 0; i < LG; ++i) {
        const int64_t r = base + warp + PCR_GW * (i0 + i);
#pragma unroll
        for (int u = 0; u < CU; ++u) {
          const int col = lane + 32 * u;
          v[i][u] = r < r1 && col < a.d ? X[r * a.ld + col] : T(0);
        }
      }
#pragma unroll
      for (int i = 0; i < LG; ++i) {
        const int64_t r = base + warp + PCR_GW * (i0 + i);
        bool fin = true;
#pragma unroll
        for (int u = 0; u < CU; ++u) fin &= isfinite((double)v[i][u]);
        const bool keep = __all_sync(0xffffffffu, fin) && r < r1;
        double* y = ys + (warp + PCR_GW * (i0 + i)) * LD;
#pragma unroll
        for (int u = 0; u < CU; ++u) {
          const int col = lane + 32 * u;
          if (col < KD) y[col] = keep && col < a.d ? (double)v[i][u] - cs[col] : 0.0;
        }
      }
    }
    __syncthreads();
    // ---- the tiles: A = Y^T (strip mi), B = Y (block nj), k = the stage's rows
#pragma unroll 1
    for (int k0 = 0; k0 < PCR_GR; k0 += 16) {
      int cur = -1;
      double af[8];
#pragma unroll
      for (int s = 0; s < PER; ++s) {
        const int ts = tile[warp * PER + s];
        if (ts < 0) continue;
        if (ts >> 8 != cur) {
          cur = ts >> 8;
#pragma unroll
          for (int v = 0; v < 8; ++v) af[v] = ys[(k0 + t + 4 * (v >> 1)) * LD + 16 * cur + g + 8 * (v & 1)];
        }
        double bf[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) bf[v] = ys[(k0 + t + 4 * v) * LD + 8 * (ts & 255) + g];
        mma_f64_16x8x16(acc[s], af, bf);
      }
    }
    __syncthreads();
  }
  double* out = a.part + (int64_t)blockIdx.x * KD * KD;
#pragma unroll
  for (int s = 0; s < PER; ++s) {
    const int ts = tile[warp * PER + s];
    if (ts < 0) continue;
    const int mi = ts >> 8, nj = ts & 255;
#pragma unroll
    for (int v = 0; v < 4; ++v) out[(16 * mi + g + 8 * (v >> 1)) * KD + 8 * nj + 2 * t + (v & 1)] = acc[s][v];
  }
}

// out[e] = sum over the parts in order of part[p][e], for the elements e of the upper-triangle tiles (others: 0)
__global__ void __launch_bounds__(256) k_pcr_reduce(const double* __restrict__ part, int parts, int KD,
                                                    double* __restrict__ out) {
  const int64_t KK = (int64_t)KD * KD;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < KK; e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / KD), c = (int)(e % KD);
    double s = 0.0;
    if (c / 8 >= 2 * (r / 16))
      for (int p = 0; p < parts; ++p) s += part[p * KK + e];
    out[e] = s;
  }
}

}  // namespace hb
