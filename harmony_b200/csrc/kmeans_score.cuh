// kmeans_score.cuh — k-means of an embedding for the NMI / ARI scores (DESIGN §15), sm_90a.  Greedy k-means++ seeding
// on the prepared rows of knn.cuh (fp32, centred on the column mean of the finite rows) with fp64 distances, and
// sklearn's Lloyd iteration around the §9 sweep (assignment), setup's tuple index and hb_pcr's segment sums (means).
// Every sum has a fixed order given the SM count and no float atomics run, so two calls give bit-identical results.
//   k_kms_colsum   one CTA per contiguous range of rows, a warp per row: each CTA's fp64 column sums and finite rows
//                  (k_pcr_mean folds them in CTA order into the mean), and each row's finite flag
//   k_kms_sqdist   the same ranges: each CTA's fp64 sum of |x - c|^2 over finite rows, with c the mean (the total
//                  variance behind the tolerance, and the check that every finite row fits the fp32 assignment) or the
//                  row's centre (the inertia)
//   k_kms_update   8 lanes per prepared row: D^2 <- min(D^2, |p - p_winner|^2), then the next round's races, two per
//                  trial (weight D^2, weight 1), one 64-bit atomicMin per race and CTA
//   k_kms_potential  8 lanes per prepared row: the round's candidates' potentials sum min(D^2, |p - p_cand|^2), one
//                  fp64 partial per CTA and candidate
//   k_kms_pick     one warp: the partials in CTA order, the candidate of the smallest potential (lowest trial on a
//                  tie), the round's seed; resets the race keys the next round's update fills
//   k_kms_gather   the seeds' caller rows -> fp64 centres
//   k_kms_labels   the merge's nearest centre -> the row's label (-1 for a non-finite row), its sort code (K for -1)
//                  and the count of labels that changed
//   k_kms_means    one warp per present label: its segment sums (k_pcr_sums' pieces) -> the fp64 mean and the count
#pragma once
#include <math_constants.h>

#include "common.cuh"
#include "knn.cuh"
#include "pcr.cuh"

namespace hb {

constexpr int KMS_MAX_K = 1024;   // the seeding makes about K passes over the rows
constexpr int KMS_MAX_T = 8;      // candidates per round: 2 + floor(ln K) <= 8 for K <= 1024
constexpr int KMS_WARPS = 8;      // warps per CTA of every kernel here
constexpr unsigned long long KMS_NO_KEY = ~0ull;
// the largest |x - m|^2 of a finite row: the assignment scores fp32 rows centred on m, whose squared distances
// (<= 4 |x - m|^2) and halved norms must stay below FLT_MAX ~ 2^128
constexpr double KMS_MAX_SQ = 0x1p124;
constexpr uint64_t KMS_SEED_TAG = 0x6b6d2b2b73636f72ull;  // "km++scor": the seeding's draws, apart from kmeans_centers'

// The uniform of (round, trial, row) under the init's key kmeans_score_key(seed, init)
__host__ __device__ __forceinline__ uint64_t kmeans_score_key(uint64_t seed, uint64_t init) {
  return hb_mix64(seed ^ KMS_SEED_TAG ^ hb_mix64(init));
}
__device__ __forceinline__ float kms_uniform(uint64_t key, int round, int trial, int64_t row) {
  return kmeans_uniform(key, (uint64_t)round * KMS_MAX_T + (uint64_t)trial, (uint64_t)row);
}
// the packed race key of a row: fp32 bits of -ln(u) / w (non-negative, so they order like the values), then the row
__device__ __forceinline__ unsigned long long kms_race_key(double e, double w, int64_t row) {
  return ((unsigned long long)__float_as_uint(__double2float_rn(e / w)) << 32) | (unsigned long long)row;
}

// ---- the statistics of the caller's rows ----------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(32 * KMS_WARPS) k_kms_colsum(const T* __restrict__ X, int64_t ld, int64_t N, int d,
                                                               int64_t rows_per_cta, double* __restrict__ part,
                                                               int* __restrict__ part_n, unsigned char* __restrict__ fin) {
  __shared__ double ss[KMS_WARPS][KNN_MAX_D];
  __shared__ int sn[KMS_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r0 = blockIdx.x * rows_per_cta, r1 = min(r0 + rows_per_cta, N);
  double s[4] = {0, 0, 0, 0};
  int n = 0;
  for (int64_t r = r0 + warp; r < r1; r += KMS_WARPS) {
    double v[4];
    bool ok = true;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = lane + 32 * u;
      v[u] = c < d ? (double)X[r * ld + c] : 0.0;
      ok &= isfinite(v[u]);
    }
    ok = __all_sync(0xffffffffu, ok);
    if (lane == 0) fin[r] = ok;
    if (ok) {
#pragma unroll
      for (int u = 0; u < 4; ++u) s[u] += v[u];
      ++n;
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) ss[warp][lane + 32 * u] = s[u];
  if (lane == 0) sn[warp] = n;
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    double t = 0.0;
    for (int w = 0; w < KMS_WARPS; ++w) t += ss[w][c];
    part[blockIdx.x * (int64_t)d + c] = t;
  }
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < KMS_WARPS; ++w) t += sn[w];
    part_n[blockIdx.x] = t;
  }
}

// fp64 sum of a value held by every lane of a warp; the butterfly leaves the same bits in every lane
__device__ __forceinline__ double kms_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// part[cta] = sum over the finite rows of the CTA's range of |x - c|^2, c = centres[labels[r]] (labels: a row with
// label < 0 is left out) or centres[0] (labels null).  far (null: not checked): set to 1 when a row's |x - c|^2
// exceeds KMS_MAX_SQ
template <typename T>
__global__ void __launch_bounds__(32 * KMS_WARPS) k_kms_sqdist(const T* __restrict__ X, int64_t ld, int64_t N, int d,
                                                               int64_t rows_per_cta, const unsigned char* __restrict__ fin,
                                                               const int32_t* __restrict__ labels,
                                                               const double* __restrict__ centres, double* __restrict__ part,
                                                               int* __restrict__ far) {
  __shared__ double sw[KMS_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r0 = blockIdx.x * rows_per_cta, r1 = min(r0 + rows_per_cta, N);
  double s = 0.0;
  for (int64_t r = r0 + warp; r < r1; r += KMS_WARPS) {
    const int l = labels ? labels[r] : 0;
    if (!fin[r] || l < 0) continue;  // warp-uniform
    const double* c = centres + (int64_t)l * d;
    double q = 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int col = lane + 32 * u;
      if (col < d) {
        const double e = (double)X[r * ld + col] - __ldg(c + col);
        q = fma(e, e, q);
      }
    }
    s += q;
    if (far && kms_warp_sum(q) > KMS_MAX_SQ && lane == 0) atomicOr(far, 1);
  }
  s = kms_warp_sum(s);
  if (lane == 0) sw[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < KMS_WARPS; ++w) t += sw[w];
    part[blockIdx.x] = t;
  }
}

// ---- seeding --------------------------------------------------------------------------------------------------------
// Eight lanes per prepared row, four rows per warp: lane g of a group holds columns g + 8 u, so a load of the warp
// reads four rows' 32-byte sectors whole, and a distance is three butterfly steps.  Lane g runs trial g's races and
// sums trial g's potential.  The grid is fixed by N and the SM count.
constexpr int KMS_GROUP = 8;                                 // lanes per row (>= KMS_MAX_T)
constexpr int KMS_PER_LANE = KNN_MAX_D / KMS_GROUP;           // columns per lane
constexpr int KMS_ROWS_PER_WARP = 32 / KMS_GROUP;

// |p - q|^2 in fp64 of a row held by a group (p: the lane's columns) and a row q in shared memory, in every lane of
// the group; the butterfly leaves the same bits in each
__device__ __forceinline__ double kms_dist2(const float (&p)[KMS_PER_LANE], const float* q, int KD, int g) {
  double s = 0.0;
#pragma unroll
  for (int u = 0; u < KMS_PER_LANE; ++u) {
    const int col = g + KMS_GROUP * u;
    if (col < KD) {
      const double e = (double)p[u] - (double)q[col];
      s = fma(e, e, s);
    }
  }
#pragma unroll
  for (int o = KMS_GROUP / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}
__device__ __forceinline__ void kms_load_row(const float* __restrict__ P, int64_t r, bool ok, int KD, int g,
                                             float (&p)[KMS_PER_LANE]) {
#pragma unroll
  for (int u = 0; u < KMS_PER_LANE; ++u) {
    const int col = g + KMS_GROUP * u;
    p[u] = ok && col < KD ? __ldg(P + r * KD + col) : 0.f;
  }
}

// keys [2][T]: trial t's race with weight D^2 (KMS_NO_KEY when no row has D^2 > 0) and with weight 1
struct KmsSeedArgs {
  const float* P;        // [N][KD] prepared rows
  const unsigned char* fin;
  double* D2;            // [N] squared distance to the nearest chosen centre; -1 for a non-finite row
  int64_t N;
  int KD, T;
  uint64_t key;          // kmeans_score_key of the init
};

// winner null: D^2 = +inf for every finite row (before the first centre).  Then the races of `round`.
__global__ void __launch_bounds__(32 * KMS_WARPS) k_kms_update(KmsSeedArgs a, const int* __restrict__ winner, int round,
                                                               unsigned long long* __restrict__ keys) {
  __shared__ float cs[KNN_MAX_D];
  __shared__ unsigned long long sk[KMS_WARPS][2 * KMS_MAX_T];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane % KMS_GROUP, grp = lane / KMS_GROUP;
  if (winner)
    for (int c = threadIdx.x; c < a.KD; c += blockDim.x) cs[c] = a.P[(int64_t)*winner * a.KD + c];
  __syncthreads();
  unsigned long long best_w = KMS_NO_KEY, best_1 = KMS_NO_KEY;  // lane g's trial
  const int64_t step = (((int64_t)gridDim.x * blockDim.x) >> 5) * KMS_ROWS_PER_WARP;
  for (int64_t base = ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5) * KMS_ROWS_PER_WARP; base < a.N;
       base += step) {  // warp-uniform: every lane reaches the shuffles
    const int64_t r = base + grp;
    const bool in = r < a.N, ok = in && a.fin[r];
    if (in && !ok && !winner && g == 0) a.D2[r] = -1.0;
    double w = CUDART_INF;
    if (winner) {
      const double old = ok ? a.D2[r] : 0.0;  // read by the group before its lane 0 stores
      float p[KMS_PER_LANE];
      kms_load_row(a.P, r, ok, a.KD, g, p);
      w = fmin(old, kms_dist2(p, cs, a.KD, g));
    }
    if (!ok) continue;
    if (g == 0) a.D2[r] = w;
    if (g < a.T) {
      const double e = -log((double)kms_uniform(a.key, round, g, r));
      if (w > 0.0 && w < CUDART_INF) best_w = min(best_w, kms_race_key(e, w, r));
      best_1 = min(best_1, kms_race_key(e, 1.0, r));
    }
  }
#pragma unroll
  for (int o = KMS_GROUP; o < 32; o <<= 1) {
    best_w = min(best_w, __shfl_xor_sync(0xffffffffu, best_w, o));
    best_1 = min(best_1, __shfl_xor_sync(0xffffffffu, best_1, o));
  }
  if (lane < KMS_MAX_T) {
    sk[warp][lane] = best_w;
    sk[warp][KMS_MAX_T + lane] = best_1;
  }
  __syncthreads();
  if (threadIdx.x < 2 * KMS_MAX_T && threadIdx.x % KMS_MAX_T < a.T) {
    unsigned long long m = KMS_NO_KEY;
    for (int w = 0; w < KMS_WARPS; ++w) m = min(m, sk[w][threadIdx.x]);
    const int t = threadIdx.x % KMS_MAX_T, weight1 = threadIdx.x / KMS_MAX_T;
    if (m != KMS_NO_KEY) atomicMin(keys + weight1 * a.T + t, m);
  }
}

// trial t's candidate: its D^2 race's winner, or its weight-1 race's when no row has D^2 > 0
__device__ __forceinline__ int kms_candidate(const unsigned long long* keys, int T, int t) {
  const unsigned long long k = keys[t] != KMS_NO_KEY ? keys[t] : keys[T + t];
  return (int)(k & 0xffffffffull);
}

__global__ void __launch_bounds__(32 * KMS_WARPS) k_kms_potential(KmsSeedArgs a, const unsigned long long* __restrict__ keys,
                                                                  double* __restrict__ part) {
  __shared__ float cs[KMS_MAX_T][KNN_MAX_D];
  __shared__ double sp[KMS_WARPS][KMS_MAX_T];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane % KMS_GROUP, grp = lane / KMS_GROUP;
  for (int e = threadIdx.x; e < a.T * a.KD; e += blockDim.x) {
    const int t = e / a.KD, c = e % a.KD;
    cs[t][c] = a.P[(int64_t)kms_candidate(keys, a.T, t) * a.KD + c];
  }
  __syncthreads();
  double acc = 0.0;  // lane g's trial, over its group's rows
  const int64_t step = (((int64_t)gridDim.x * blockDim.x) >> 5) * KMS_ROWS_PER_WARP;
  for (int64_t base = ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5) * KMS_ROWS_PER_WARP; base < a.N;
       base += step) {  // warp-uniform
    const int64_t r = base + grp;
    const double w = r < a.N ? a.D2[r] : -1.0;
    const bool ok = w >= 0.0;
    float p[KMS_PER_LANE];
    kms_load_row(a.P, r, ok, a.KD, g, p);
#pragma unroll 1
    for (int t = 0; t < a.T; ++t) {
      const double d2 = kms_dist2(p, cs[t], a.KD, g);
      if (ok && g == t) acc += fmin(w, d2);
    }
  }
#pragma unroll
  for (int o = KMS_GROUP; o < 32; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane < KMS_MAX_T) sp[warp][lane] = acc;
  __syncthreads();
  if (threadIdx.x < a.T) {
    double s = 0.0;
    for (int w = 0; w < KMS_WARPS; ++w) s += sp[w][threadIdx.x];
    part[(int64_t)blockIdx.x * a.T + threadIdx.x] = s;
  }
}

// One warp.  round 0: the weight-1 race of trial 0 wins; later rounds: the candidate of the smallest potential.  The
// winner goes to seeds[round] and *winner; the T races of `reset` (the next round's) are cleared for k_kms_update.
__global__ void __launch_bounds__(32) k_kms_pick(const double* __restrict__ part, int ctas, int T,
                                                 const unsigned long long* __restrict__ keys, int round,
                                                 int32_t* __restrict__ seeds, int* __restrict__ winner,
                                                 unsigned long long* __restrict__ reset) {
  __shared__ double pot[KMS_MAX_T];
  const int lane = threadIdx.x;
  if (round > 0 && lane < T) {
    double s = 0.0;
    for (int c = 0; c < ctas; ++c) s += part[(int64_t)c * T + lane];
    pot[lane] = s;
  }
  __syncwarp();
  if (lane == 0) {
    int w;
    if (round == 0) {
      w = (int)(keys[T] & 0xffffffffull);
    } else {
      int bt = 0;
      for (int t = 1; t < T; ++t)
        if (pot[t] < pot[bt]) bt = t;
      w = kms_candidate(keys, T, bt);
    }
    seeds[round] = w;
    *winner = w;
  }
  if (lane < 2 * T) reset[lane] = KMS_NO_KEY;
}

// centres[k][.] = the caller's row seeds[k] in fp64
template <typename T>
__global__ void k_kms_gather(const T* __restrict__ X, int64_t ld, int d, const int32_t* __restrict__ seeds, int K,
                             double* __restrict__ centres) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < K * d; e += gridDim.x * blockDim.x)
    centres[e] = (double)X[(int64_t)seeds[e / d] * ld + e % d];
}

// ---- Lloyd ----------------------------------------------------------------------------------------------------------
// labels[i] (the merge's nearest centre) -> -1 for a non-finite row; code[i] = the label, K for -1; *changed += the
// rows whose label differs from old[i]
__global__ void __launch_bounds__(32 * KMS_WARPS) k_kms_labels(int32_t* __restrict__ labels, const int32_t* __restrict__ old,
                                                               const unsigned char* __restrict__ fin, int64_t N, int K,
                                                               int* __restrict__ code, int* __restrict__ changed) {
  __shared__ int sc[KMS_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int n = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x; base < N; base += stride) {  // whole warps stay in the loop
    const int64_t i = base + threadIdx.x;
    bool diff = false;
    if (i < N) {
      const int l = fin[i] ? labels[i] : -1;
      labels[i] = l;
      code[i] = l < 0 ? K : l;
      diff = l != old[i];
    }
    n += __popc(__ballot_sync(0xffffffffu, diff));
  }
  if (lane == 0) sc[warp] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < KMS_WARPS; ++w) t += sc[w];
    if (t) atomicAdd(changed, t);
  }
}

// One warp per tuple q of the sort by code (uniq[q] its code): a code below K gets the mean of its finite rows, or
// keeps its centre when it has none, and its count
__global__ void __launch_bounds__(32 * PCR_WARPS) k_kms_means(PcrSumArgs a, const unsigned long long* __restrict__ uniq,
                                                              int K, double* __restrict__ centres, int* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * PCR_WARPS + (threadIdx.x >> 5);
  if (q >= a.J || uniq[q] >= (unsigned long long)K) return;
  double s[4];
  const int n = pcr_batch_sum(a, q, lane, s);
  const int64_t k = (int64_t)uniq[q];
  if (lane == 0) counts[k] = n;
  if (n == 0) return;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int col = lane + 32 * u;
    if (col < a.d) centres[k * a.d + col] = s[u] / n;
  }
}

}  // namespace hb
