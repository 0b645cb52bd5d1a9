// lisi.cuh — the Local Inverse Simpson's Index of every row of an embedding (DESIGN §10), sm_90a.
//   k_lisi  one warp per row over the row's k <= 128 neighbours (hb_knn's sweep, knn.cuh): the fp64 bisection of the
//           neighbour weights P_j ~ exp(-beta D_j) to the perplexity's entropy, then for every label set the inverse
//           of the Simpson index sum_labels (sum of P_j over the neighbours with that label)^2.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int LISI_MAX_K = 128;              // the sweep's longest list (KNN_SWEEP_MAX_K)
constexpr int LISI_E = LISI_MAX_K / 32;      // distances per lane
constexpr int LISI_WARPS = 4;                // rows per CTA
constexpr int LISI_MAX_EVALS = 50;
constexpr double LISI_TOL = 1e-5;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// idx / dist [N][k]: each row's neighbours by ascending distance, idx = -1 (dist = +inf) past the last one found.
// labels [n_sets][labels_ld]: any int32 codes, only equality counts.  lisi [N][n_sets]: 1 / Simpson, -1 for a row whose
// final entropy is exactly 0, NaN for a row without neighbours.
__global__ void __launch_bounds__(32 * LISI_WARPS) k_lisi(const int32_t* __restrict__ idx, const float* __restrict__ dist,
                                                          int64_t N, int k, const int32_t* __restrict__ labels,
                                                          int64_t labels_ld, int n_sets, double log_p,
                                                          double* __restrict__ lisi) {
  __shared__ double Ps[LISI_WARPS][LISI_MAX_K];
  __shared__ int Ls[LISI_WARPS][LISI_MAX_K];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * LISI_WARPS + warp;
  if (i >= N) return;
  int j[LISI_E];
  double D[LISI_E];
  bool any = false;
#pragma unroll
  for (int u = 0; u < LISI_E; ++u) {
    const int e = lane + 32 * u;
    j[u] = e < k ? idx[i * k + e] : -1;
    D[u] = j[u] >= 0 ? (double)dist[i * k + e] : 0.0;
    any |= j[u] >= 0;
  }
  if (!__any_sync(0xffffffffu, any)) {
    for (int s = lane; s < n_sets; s += 32) lisi[i * n_sets + s] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  // H(beta) on distances shifted by the row's smallest (entry 0: the list ascends and starts with a neighbour): the
  // same function, and the sum of the weights is at least 1, so it neither underflows nor overflows
  const double d0 = __shfl_sync(0xffffffffu, D[0], 0);
#pragma unroll
  for (int u = 0; u < LISI_E; ++u) D[u] -= d0;
  double beta = 1.0, bmin = -HUGE_VAL, bmax = HUGE_VAL, H = 0.0, sum = 1.0;
  double P[LISI_E];
  for (int t = 0; t < LISI_MAX_EVALS; ++t) {
    double s = 0.0, sd = 0.0;
#pragma unroll
    for (int u = 0; u < LISI_E; ++u) {
      P[u] = j[u] >= 0 ? exp(-beta * D[u]) : 0.0;
      s += P[u];
      sd += D[u] * P[u];
    }
    s = warp_sum_f64(s);
    sd = warp_sum_f64(sd);
    H = log(s) + beta * sd / s;
    sum = s;
    const double diff = H - log_p;
    if (fabs(diff) < LISI_TOL) break;
    if (diff > 0) {
      bmin = beta;
      beta = bmax == HUGE_VAL ? 2.0 * beta : (beta + bmax) / 2;
    } else {
      bmax = beta;
      beta = bmin == -HUGE_VAL ? beta / 2 : (beta + bmin) / 2;
    }
  }
  if (H == 0.0) {
    for (int s = lane; s < n_sets; s += 32) lisi[i * n_sets + s] = -1.0;
    return;
  }
#pragma unroll
  for (int u = 0; u < LISI_E; ++u) {
    P[u] /= sum;
    if (lane + 32 * u < k) Ps[warp][lane + 32 * u] = P[u];
  }
  // Simpson = sum_e P_e * (sum of P_m over the entries m with e's label): 4 k compares per lane, no level count
  for (int set = 0; set < n_sets; ++set) {
    const int32_t* lab = labels + (int64_t)set * labels_ld;
    int l[LISI_E];
#pragma unroll
    for (int u = 0; u < LISI_E; ++u) {
      l[u] = j[u] >= 0 ? lab[j[u]] : 0;  // a missing neighbour has P = 0: its label adds nothing
      if (lane + 32 * u < k) Ls[warp][lane + 32 * u] = l[u];
    }
    __syncwarp();
    double acc[LISI_E] = {};
    for (int m = 0; m < k; ++m) {
      const double pm = Ps[warp][m];
      const int lm = Ls[warp][m];
#pragma unroll
      for (int u = 0; u < LISI_E; ++u) acc[u] += lm == l[u] ? pm : 0.0;
    }
    double S = 0.0;
#pragma unroll
    for (int u = 0; u < LISI_E; ++u) S += P[u] * acc[u];
    S = warp_sum_f64(S);
    if (lane == 0) lisi[i * n_sets + set] = 1.0 / S;
    __syncwarp();  // Ls is rewritten by the next set
  }
}

}  // namespace hb
