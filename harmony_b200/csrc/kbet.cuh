// kbet.cuh — kBET's per-cell test of the batch mix among a cell's nearest neighbours of its own cell type (DESIGN §13),
// sm_90a.  The neighbour lists come from k_knn_tc's grouped sweep over hb_silhouette's (label, batch) index and
// k_knn_merge (knn.cuh); everything here is per row.
//   chi2_sf  the chi-square upper tail Q(dof / 2, x / 2) in fp64, on the host (hb_debug_chi2_sf) and the device
//   k_kbet   one warp per sorted row: the batch counts among the row and its k0 - 1 nearest rows of its label, the
//            statistic sum_b (o_b - k0 p_b)^2 / (k0 p_b) and its p-value
#pragma once
#include "knn.cuh"
#include "lisi.cuh"

namespace hb {

constexpr int KBET_MAX_K0 = KNN_SWEEP_MAX_K + 1;  // the cell and the sweep's longest list
constexpr int KBET_E = (KBET_MAX_K0 + 31) / 32;   // neighbourhood entries per lane
constexpr int KBET_WARPS = 4;                     // rows per CTA

// The regularised upper incomplete gamma Q(a, y) at a = dof / 2, y = x / 2: 1 at x <= 0, 0 at x = +inf.  The prefactor
// y^a e^-y / Gamma(a) is taken in logs and applied last, so no intermediate term underflows; below y = a + 1 the series
// of P = 1 - Q (which is then at most 0.92, so 1 - P loses nothing), above it the continued fraction of Q by the
// modified Lentz method.  Both stop at a relative step below 2^-56.
__host__ __device__ inline double chi2_sf(double x, int dof) {
  if (x != x) return x;
  if (x <= 0.0) return 1.0;
  if (x > 1.7976931348623157e308) return 0.0;
  const double a = 0.5 * dof, y = 0.5 * x;
  const double lp = a * log(y) - lgamma(a) - y;
  if (y < a + 1.0) {
    double term = 1.0 / a, sum = term;
    for (int n = 1; n < 1000000 && term > sum * 1.4e-17; ++n) {
      term *= y / (a + n);
      sum += term;
    }
    return 1.0 - exp(lp) * sum;
  }
  const double tiny = 1e-300;
  double b = y + 1.0 - a, c = 1.0 / tiny, d = 1.0 / b, f = d;
  for (int n = 1; n < 1000000; ++n) {
    const double an = -n * (n - a);
    b += 2.0;
    d = an * d + b;
    if (fabs(d) < tiny) d = tiny;
    c = b + an / c;
    if (fabs(c) < tiny) c = tiny;
    d = 1.0 / d;
    const double step = d * c;
    f *= step;
    if (fabs(step - 1.0) < 1.4e-17) break;
  }
  return exp(lp) * f;
}

// What k_kbet needs of each (label, batch) pair: its label's k0 (0: the label is not tested), finite rows n_l,
// degrees of freedom B_l - 1 and pairs [p0, p1)
struct KbetPair {
  int k0, n, dof, p0, p1;
};

struct KbetArgs {
  const int* list;        // [N][kmax] each sorted row's nearest other rows of its label (sorted positions), -1: none
  const float* hx;        // [N] |x - c|^2 / 2 in sorted order; not finite: the row takes no part
  const int* pstart;      // [J + 1] first sorted row of each pair
  const int* count;       // [J] finite rows of each pair
  const KbetPair* pairs;  // [J]
  const int* sort_perm;   // sorted row -> caller's row
  double* stat;           // [N] in the caller's order
  double* pval;
  int32_t* idx;           // [N][idx_ld] in the caller's order and numbering, or null
  int64_t N, idx_ld;
  int J, kmax;
};

// the last pair of [lo, hi) starting at or before sorted row i
__device__ __forceinline__ int kbet_pair_of(const int* __restrict__ pstart, int lo, int hi, int i) {
  --hi;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(pstart + mid) <= i)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// One warp per sorted row.  With o_b the batch counts over the k0 cells and e_b = k0 n_{l,b} / n_l, the statistic is
// the sum over the batches present of (o_b - e_b)^2 / e_b plus the absent ones' e_b, k0 (n_l - their n_{l,b}) / n_l:
// every term is positive, so nothing cancels.  A batch's term is added by its first entry (no earlier entry of the
// same pair): all-pairs compares of at most KBET_MAX_K0 pair ids in shared memory, no per-batch array.
__global__ void __launch_bounds__(32 * KBET_WARPS) k_kbet(KbetArgs a) {
  __shared__ int Ls[KBET_WARPS][32 * KBET_E];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * KBET_WARPS + warp;
  if (i >= a.N) return;
  const KbetPair t = a.pairs[kbet_pair_of(a.pstart, 0, a.J, (int)i)];
  const int k0 = t.k0, m = k0 - 1;
  const int* row = a.list + i * a.kmax;
  bool ok = k0 > 0 && a.hx[i] < KNN_INF;  // warp-uniform
  int q[KBET_E];
  if (ok) {
    bool full = true;
#pragma unroll
    for (int u = 0; u < KBET_E; ++u) {
      const int e = lane + 32 * u;
      q[u] = -1;
      if (e < k0) {
        const int j = e < m ? row[e] : (int)i;
        full &= j >= 0;  // a list falls short only where fp32 distances overflow
        q[u] = j >= 0 ? kbet_pair_of(a.pstart, t.p0, t.p1, j) : -1;
        Ls[warp][e] = q[u];
      }
    }
    ok = __all_sync(0xffffffffu, full);
    __syncwarp();
  }
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  double st = nan, pv = nan;
  if (ok) {
    double sum = 0.0;
    int present = 0;
#pragma unroll
    for (int u = 0; u < KBET_E; ++u) {
      const int e = lane + 32 * u;
      if (e < k0) {
        int o = 0;
        bool first = true;
        for (int r = 0; r < k0; ++r) {
          const bool same = Ls[warp][r] == q[u];
          o += same;
          first &= !(same && r < e);
        }
        if (first) {
          const int c = __ldg(a.count + q[u]);
          const double eb = (double)k0 * c / t.n, dv = o - eb;
          sum += dv * dv / eb;
          present += c;
        }
      }
    }
    sum = warp_sum_f64(sum);
    present = __reduce_add_sync(0xffffffffu, present);
    st = sum + (double)k0 * (t.n - present) / t.n;
    pv = chi2_sf(st, t.dof);
  }
  const int64_t ci = a.sort_perm[i];
  if (lane == 0) {
    a.stat[ci] = st;
    a.pval[ci] = pv;
  }
  if (a.idx)
    for (int64_t e = lane; e < a.idx_ld; e += 32) a.idx[ci * a.idx_ld + e] = ok && e < m ? a.sort_perm[row[e]] : -1;
}

}  // namespace hb
