// silhouette.cuh — the silhouette width of every row of an embedding (DESIGN §11), sm_90a.
//   k_silhouette_phi    labels / groups -> the (group, label) levels build_tuple_index (tuples.cuh) sorts the rows by,
//                       group most significant; a code out of range becomes a level of no covariate
//   k_silhouette_count  finite rows of each (group, label) pair: rows in sorted order whose prepared hx is finite
//   k_silhouette_tc     one CTA per tile of <= TQ sorted rows of one group.  The group's rows stream past the tile once
//                       through k_knn_tc's operand pipeline (Q hi / lo resident, cp.async stages of KNN_TN rows, 3xTF32
//                       m64n64k8); the epilogue turns each score into a distance and folds the distances into per-pair
//                       sums: a tile's columns fall into a few runs of one pair, each run is summed in fp32 per quad
//                       (a row's 64 columns lie in one quad, umma::frag_col) and added to the row's fp64 sum, and a run
//                       that closes a pair sets the row's a (its own pair) or lowers its b (any other).
#pragma once
#include "knn.cuh"

namespace hb {

// phi [n][2]: (group, n_groups + label), or -1 (no covariate's level) for a code outside 0..n_groups-1 / 0..n_labels-1
__global__ void k_silhouette_phi(const int32_t* __restrict__ labels, const int32_t* __restrict__ groups, int64_t n,
                                 int n_labels, int n_groups, int* __restrict__ phi) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = groups ? groups[i] : 0, l = labels[i];
    phi[2 * i] = g >= 0 && g < n_groups ? g : -1;
    phi[2 * i + 1] = l >= 0 && l < n_labels ? n_groups + l : -1;
  }
}

// count[p] += finite rows of pair p (pstart [J + 1] ascending); a warp adds once per pair it sees
__global__ void k_silhouette_count(const float* __restrict__ hx, int64_t n, const int* __restrict__ pstart, int J,
                                   int* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const int64_t s = base + lane;
    const bool act = s < n;
    int p = -1 - lane;  // inactive lanes: a pair of their own
    if (act) {
      int lo = 0, hi = J - 1;  // the last pair starting at or before s
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pstart[mid] <= s)
          lo = mid;
        else
          hi = mid - 1;
      }
      p = lo;
    }
    const unsigned same = __match_any_sync(0xffffffffu, p);
    const unsigned fin = __ballot_sync(0xffffffffu, act && hx[act ? s : 0] < KNN_INF) & same;
    if (act && lane == __ffs(same) - 1 && fin) atomicAdd(count + p, __popc(fin));
  }
}

struct SilArgs {
  const float* Xp;        // [N][KD] prepared rows in sorted order
  const float* hx;        // [N] |x - c|^2 / 2; not finite: the row takes no part
  const int* pstart;      // [J + 1] first sorted row of each pair
  const int* count;       // [J] finite rows of each pair
  const int4* tiles;      // {first row, end row, first pair, end pair of the rows' group}
  const int* sort_perm;   // sorted row -> caller's row
  double* out;            // [N] in the caller's order
  int KD, stages;
};

// grid = tiles, 2 TQ threads: warpgroup g multiplies the rows [64 g, 64 g + 64) of the tile
template <int TQ>
__global__ void __launch_bounds__(2 * TQ, 1) k_silhouette_tc(SilArgs a) {
  constexpr int TN = KNN_TN;
  constexpr int THREADS = 2 * TQ, NACC = TN / 2, NG = TN / 8;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int KD = a.KD, KD4 = KD >> 2, S = a.stages;
  float* Qhi = reinterpret_cast<float*>(smem_raw);  // [KD/4][TQ][4]
  float* Qlo = Qhi + (size_t)TQ * KD;
  float* Braw = Qlo + (size_t)TQ * KD;              // [S][KD/4][TN][4]  raw rows = hi operand
  float* Blo = Braw + (size_t)S * TN * KD;
  float* hxs = Blo + (size_t)TN * KD;               // [2][TN]  hx of the tile, +inf past the group
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, w4 = warp & 3;
  const int4 tile = a.tiles[blockIdx.x];
  const int q0 = tile.x, q1 = tile.y, gp0 = tile.z, gp1 = tile.w;
  const int x0 = a.pstart[gp0], x1 = a.pstart[gp1];
  const int xtiles = (x1 - x0 + TN - 1) / TN;

  // reference tile t of the group -> stage buffer (row per thread, one 16-byte piece per chunk) and its hx
  auto issue = [&](int t) {
    float* dst = Braw + (size_t)(S == 2 ? (t & 1) : 0) * TN * KD;
    const int r = tid % TN;
    const int j = x0 + t * TN + r;
    if (j < x1) {
      const float* src = a.Xp + (size_t)j * KD;
      const unsigned d0 = umma::smem_u32(dst + (size_t)r * 4);
      for (int c = tid / TN; c < KD4; c += THREADS / TN)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d0 + (unsigned)c * (TN * 16u)), "l"(src + 4 * c) : "memory");
    }
    if (tid < TN) hxs[(t & 1) * TN + tid] = j < x1 ? a.hx[j] : KNN_INF;
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  issue(0);

  for (int i = tid; i < TQ * KD4; i += THREADS) {
    const int r = i % TQ, c = i / TQ;
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < q1) z = *reinterpret_cast<const float4*>(a.Xp + (size_t)(q0 + r) * KD + 4 * c);
    const float4 l4 = umma::tf32_lo(z);
    *reinterpret_cast<float4*>(Qhi + ((size_t)c * TQ + r) * 4) = z;
    *reinterpret_cast<float4*>(Qlo + ((size_t)c * TQ + r) * 4) = l4;
  }

  // this thread's two rows of the tile (accumulator elements with bit 1 clear / set), their |q - c|^2 / 2 and pairs
  const int row0 = 64 * wg + 16 * w4 + (lane >> 2), row1 = row0 + 8;
  const int i0 = q0 + row0, i1 = q0 + row1;
  const float hq0 = i0 < q1 ? a.hx[i0] : 0.f, hq1 = i1 < q1 ? a.hx[i1] : 0.f;
  auto pair_of = [&](int i) {
    int lo = gp0, hi = gp1 - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (a.pstart[mid] <= i)
        lo = mid;
      else
        hi = mid - 1;
    }
    return lo;
  };
  const int op0 = pair_of(i0), op1 = pair_of(i1);
  double sum0 = 0.0, sum1 = 0.0;                      // the open pair's distances so far
  double own0 = 0.0, own1 = 0.0;                      // the sum over the row's own pair
  double b0 = __longlong_as_double(0x7ff0000000000000ll), b1 = b0;  // +inf: no other pair yet
  int cur = gp0;                                      // the open pair (the same in every thread)
  __syncthreads();

  const uint32_t lboA = TQ * 16, lboB = TN * 16, sbo = 128;
  const uint32_t aH = umma::smem_u32(Qhi) + wg * 64 * 16, aL = umma::smem_u32(Qlo) + wg * 64 * 16;
  const uint32_t bL = umma::smem_u32(Blo);

  for (int t = 0; t < xtiles; ++t) {
    float* raw = Braw + (size_t)(S == 2 ? (t & 1) : 0) * TN * KD;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // tile t is in shared memory; the MMAs of tile t - 1 are complete in every warp
    if (S == 2 && t + 1 < xtiles) issue(t + 1);
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
    const int j0 = x0 + t * TN, jend = min(j0 + TN, x1);
    const float* hxt = hxs + (t & 1) * TN;
    // distances, 0 for the row itself, a column that takes no part and a column past the group (hx = +inf)
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const float2 h2 = *reinterpret_cast<const float2*>(hxt + 8 * g + 2 * (lane & 3));
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * g + e;
        const float hj = (e & 1) ? h2.y : h2.x, hq = (e & 2) ? hq1 : hq0;
        const bool self = j0 + umma::frag_col(i, lane) == ((e & 2) ? i1 : i0);
        const float d2 = fmaxf(0.f, 2.f * ((hq + hj) - acc[i]));
        acc[i] = hj < KNN_INF && !self ? sqrtf(d2) : 0.f;
      }
    }
    if (S == 1 && t + 1 < xtiles) {
      __syncthreads();  // both warpgroups are done with the only stage
      issue(t + 1);
    }
    // the tile's runs of one pair, in order; every thread walks the same runs
    for (int rs = j0; rs < jend;) {
      const int pe = __ldg(a.pstart + cur + 1), re = min(pe, jend);
      float f0 = 0.f, f1 = 0.f;
      if (rs == j0 && re == jend) {  // one run covers the tile (columns past it are 0)
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
          if (i & 2)
            f1 += acc[i];
          else
            f0 += acc[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
          const int j = j0 + umma::frag_col(i, lane);
          const float v = j >= rs && j < re ? acc[i] : 0.f;
          if (i & 2)
            f1 += v;
          else
            f0 += v;
        }
      }
      f0 += __shfl_xor_sync(0xffffffffu, f0, 1);
      f1 += __shfl_xor_sync(0xffffffffu, f1, 1);
      f0 += __shfl_xor_sync(0xffffffffu, f0, 2);
      f1 += __shfl_xor_sync(0xffffffffu, f1, 2);
      sum0 += (double)f0;
      sum1 += (double)f1;
      if (re == pe) {  // the run closes pair cur
        const int n = __ldg(a.count + cur);
        if (cur == op0)
          own0 = sum0;
        else if (n > 0)
          b0 = fmin(b0, sum0 / n);
        if (cur == op1)
          own1 = sum1;
        else if (n > 0)
          b1 = fmin(b1, sum1 / n);
        sum0 = sum1 = 0.0;
        ++cur;
      }
      rs = re;
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");

  if ((lane & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = h ? i1 : i0;
      if (i >= q1) continue;
      const double nan = __longlong_as_double(0x7ff8000000000000ll);
      const double b = h ? b1 : b0, own = h ? own1 : own0;
      const int n = __ldg(a.count + (h ? op1 : op0));
      double s;
      if (!((h ? hq1 : hq0) < KNN_INF) || !(b < __longlong_as_double(0x7ff0000000000000ll)))
        s = nan;  // the row takes no part, or no other label of its group has a finite row
      else if (n == 1)
        s = 0.0;
      else {
        const double av = own / (n - 1), m = fmax(av, b);
        s = m > 0.0 ? (b - av) / m : 0.0;
      }
      a.out[a.sort_perm[i]] = s;
    }
  }
}

}  // namespace hb
