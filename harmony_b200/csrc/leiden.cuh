// leiden.cuh — the kernels of hb_umap_graph and hb_leiden (DESIGN §16): umap's smooth kNN distances and fuzzy union
// of a neighbour graph, and the local moving, refinement and aggregation of deterministic Leiden on a CSR graph.
// Every sum that decides something runs in a fixed order (a thread's own loop, or a fixed lane stride and xor tree),
// so two calls give bit-identical results.  Included by harmony_b200.cu.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int UMAP_MAX_K = 128;       // listed neighbours per row (hb_knn's k <= 64)
constexpr int LEIDEN_SUM_THREADS = 1024;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- hb_umap_graph
// One warp per row: rho (the smallest positive listed distance), umap's bisection for sigma (before the floor), the
// sum and count of the listed distances.  A listed entry has idx >= 0 and a finite distance.
__global__ void k_umap_sigma(const int32_t* __restrict__ idx, const float* __restrict__ dist, int64_t N, int k,
                             double target, double* __restrict__ rho, double* __restrict__ sigma,
                             double* __restrict__ row_sum, double* __restrict__ row_cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < N; i += warps) {
    double d[UMAP_MAX_K / 32];
    bool ok[UMAP_MAX_K / 32];
    double mn = INFINITY, sum = 0.0, cnt = 0.0;
#pragma unroll
    for (int t = 0; t < UMAP_MAX_K / 32; ++t) {
      const int m = lane + 32 * t;
      ok[t] = false;
      d[t] = 0.0;
      if (m < k) {
        const float x = dist[i * k + m];
        ok[t] = idx[i * k + m] >= 0 && isfinite(x);
        if (ok[t]) {
          d[t] = (double)x;
          sum += d[t];
          cnt += 1.0;
          if (d[t] > 0.0) mn = fmin(mn, d[t]);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    sum = warp_sum_d(sum);
    cnt = warp_sum_d(cnt);
    const double r = isfinite(mn) ? mn : 0.0;
    double lo = 0.0, hi = INFINITY, mid = 1.0;
    for (int it = 0; it < 64; ++it) {
      double ps = 0.0;
#pragma unroll
      for (int t = 0; t < UMAP_MAX_K / 32; ++t)
        if (ok[t]) {
          const double x = d[t] - r;
          ps += x > 0.0 ? exp(-(x / mid)) : 1.0;
        }
      ps = warp_sum_d(ps);
      if (fabs(ps - target) < 1e-5) break;
      if (ps > target) {
        hi = mid;
        mid = (lo + hi) / 2.0;
      } else {
        lo = mid;
        mid = isinf(hi) ? mid * 2.0 : (lo + hi) / 2.0;
      }
    }
    if (lane == 0) {
      rho[i] = r;
      sigma[i] = mid;
      row_sum[i] = sum;
      row_cnt[i] = cnt;
    }
  }
}

// The sum of x[0..n) in a fixed order: thread t of one block adds x[t], x[t + T], ..., then a fixed tree
__global__ void __launch_bounds__(LEIDEN_SUM_THREADS) k_sum_fixed(const double* __restrict__ x, int64_t n,
                                                                  double* __restrict__ out) {
  __shared__ double part[LEIDEN_SUM_THREADS];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += LEIDEN_SUM_THREADS) s += x[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int w = LEIDEN_SUM_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = part[0];
}

// The neighbour lists: every entry -1 or a row in 0..N-1, and no row listing one row twice.  The smallest bad entry,
// times 2 plus the reason (0: range, 1: repeat), into *bad.  Read only.
__global__ void k_umap_check(const int32_t* __restrict__ idx, int64_t N, int k, unsigned long long* __restrict__ bad) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N * k; e += (int64_t)gridDim.x * blockDim.x) {
    const int j = idx[e];
    int why = -1;
    if (j < -1 || j >= N) why = 0;
    else if (j >= 0)
      for (int64_t f = e - e % k; f < e; ++f)
        if (idx[f] == j) {
          why = 1;
          break;
        }
    if (why >= 0) atomicMin(bad, (unsigned long long)e * 2ull + why);
  }
}

// The weight of every listed entry after umap's floor on sigma (w[i][m], 0 where nothing is listed or j = i), and
// the number of symmetric entries it emits: (i, j) always when w_ij + w_ji > 0, and (j, i) too when j does not list i
__global__ void k_umap_weights(const int32_t* __restrict__ idx, const float* __restrict__ dist, int64_t N, int k,
                               const double* __restrict__ rho, const double* __restrict__ sigma,
                               const double* __restrict__ row_sum, const double* __restrict__ row_cnt,
                               const double* __restrict__ totals, double* __restrict__ w) {
  const double mean_all = totals[0] / (totals[1] + (double)N);  // umap's mean over all rows, self entries included
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N * k; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / k;
    const int j = idx[e];
    const float x = dist[e];
    double v = 0.0;
    if (j >= 0 && isfinite(x) && j != i) {
      double s = sigma[i];
      const double floor_s = 1e-3 * (rho[i] > 0.0 ? row_sum[i] / (row_cnt[i] + 1.0) : mean_all);
      if (s < floor_s) s = floor_s;
      const double t = (double)x - rho[i];
      v = (t <= 0.0 || s == 0.0) ? 1.0 : exp(-(t / s));
    }
    w[e] = v;
  }
}
// w_ji: the weight row j gives i (0 if j does not list i)
__device__ __forceinline__ double umap_back(const int32_t* __restrict__ idx, const double* __restrict__ w, int k,
                                            int64_t j, int64_t i, bool* listed) {
  for (int m = 0; m < k; ++m)
    if (idx[j * k + m] == (int32_t)i && w[j * k + m] > 0.0) {
      *listed = true;
      return w[j * k + m];
    }
  *listed = false;
  return 0.0;
}
// emit = false: cnt[e] = entries emitted for listed entry e; emit = true: write them at pos[e] (the scan of cnt)
template <bool EMIT>
__global__ void k_umap_sym(const int32_t* __restrict__ idx, int64_t N, int k, const double* __restrict__ w,
                           int* __restrict__ cnt, const int* __restrict__ pos, int* __restrict__ out_row,
                           int* __restrict__ out_col, double* __restrict__ out_w) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N * k; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / k;
    const double a = w[e];
    int c = 0;
    if (a > 0.0) {
      const int j = idx[e];
      bool back = false;
      const double b = umap_back(idx, w, k, j, i, &back);
      const double p = a + b - a * b;
      if (p > 0.0) {
        c = back ? 1 : 2;
        if (EMIT) {
          const int q = pos[e];
          out_row[q] = (int)i;
          out_col[q] = j;
          out_w[q] = p;
          if (!back) {
            out_row[q + 1] = j;
            out_col[q + 1] = (int)i;
            out_w[q + 1] = p;
          }
        }
      }
    }
    if (!EMIT) cnt[e] = c;
  }
}
// The sorted entries (perm into the emitted ones) into the caller's CSR; indptr from the row starts
__global__ void k_umap_write(const int* __restrict__ perm, int64_t nnz, const int* __restrict__ col,
                             const double* __restrict__ wv, int32_t* __restrict__ indices, float* __restrict__ data) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < nnz; p += (int64_t)gridDim.x * blockDim.x) {
    const int e = perm[p];
    indices[p] = col[e];
    data[p] = (float)wv[e];
  }
}
__global__ void k_indptr64(const int* __restrict__ start, int64_t n1, int64_t* __restrict__ indptr) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n1; i += (int64_t)gridDim.x * blockDim.x)
    indptr[i] = start[i];
}

// ---- hb_leiden: the caller's graph
// indptr: 0 at row 0, nnz at row N, never decreasing; the smallest bad row into *bad
__global__ void k_leiden_check_rows(const int64_t* __restrict__ indptr, int64_t N, int64_t nnz,
                                    unsigned long long* __restrict__ bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= N; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a = indptr[i];
    const bool ok = (i == 0 ? a == 0 : a >= indptr[i - 1]) && (i < N || a == nnz) && a <= nnz;
    if (!ok) atomicMin(bad, (unsigned long long)i);
  }
}
// Every entry (i, j): 0 <= j < N, j != i, above the row's previous entry and a finite weight > 0 (MIRROR false); then,
// on a graph that passed those, (j, i) listed with the same weight (MIRROR true), so that the binary search runs on
// sorted rows only.  The smallest bad entry, times 8 plus the reason, into *bad.  One warp per row.
template <typename T, bool MIRROR>
__global__ void k_leiden_check_entries(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                       const T* __restrict__ data, int64_t N, unsigned long long* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < N; i += warps) {
    const int64_t a = indptr[i], b = indptr[i + 1];
    for (int64_t e = a + lane; e < b; e += 32) {
      const int j = indices[e];
      const T v = data[e];
      int why = 0;
      if (!MIRROR) {
        if (j < 0 || j >= N) why = 1;
        else if (j == i) why = 2;
        else if (e > a && indices[e - 1] >= j) why = 3;
        else if (!(isfinite((double)v) && v > (T)0)) why = 4;
      } else {
        int64_t lo = indptr[j], hi = indptr[j + 1];
        while (lo < hi) {  // the first entry of row j at or above i
          const int64_t m = (lo + hi) >> 1;
          if (indices[m] < i) lo = m + 1;
          else hi = m;
        }
        if (lo >= indptr[j + 1] || indices[lo] != (int32_t)i) why = 5;
        else if (data[lo] != v) why = 6;
      }
      if (why) atomicMin(bad, (unsigned long long)e * 8ull + why);
    }
  }
}
// The caller's graph as the level-0 graph: int row starts, columns, fp64 weights and each entry's row
template <typename T>
__global__ void k_leiden_level0(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                const T* __restrict__ data, int64_t N, int* __restrict__ ip, int* __restrict__ col,
                                double* __restrict__ w, int* __restrict__ row) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i <= N; i += warps) {
    if (lane == 0) ip[i] = (int)indptr[i];
    if (i == N) continue;
    for (int64_t e = indptr[i] + lane; e < indptr[i + 1]; e += 32) {
      col[e] = indices[e];
      w[e] = (double)data[e];
      row[e] = (int)i;
    }
  }
}
// out[s] = the sum of vals[perm[p]] (perm null: vals[p]) over p in [start[s], start[s + 1]): one warp per segment,
// fixed lane stride and tree.  `rows` segments.
__global__ void k_seg_sum(const double* __restrict__ vals, const int* __restrict__ perm, const int* __restrict__ start,
                          int rows, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += warps) {
    double t = 0.0;
    for (int p = start[s] + lane; p < start[s + 1]; p += 32) t += vals[perm ? perm[p] : p];
    t = warp_sum_d(t);
    if (lane == 0) out[s] = t;
  }
}
// key[p] = code[of[perm[p]]] (perm null: p; of null: the index itself) — the sort keys of the next radix passes
__global__ void k_gather_key(const int* __restrict__ code, const int* __restrict__ of, const int* __restrict__ perm,
                             int64_t n, int* __restrict__ key) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int e = perm ? perm[p] : (int)p;
    key[p] = code[of ? of[e] : e];
  }
}

struct LeidenMoveArgs {
  const int *ip, *col, *perm;    // the level graph and its entries sorted by (row, community of the column)
  const double *w, *k, *tot;     // weights, degrees and community totals
  const int* comm;
  int* next;
  int n, parity;
  double gamma, inv2m;
  int* moved;
};
// Local moving, one thread per vertex: the gain of each adjacent community and of staying, in fp64 from the state
// at the start of the sweep; the best (the smaller id on a tie), taken when it beats staying in the sweep's direction
__global__ void k_leiden_move(LeidenMoveArgs a) {
  int moves = 0;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < a.n; v += gridDim.x * blockDim.x) {
    const int own = a.comm[v];
    const double kv = a.k[v], f = a.gamma * kv * a.inv2m;
    double w_own = 0.0, best_g = -INFINITY, run = 0.0;
    int best_c = -1, cur = -1;
    for (int p = a.ip[v]; p <= a.ip[v + 1]; ++p) {
      int c = -1;
      double x = 0.0;
      if (p < a.ip[v + 1]) {
        const int e = a.perm[p], j = a.col[e];
        if (j == v) continue;
        c = a.comm[j];
        x = a.w[e];
      }
      if (c != cur) {
        if (cur >= 0) {
          if (cur == own) w_own = run;
          else {
            const double g = run - f * a.tot[cur];
            if (g > best_g) {
              best_g = g;
              best_c = cur;
            }
          }
        }
        cur = c;
        run = 0.0;
      }
      run += x;
    }
    const double stay = w_own - f * (a.tot[own] - kv);
    int target = own;
    if (best_c >= 0 && (best_g > stay || (best_g == stay && best_c < own))) target = best_c;
    const bool allowed = a.parity == 0 ? target < own : target > own;
    const bool go = target != own && best_g > stay && allowed;
    a.next[v] = go ? target : own;
    moves += go;
  }
  if (moves) atomicAdd(a.moved, moves);
}

struct LeidenRefineArgs {
  const int *ip, *col, *perm;  // entries sorted by (row, sub-community of the column)
  const double *w, *k, *tot;   // weights, degrees, totals of the communities of P
  const int *comm, *sub, *sub_start;  // P, the sub-communities, the starts of the vertices sorted by sub
  const double *sub_tot, *sub_ext, *win;  // each sub's total and weight to the rest of its community; w(v, C \ v)
  int* target;
  int* proposed;
  int n;
  double gamma, inv2m;
};
// ext[v] = the weight from v to the rest of its community outside its own sub-community; win[v] = w(v, C \ v)
__global__ void k_leiden_ext(const int* __restrict__ ip, const int* __restrict__ col, const double* __restrict__ w,
                             const int* __restrict__ comm, const int* __restrict__ sub, int n, double* __restrict__ ext,
                             double* __restrict__ win) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    double x = 0.0, y = 0.0;
    for (int e = ip[v]; e < ip[v + 1]; ++e) {
      const int j = col[e];
      if (j == v || comm[j] != comm[v]) continue;
      y += w[e];
      if (sub[j] != sub[v]) x += w[e];
    }
    ext[v] = x;
    if (win) win[v] = y;
  }
}
// A singleton v that is well connected to its community proposes the well-connected sub-community of the largest
// positive gain (the smaller id on a tie) and marks it proposed
__global__ void k_leiden_propose(LeidenRefineArgs a) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < a.n; v += gridDim.x * blockDim.x) {
    int best_s = -1;
    const int own = a.comm[v];
    const double kv = a.k[v], T = a.tot[own];
    const bool single = a.sub[v] == v && a.sub_start[v + 1] - a.sub_start[v] == 1;
    if (single && a.win[v] >= a.gamma * kv * (T - kv) * a.inv2m) {
      double best = 0.0, run = 0.0;
      int cur = -1;
      for (int p = a.ip[v]; p <= a.ip[v + 1]; ++p) {
        int s = -1;
        double x = 0.0;
        if (p < a.ip[v + 1]) {
          const int e = a.perm[p], j = a.col[e];
          if (j == v || a.comm[j] != own) continue;
          s = a.sub[j];
          x = a.w[e];
        }
        if (s != cur) {
          if (cur >= 0) {
            const double St = a.sub_tot[cur];
            const bool wc = a.sub_ext[cur] >= a.gamma * St * (T - St) * a.inv2m;
            const double g = run - a.gamma * kv * St * a.inv2m;
            if (wc && g > best) {
              best = g;
              best_s = cur;
            }
          }
          cur = s;
          run = 0.0;
        }
        run += x;
      }
    }
    a.target[v] = best_s;
    if (best_s >= 0) a.proposed[best_s] = 1;
  }
}
// A proposer that no one proposed to joins its target
__global__ void k_leiden_join(const int* __restrict__ target, const int* __restrict__ proposed, int n,
                              int* __restrict__ sub, int* __restrict__ moved) {
  int moves = 0;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    if (target[v] >= 0 && !proposed[v]) {
      sub[v] = target[v];
      ++moves;
    }
  if (moves) atomicAdd(moved, moves);
}
// used[s] = 1 for a non-empty sub-community
__global__ void k_leiden_used(const int* __restrict__ sub_start, int n, int* __restrict__ used) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= n; s += gridDim.x * blockDim.x)
    used[s] = s < n && sub_start[s + 1] > sub_start[s];
}
// vmap[v] = the next level's vertex of v; cmin[c] = the smallest next-level vertex of community c; orig -> next level
__global__ void k_leiden_vmap(const int* __restrict__ sub, const int* __restrict__ newid, const int* __restrict__ comm,
                              int n, int* __restrict__ vmap, int* __restrict__ cmin) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const int s = newid[sub[v]];
    vmap[v] = s;
    atomicMin(cmin + comm[v], s);
  }
}
__global__ void k_leiden_next_comm(const int* __restrict__ vmap, const int* __restrict__ comm,
                                   const int* __restrict__ cmin, int n, int* __restrict__ next_comm) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    next_comm[vmap[v]] = cmin[comm[v]];
}
__global__ void k_leiden_compose(int* __restrict__ orig, int64_t N, const int* __restrict__ vmap) {
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < N; o += (int64_t)gridDim.x * blockDim.x)
    orig[o] = vmap[orig[o]];
}
// head[p] = whether sorted entry p starts a new (vmap[row], vmap[col]) pair; the last word is 0 for the scan
__global__ void k_leiden_heads(const int* __restrict__ perm, const int* __restrict__ row, const int* __restrict__ col,
                               const int* __restrict__ vmap, int nnz, int* __restrict__ head) {
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p <= nnz; p += gridDim.x * blockDim.x) {
    if (p == nnz) {
      head[p] = 0;
      continue;
    }
    const int e = perm[p];
    bool h = p == 0;
    if (!h) {
      const int f = perm[p - 1];
      h = vmap[row[e]] != vmap[row[f]] || vmap[col[e]] != vmap[col[f]];
    }
    head[p] = h;
  }
}
// After the scan of head: seg_start[q] = first sorted entry of pair q, and the pair's row and column
__global__ void k_leiden_segs(const int* __restrict__ perm, const int* __restrict__ row, const int* __restrict__ col,
                              const int* __restrict__ vmap, const int* __restrict__ pos, int nnz,
                              int* __restrict__ seg_start, int* __restrict__ seg_row, int* __restrict__ seg_col) {
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += gridDim.x * blockDim.x)
    if (pos[p + 1] != pos[p]) {
      const int q = pos[p], e = perm[p];
      seg_start[q] = p;
      seg_row[q] = vmap[row[e]];
      seg_col[q] = vmap[col[e]];
    }
}
// in[v] = the weight of v's row to its own label, one warp per row (fixed order)
__global__ void k_leiden_inner(const int* __restrict__ ip, const int* __restrict__ col, const double* __restrict__ w,
                               const int* __restrict__ lab, int n, double* __restrict__ in) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); v < n; v += warps) {
    double t = 0.0;
    for (int e = ip[v] + lane; e < ip[v + 1]; e += 32)
      if (lab[col[e]] == lab[v]) t += w[e];
    t = warp_sum_d(t);
    if (lane == 0) in[v] = t;
  }
}
// Community sizes and smallest members for the final numbering
__global__ void k_leiden_sizes(const int* __restrict__ lab, int64_t N, int* __restrict__ size, int* __restrict__ first) {
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < N; o += (int64_t)gridDim.x * blockDim.x) {
    atomicAdd(size + lab[o], 1);
    atomicMin(first + lab[o], (int)o);
  }
}
__global__ void k_leiden_relabel(const int* __restrict__ lab, int64_t N, const int* __restrict__ rank,
                                 int32_t* __restrict__ out) {
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < N; o += (int64_t)gridDim.x * blockDim.x)
    out[o] = rank[lab[o]];
}

}  // namespace hb
