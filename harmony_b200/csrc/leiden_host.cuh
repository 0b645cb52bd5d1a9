// leiden_host.cuh — hb_umap_graph and hb_leiden (DESIGN §16): the checks and launches of leiden.cuh, sort.cuh's
// stable radix sort and chained scan for every grouping, and the loops of local moving, refinement, aggregation and
// iterations on the host.  The calls need no setup and touch no state of a Harmony run or a mapping.  Included by
// harmony_b200.cu.
#pragma once

namespace {

constexpr int LEIDEN_MAX_SWEEPS = 128;      // local-moving sweeps per level
constexpr int LEIDEN_MAX_ROUNDS = 1024;     // refinement rounds per level
constexpr int LEIDEN_MAX_LEVELS = 1024;     // levels per iteration
constexpr int LEIDEN_MAX_ITERATIONS = 64;   // iterations of n_iterations = -1

struct LeidenRun {
  hb_handle* h;
  int64_t N;
  double gamma, inv2m;
  LeidenGraph* g0;
  int64_t levels = 0, sweeps = 0, rounds = 0;
  bool capped = false;
};

int leiden_grid(hb_handle* h, int64_t n) { return grid_for(n, 256, h->num_sms * 8); }

// vertices of g sorted by code (B.vperm) and the code starts (B.vstart, n + 1)
int sort_vertices(hb_handle* h, const LeidenGraph& g, const int* code) {
  LeidenBufs& B = score_scratch(h).leiden;
  TRY(launch(h, k_gather_key, dim3(leiden_grid(h, g.n)), dim3(256), 0, code, (const int*)nullptr, (const int*)nullptr,
             (int64_t)g.n, B.key.p));
  return sort_by_code(h, B.sort, B.key.p, g.n, g.n, nullptr, B.vperm.p, nullptr, B.vstart.p);
}
// sums over the segments of sort_vertices into out
int vertex_sums(hb_handle* h, const LeidenGraph& g, const double* vals, double* out) {
  LeidenBufs& B = score_scratch(h).leiden;
  return launch(h, k_seg_sum, dim3(grid_for((int64_t)g.n * 32, 256, h->num_sms * 8)), dim3(256), 0, vals,
                (const int*)B.vperm.p, (const int*)B.vstart.p, g.n, out);
}
// The n entries whose minor keys B.key holds, sorted stably by (major, minor) into B.eperm (by the minor key alone:
// B.eperm1), both keys codes below n_codes.  An entry's major key is code[of[e]] (of null: code[e]); starts: the
// majors' starts, if not null.
int sort_pairs(hb_handle* h, int64_t n, int n_codes, const int* code, const int* of, int* starts) {
  LeidenBufs& B = score_scratch(h).leiden;
  TRY(sort_by_code(h, B.sort, B.key.p, n, n_codes, nullptr, B.eperm1.p, nullptr, nullptr));
  TRY(launch(h, k_gather_key, dim3(leiden_grid(h, n)), dim3(256), 0, code, of, (const int*)B.eperm1.p, n, B.key.p));
  return sort_by_code(h, B.sort, B.key.p, n, n_codes, B.eperm1.p, B.eperm.p, nullptr, starts);
}
// g's entries sorted by (row, code[col]) into B.eperm (code_row null: by the row itself, else by code_row[row])
int sort_entries(hb_handle* h, const LeidenGraph& g, const int* code_col, const int* code_row) {
  LeidenBufs& B = score_scratch(h).leiden;
  TRY(launch(h, k_gather_key, dim3(leiden_grid(h, g.nnz)), dim3(256), 0, code_col, (const int*)g.col.p,
             (const int*)nullptr, (int64_t)g.nnz, B.key.p));
  return sort_pairs(h, g.nnz, g.n, code_row ? code_row : (const int*)g.row.p,
                    code_row ? (const int*)g.row.p : (const int*)nullptr, nullptr);
}

// Local moving of g from the partition in B.comm; *moved = whether any vertex moved
int leiden_move(LeidenRun& r, const LeidenGraph& g, bool* moved) {
  hb_handle* h = r.h;
  RegionScope rs(h, "leiden_move");
  LeidenBufs& B = score_scratch(h).leiden;
  int* cnt = B.small.p;
  *moved = false;
  int quiet = 0;
  for (int s = 0;; ++s) {
    if (s == LEIDEN_MAX_SWEEPS) {
      r.capped = true;
      break;
    }
    TRY(sort_vertices(h, g, B.comm.p));
    TRY(vertex_sums(h, g, g.deg.p, B.tot.p));
    TRY(sort_entries(h, g, B.comm.p, nullptr));
    CK(cudaMemsetAsync(cnt, 0, sizeof(int), h->stream));
    const LeidenMoveArgs a{g.ip.p, g.col.p, B.eperm.p, g.w.p, g.deg.p, B.tot.p, B.comm.p, B.next.p, g.n, s & 1,
                           r.gamma, r.inv2m, cnt};
    TRY(launch(h, k_leiden_move, dim3(leiden_grid(h, g.n)), dim3(256), 0, a));
    int m = 0;
    TRY(read_back(h, cnt, &m));
    ++r.sweeps;
    swap_bufs(B.comm, B.next);
    if (m) *moved = true;
    quiet = m ? 0 : quiet + 1;
    if (quiet == 2) break;
  }
  return 0;
}

// Refinement of the partition B.comm of g into B.sub; *moved = whether any vertex joined a sub-community
int leiden_refine(LeidenRun& r, const LeidenGraph& g, bool* moved) {
  hb_handle* h = r.h;
  RegionScope rs(h, "leiden_refine");
  LeidenBufs& B = score_scratch(h).leiden;
  const dim3 grid(leiden_grid(h, g.n)), block(256);
  int* cnt = B.small.p;
  *moved = false;
  TRY(sort_vertices(h, g, B.comm.p));
  TRY(vertex_sums(h, g, g.deg.p, B.tot.p));
  k_identity_perm<<<grid, block, 0, h->stream>>>(g.n, B.sub.p, B.target.p);
  CKL();
  TRY(launch(h, k_leiden_ext, grid, block, 0, (const int*)g.ip.p, (const int*)g.col.p, (const double*)g.w.p,
             (const int*)B.comm.p, (const int*)B.sub.p, g.n, B.ext.p, B.win.p));
  for (int round = 0;; ++round) {
    TRY(sort_vertices(h, g, B.sub.p));
    TRY(vertex_sums(h, g, g.deg.p, B.sub_tot.p));
    TRY(launch(h, k_leiden_ext, grid, block, 0, (const int*)g.ip.p, (const int*)g.col.p, (const double*)g.w.p,
               (const int*)B.comm.p, (const int*)B.sub.p, g.n, B.ext.p, (double*)nullptr));
    TRY(vertex_sums(h, g, B.ext.p, B.sub_ext.p));
    if (round == LEIDEN_MAX_ROUNDS) {  // the sub-communities of this round's sort stand
      r.capped = true;
      break;
    }
    TRY(sort_entries(h, g, B.sub.p, nullptr));
    CK(cudaMemsetAsync(B.proposed.p, 0, sizeof(int) * g.n, h->stream));
    CK(cudaMemsetAsync(cnt, 0, sizeof(int), h->stream));
    const LeidenRefineArgs a{g.ip.p, g.col.p, B.eperm.p, g.w.p, g.deg.p, B.tot.p, B.comm.p, B.sub.p, B.vstart.p,
                             B.sub_tot.p, B.sub_ext.p, B.win.p, B.target.p, B.proposed.p, g.n, r.gamma, r.inv2m};
    TRY(launch(h, k_leiden_propose, grid, block, 0, a));
    TRY(launch(h, k_leiden_join, grid, block, 0, (const int*)B.target.p, (const int*)B.proposed.p, g.n, B.sub.p, cnt));
    int m = 0;
    TRY(read_back(h, cnt, &m));
    ++r.rounds;
    if (!m) break;
    *moved = true;
  }
  return 0;
}

// One vertex per sub-community of g (B.sub, sorted in B.vstart) into `next`; B.comm becomes the next level's start
// partition and B.omap the next level's vertex of every caller row
int leiden_aggregate(LeidenRun& r, const LeidenGraph& g, LeidenGraph& next) {
  hb_handle* h = r.h;
  RegionScope rs(h, "leiden_aggregate");
  LeidenBufs& B = score_scratch(h).leiden;
  const cudaStream_t st = h->stream;
  const dim3 grid(leiden_grid(h, g.n)), block(256);
  TRY(launch(h, k_leiden_used, dim3(leiden_grid(h, (int64_t)g.n + 1)), block, 0, (const int*)B.vstart.p, g.n, B.newid.p));
  TRY(chained_scan(h, st, B.newid.p, (int64_t)g.n + 1, 1, B.sort.scan));
  int n2 = 0;
  TRY(read_back(h, B.newid.p + g.n, &n2));
  CK(cudaMemsetAsync(B.cmin.p, 0x7f, sizeof(int) * g.n, st));
  TRY(launch(h, k_leiden_vmap, grid, block, 0, (const int*)B.sub.p, (const int*)B.newid.p, (const int*)B.comm.p, g.n,
             B.vmap.p, B.cmin.p));
  TRY(launch(h, k_leiden_next_comm, grid, block, 0, (const int*)B.vmap.p, (const int*)B.comm.p, (const int*)B.cmin.p,
             g.n, B.next.p));
  TRY(launch(h, k_leiden_compose, dim3(leiden_grid(h, r.N)), block, 0, B.omap.p, r.N, (const int*)B.vmap.p));
  TRY(sort_entries(h, g, B.vmap.p, B.vmap.p));  // rows keyed by vmap too: (vmap[row], vmap[col]) order
  const dim3 egrid(leiden_grid(h, (int64_t)g.nnz + 1));
  TRY(launch(h, k_leiden_heads, egrid, block, 0, (const int*)B.eperm.p, (const int*)g.row.p, (const int*)g.col.p,
             (const int*)B.vmap.p, g.nnz, B.head.p));
  TRY(chained_scan(h, st, B.head.p, (int64_t)g.nnz + 1, 1, B.sort.scan));
  int nnz2 = 0;
  TRY(read_back(h, B.head.p + g.nnz, &nnz2));
  TRY(next.reserve(h, n2, nnz2));
  CK(B.seg_start.reserve((size_t)nnz2 + 1));
  TRY(launch(h, k_leiden_segs, egrid, block, 0, (const int*)B.eperm.p, (const int*)g.row.p, (const int*)g.col.p,
             (const int*)B.vmap.p, (const int*)B.head.p, g.nnz, B.seg_start.p, next.row.p, next.col.p));
  CK(cudaMemcpyAsync(B.seg_start.p + nnz2, &g.nnz, sizeof(int), cudaMemcpyHostToDevice, st));
  TRY(launch(h, k_seg_sum, dim3(grid_for((int64_t)nnz2 * 32, 256, h->num_sms * 8)), block, 0, (const double*)g.w.p,
             (const int*)B.eperm.p, (const int*)B.seg_start.p, nnz2, next.w.p));
  k_tuple_starts<<<leiden_grid(h, (int64_t)nnz2 + 1), 256, 0, st>>>(next.row.p, nnz2, n2, next.ip.p);
  CKL();
  TRY(launch(h, k_seg_sum, dim3(grid_for((int64_t)n2 * 32, 256, h->num_sms * 8)), block, 0, (const double*)next.w.p,
             (const int*)nullptr, (const int*)next.ip.p, n2, next.deg.p));
  swap_bufs(B.comm, B.next);
  CK(cudaStreamSynchronize(st));  // the host's nnz word is read by the copy above
  return 0;
}

// Final numbering of B.lab into `labels`: by decreasing size, ties by the smallest member; the number of communities
int leiden_number(LeidenRun& r, int32_t* labels, int* n_comm) {
  hb_handle* h = r.h;
  LeidenBufs& B = score_scratch(h).leiden;
  const cudaStream_t st = h->stream;
  const int64_t N = r.N;
  CK(cudaMemsetAsync(B.size.p, 0, sizeof(int) * N, st));
  CK(cudaMemsetAsync(B.first.p, 0x7f, sizeof(int) * N, st));
  TRY(launch(h, k_leiden_sizes, dim3(leiden_grid(h, N)), dim3(256), 0, (const int*)B.lab.p, N, B.size.p, B.first.p));
  std::vector<int> size(N), first(N);
  CK(cudaMemcpyAsync(size.data(), B.size.p, sizeof(int) * N, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(first.data(), B.first.p, sizeof(int) * N, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::vector<int> order;
  for (int64_t c = 0; c < N; ++c)
    if (size[c]) order.push_back((int)c);
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    return size[a] != size[b] ? size[a] > size[b] : first[a] < first[b];
  });
  std::vector<int> rank(N, -1);
  for (size_t q = 0; q < order.size(); ++q) rank[order[q]] = (int)q;
  CK(cudaMemcpyAsync(B.size.p, rank.data(), sizeof(int) * N, cudaMemcpyHostToDevice, st));
  TRY(launch(h, k_leiden_relabel, dim3(leiden_grid(h, N)), dim3(256), 0, (const int*)B.lab.p, N, (const int*)B.size.p,
             labels));
  CK(cudaStreamSynchronize(st));  // rank goes on return
  *n_comm = (int)order.size();
  return 0;
}

// Q of `labels` on the level-0 graph: (sum of the weight inside communities - gamma sum tot_c^2 / 2m) / 2m
int leiden_quality(LeidenRun& r, const int32_t* labels, double* Q) {
  hb_handle* h = r.h;
  LeidenBufs& B = score_scratch(h).leiden;
  const LeidenGraph& g = *r.g0;
  TRY(launch(h, k_leiden_inner, dim3(grid_for((int64_t)g.n * 32, 256, h->num_sms * 8)), dim3(256), 0,
             (const int*)g.ip.p, (const int*)g.col.p, (const double*)g.w.p, (const int*)labels, g.n, B.ext.p));
  TRY(launch(h, k_sum_fixed, dim3(1), dim3(LEIDEN_SUM_THREADS), 0, (const double*)B.ext.p, (int64_t)g.n, B.dsmall.p));
  TRY(sort_vertices(h, g, labels));
  TRY(vertex_sums(h, g, g.deg.p, B.tot.p));
  std::vector<double> tot(g.n);
  double in = 0.0;
  CK(cudaMemcpyAsync(tot.data(), B.tot.p, sizeof(double) * g.n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(&in, B.dsmall.p, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  double sq = 0.0;
  for (double t : tot) sq += t * t;
  *Q = (in - r.gamma * sq * r.inv2m) * r.inv2m;
  return 0;
}

// One iteration from the start partition in B.comm (level 0); the result's labels (unnumbered) into B.lab
int leiden_iteration(LeidenRun& r) {
  hb_handle* h = r.h;
  LeidenBufs& B = score_scratch(h).leiden;
  k_identity_perm<<<leiden_grid(h, r.N), 256, 0, h->stream>>>(r.N, B.omap.p, B.target.p);
  CKL();
  LeidenGraph* g = r.g0;
  LeidenGraph* spare[2] = {&B.level[0], &B.level[1]};
  int which = 0;
  for (int level = 0;; ++level) {
    bool moved = false, refined = false;  // moved: reported by local moving, not needed to end the level loop
    TRY(leiden_move(r, *g, &moved));
    ++r.levels;
    if (level + 1 == LEIDEN_MAX_LEVELS) r.capped = true;
    if (level + 1 < LEIDEN_MAX_LEVELS) TRY(leiden_refine(r, *g, &refined));
    if (!refined || level + 1 == LEIDEN_MAX_LEVELS) break;  // the next level would repeat this one
    LeidenGraph* next = spare[which];
    which ^= 1;
    TRY(leiden_aggregate(r, *g, *next));
    g = next;
  }
  return launch(h, k_gather_key, dim3(leiden_grid(h, r.N)), dim3(256), 0, (const int*)B.comm.p, (const int*)B.omap.p,
                (const int*)nullptr, r.N, B.lab.p);
}

template <typename T>
int leiden_run(hb_handle* h, const int64_t* indptr, const int32_t* indices, const T* data, int64_t N, int64_t nnz,
               double gamma, int n_iterations, int32_t* labels, int* n_comm, double* Q, int* n_iter, int64_t* stats) {
  LeidenBufs& B = score_scratch(h).leiden;
  const cudaStream_t st = h->stream;
  // ---- the caller's graph, read only until it passes
  unsigned long long bad = 0;
  TRY(run_check(h, &bad, k_leiden_check_rows, dim3(leiden_grid(h, N + 1)), indptr, N, nnz));
  if (bad != ~0ull) return fail(h, 2, "hb_leiden: indptr[%llu] breaks 0 = indptr[0] <= ... <= indptr[N] = nnz = %lld", bad, (long long)nnz);
  const dim3 cgrid(grid_for(N * 32, 256, h->num_sms * 8));
  TRY(run_check(h, &bad, k_leiden_check_entries<T, false>, cgrid, indptr, indices, data, N));
  if (bad == ~0ull)  // rows in range, sorted and without diagonal: now the mirrors
    TRY(run_check(h, &bad, k_leiden_check_entries<T, true>, cgrid, indptr, indices, data, N));
  if (bad != ~0ull) {
    const int64_t e = (int64_t)(bad / 8);
    std::vector<int64_t> ip(N + 1);
    CK(cudaMemcpyAsync(ip.data(), indptr, sizeof(int64_t) * (N + 1), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const int64_t row = std::upper_bound(ip.begin(), ip.end(), e) - ip.begin() - 1;
    static const char* why[] = {"", "is not a row in 0..N-1", "is on the diagonal", "does not ascend within its row",
                                "has a weight that is not finite and > 0", "has no mirror entry (j, i)",
                                "has a weight that differs from its mirror (j, i)"};
    int j = 0;
    TRY(read_back(h, indices + e, &j));
    return fail(h, 2, "hb_leiden: the graph is not a symmetric CSR without diagonal: row %lld, entry %lld (column %d) %s",
                (long long)row, (long long)e, j, why[bad % 8]);
  }
  // ---- level 0 and the buffers of every level (no level is larger)
  LeidenGraph& g0 = B.g0;
  TRY(g0.reserve(h, (int)N, (int)nnz));
  const int64_t nv = std::max<int64_t>(N, 1), ne = std::max<int64_t>(nnz, 1);
  for (DevBuf<int>* b : {&B.comm, &B.next, &B.vperm, &B.sub, &B.target, &B.proposed, &B.cmin, &B.vmap, &B.omap, &B.lab,
                         &B.size, &B.first, &B.key, &B.eperm, &B.eperm1})
    CK(b->reserve((size_t)std::max(nv, (b == &B.key || b == &B.eperm || b == &B.eperm1) ? ne : nv)));
  for (DevBuf<int>* b : {&B.vstart, &B.newid}) CK(b->reserve((size_t)N + 1));
  CK(B.head.reserve((size_t)nnz + 1));
  for (DevBuf<double>* b : {&B.tot, &B.ext, &B.win, &B.sub_tot, &B.sub_ext}) CK(b->reserve((size_t)nv));
  CK(B.small.reserve(4));
  CK(B.dsmall.reserve(4));
  TRY(launch(h, k_leiden_level0<T>, dim3(grid_for((N + 1) * 32, 256, h->num_sms * 8)), dim3(256), 0, indptr, indices,
             data, N, g0.ip.p, g0.col.p, g0.w.p, g0.row.p));
  TRY(launch(h, k_seg_sum, dim3(grid_for(N * 32, 256, h->num_sms * 8)), dim3(256), 0, (const double*)g0.w.p,
             (const int*)nullptr, (const int*)g0.ip.p, (int)N, g0.deg.p));
  TRY(launch(h, k_sum_fixed, dim3(1), dim3(LEIDEN_SUM_THREADS), 0, (const double*)g0.deg.p, N, B.dsmall.p));
  double two_m = 0.0;
  CK(cudaMemcpyAsync(&two_m, B.dsmall.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  LeidenRun r{h, N, gamma, two_m > 0.0 ? 1.0 / two_m : 0.0, &g0};
  k_identity_perm<<<leiden_grid(h, N), 256, 0, st>>>(N, B.lab.p, B.target.p);  // singletons
  CKL();
  int iters = 0;
  std::vector<int32_t> prev, cur(N);
  if (two_m > 0.0) {
    const int cap = n_iterations < 0 ? LEIDEN_MAX_ITERATIONS : n_iterations;
    for (int it = 0; it < cap; ++it) {
      CK(cudaMemcpyAsync(B.comm.p, it == 0 ? B.lab.p : labels, sizeof(int) * N, cudaMemcpyDeviceToDevice, st));
      TRY(leiden_iteration(r));
      TRY(leiden_number(r, labels, n_comm));
      ++iters;
      if (n_iterations >= 0) continue;
      CK(cudaMemcpyAsync(cur.data(), labels, sizeof(int32_t) * N, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (cur == prev) break;
      prev = cur;
      if (it + 1 == cap) r.capped = true;
    }
  }
  if (iters == 0) TRY(leiden_number(r, labels, n_comm));  // no edge or no iteration: the start partition
  if (two_m > 0.0) TRY(leiden_quality(r, labels, Q));
  else *Q = 0.0;
  *n_iter = iters;
  if (stats) {
    stats[0] = r.levels;
    stats[1] = r.sweeps;
    stats[2] = r.rounds;
  }
  if (r.capped)
    h->warnings.push_back("hb_leiden: a cap on sweeps, refinement rounds, levels or iterations was reached; the "
                          "partition may not have converged");
  return 0;
}

int run_leiden(hb_handle* h, const int64_t* indptr, const int32_t* indices, const void* data, int dtype, int64_t N,
               int64_t nnz, double gamma, int n_iterations, int32_t* labels, int32_t* n_comm, double* Q, int32_t* n_iter,
               int64_t* stats, cudaStream_t caller) {
  if (N < 1 || N >= (1LL << 31)) return fail(h, 2, "hb_leiden: N = %lld rows are not supported (1 <= N < 2^31)", (long long)N);
  if (nnz < 0 || nnz >= (1LL << 31)) return fail(h, 2, "hb_leiden: nnz = %lld entries are not supported (nnz < 2^31)", (long long)nnz);
  if (!(gamma > 0.0) || !std::isfinite(gamma)) return fail(h, 2, "hb_leiden: resolution = %g must be finite and > 0", gamma);
  if (n_iterations < -1) return fail(h, 2, "hb_leiden: n_iterations = %d (-1: until no label changes, or >= 0)", n_iterations);
  if (dtype != HB_FLOAT32 && dtype != HB_FLOAT64) return fail(h, 2, "hb_leiden: unknown data dtype %d", dtype);
  if (!n_comm || !Q || !n_iter) return fail(h, 2, "hb_leiden: null n_comm, Q or n_iter");
  TRY(check_device_ptr(h, indptr, "indptr"));
  if (nnz > 0) {
    TRY(check_device_ptr(h, indices, "indices"));
    TRY(check_device_ptr(h, data, "data"));
  }
  TRY(check_device_ptr(h, labels, "labels"));
  return run_score(h, caller, "leiden", [&] {
    if (dtype == HB_FLOAT32)
      return leiden_run(h, indptr, indices, (const float*)data, N, nnz, gamma, n_iterations, labels, n_comm, Q, n_iter, stats);
    return leiden_run(h, indptr, indices, (const double*)data, N, nnz, gamma, n_iterations, labels, n_comm, Q, n_iter, stats);
  });
}

// ---- hb_umap_graph
int umap_run(hb_handle* h, const int32_t* idx, const float* dist, int64_t N, int k, int n_neighbors, int64_t* indptr,
             int32_t* indices, float* data, int64_t* nnz_out) {
  LeidenBufs& B = score_scratch(h).leiden;
  const cudaStream_t st = h->stream;
  const int64_t Nk = N * k;
  unsigned long long bad = 0;
  TRY(run_check(h, &bad, k_umap_check, dim3(grid_for(Nk, 256, h->num_sms * 8)), idx, N, k));
  if (bad != ~0ull) {
    const int64_t e = (int64_t)(bad / 2);
    int j = 0;
    TRY(read_back(h, idx + e, &j));
    if (bad % 2 == 0)
      return fail(h, 2, "hb_umap_graph: idx[%lld][%lld] = %d is not -1 or a row in 0..%lld", (long long)(e / k),
                  (long long)(e % k), j, (long long)(N - 1));
    return fail(h, 2, "hb_umap_graph: idx[%lld][%lld] = %d repeats an earlier entry of its row", (long long)(e / k),
                (long long)(e % k), j);
  }
  for (DevBuf<double>* b : {&B.rho, &B.sigma, &B.rsum, &B.rcnt}) CK(b->reserve((size_t)N));
  CK(B.uw.reserve((size_t)Nk));
  CK(B.ucnt.reserve((size_t)Nk + 1));
  CK(B.dsmall.reserve(4));
  TRY(launch(h, k_umap_sigma, dim3(grid_for(N * 32, 256, h->num_sms * 8)), dim3(256), 0, idx, dist, N, k,
             std::log2((double)n_neighbors), B.rho.p, B.sigma.p, B.rsum.p, B.rcnt.p));
  TRY(launch(h, k_sum_fixed, dim3(1), dim3(LEIDEN_SUM_THREADS), 0, (const double*)B.rsum.p, N, B.dsmall.p));
  TRY(launch(h, k_sum_fixed, dim3(1), dim3(LEIDEN_SUM_THREADS), 0, (const double*)B.rcnt.p, N, B.dsmall.p + 1));
  const dim3 grid(grid_for(Nk, 256, h->num_sms * 8)), block(256);
  TRY(launch(h, k_umap_weights, grid, block, 0, idx, dist, N, k, (const double*)B.rho.p, (const double*)B.sigma.p,
             (const double*)B.rsum.p, (const double*)B.rcnt.p, (const double*)B.dsmall.p, B.uw.p));
  TRY(launch(h, k_umap_sym<false>, grid, block, 0, idx, N, k, (const double*)B.uw.p, B.ucnt.p, (const int*)nullptr,
             (int*)nullptr, (int*)nullptr, (double*)nullptr));
  CK(cudaMemsetAsync(B.ucnt.p + Nk, 0, sizeof(int), st));
  TRY(chained_scan(h, st, B.ucnt.p, Nk + 1, 1, B.sort.scan));
  int nnz = 0;
  TRY(read_back(h, B.ucnt.p + Nk, &nnz));
  const int64_t ne = std::max(nnz, 1);
  CK(B.urow.reserve((size_t)ne));
  CK(B.ucol.reserve((size_t)ne));
  CK(B.uwv.reserve((size_t)ne));
  CK(B.key.reserve((size_t)ne));
  CK(B.eperm.reserve((size_t)ne));
  CK(B.eperm1.reserve((size_t)ne));
  CK(B.vstart.reserve((size_t)N + 1));
  TRY(launch(h, k_umap_sym<true>, grid, block, 0, idx, N, k, (const double*)B.uw.p, (int*)nullptr,
             (const int*)B.ucnt.p, B.urow.p, B.ucol.p, B.uwv.p));
  // (row, col) order, and the row starts
  CK(cudaMemcpyAsync(B.key.p, B.ucol.p, sizeof(int) * nnz, cudaMemcpyDeviceToDevice, st));
  TRY(sort_pairs(h, nnz, (int)N, B.urow.p, nullptr, B.vstart.p));
  const dim3 egrid(leiden_grid(h, ne));
  TRY(launch(h, k_indptr64, dim3(leiden_grid(h, N + 1)), block, 0, (const int*)B.vstart.p, N + 1, indptr));
  if (nnz > 0)
    TRY(launch(h, k_umap_write, egrid, block, 0, (const int*)B.eperm.p, (int64_t)nnz, (const int*)B.ucol.p,
               (const double*)B.uwv.p, indices, data));
  *nnz_out = nnz;
  CK(cudaStreamSynchronize(st));
  return 0;
}

int run_umap_graph(hb_handle* h, const int32_t* idx, int64_t idx_ld, const float* dist, int64_t dist_ld, int64_t N,
                   int k, int n_neighbors, int64_t* indptr, int32_t* indices, float* data, int64_t* nnz,
                   cudaStream_t caller) {
  if (N < 1 || N >= (1LL << 31)) return fail(h, 2, "hb_umap_graph: N = %lld rows are not supported (1 <= N < 2^31)", (long long)N);
  if (k < 1 || k > UMAP_MAX_K) return fail(h, 2, "hb_umap_graph: k = %d is not supported (1 <= k <= %d)", k, UMAP_MAX_K);
  if (idx_ld != k || dist_ld != k) return fail(h, 2, "hb_umap_graph: idx and dist must be contiguous [N][k] rows");
  if (2 * N * (int64_t)k >= (1LL << 31)) return fail(h, 2, "hb_umap_graph: 2 N k = %lld entries are not supported (< 2^31)", (long long)(2 * N * k));
  if (n_neighbors < 2) return fail(h, 2, "hb_umap_graph: n_neighbors = %d, at least 2 are needed", n_neighbors);
  if (!nnz) return fail(h, 2, "hb_umap_graph: null nnz");
  TRY(check_device_ptr(h, idx, "idx"));
  TRY(check_device_ptr(h, dist, "dist"));
  TRY(check_device_ptr(h, indptr, "indptr"));
  TRY(check_device_ptr(h, indices, "indices"));
  TRY(check_device_ptr(h, data, "data"));
  return run_score(h, caller, "umap_graph",
                   [&] { return umap_run(h, idx, dist, N, k, n_neighbors, indptr, indices, data, nnz); });
}

}  // namespace
