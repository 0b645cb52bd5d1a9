// score_host.cuh — what the score calls (hb_knn, hb_lisi, hb_silhouette, hb_graph_components, hb_kbet, hb_pcr,
// hb_kmeans, hb_umap_graph,
// hb_leiden; DESIGN §9-§16) share on the host: their scratch, their shape refusals, the read-back of their read-only
// checks, the sorted indexes and sums they build, the preparation and sweep of knn.cuh, and the way each call is
// ordered on the caller's stream.  Included by harmony_b200.cu before the calls' own *_host.cuh.
#pragma once

namespace {

// The buffers of hb_umap_graph and hb_leiden (DESIGN §16), which run alone
// The level graph: n vertices, nnz entries, row starts, columns, fp64 weights, each entry's row, degrees
struct LeidenGraph {
  int n = 0, nnz = 0;
  DevBuf<int> ip, col, row;
  DevBuf<double> w, deg;
  int reserve(hb_handle* h, int n_, int nnz_) {
    n = n_;
    nnz = nnz_;
    CK(ip.reserve((size_t)n + 1));
    CK(col.reserve((size_t)std::max(nnz, 1)));
    CK(row.reserve((size_t)std::max(nnz, 1)));
    CK(w.reserve((size_t)std::max(nnz, 1)));
    CK(deg.reserve((size_t)std::max(n, 1)));
    return 0;
  }
};

template <typename T>
void swap_bufs(DevBuf<T>& a, DevBuf<T>& b) {
  std::swap(a.p, b.p);
  std::swap(a.n, b.n);
}
struct LeidenBufs {
  LeidenGraph g0, level[2];                    // the caller's graph, and the aggregated levels in turn
  DevBuf<int> key;                              // the sort keys
  SortScratch sort;                             // every sort's scratch, and the chain state of the call's scans
  DevBuf<int> eperm, eperm1;                    // entries sorted by (row, code of the column), and the first pass
  DevBuf<int> vperm, vstart;                    // vertices sorted by a code, and the code starts [n + 1]
  DevBuf<int> comm, next, sub, target, proposed;  // the partition, the sweep's result, sub-communities, proposals
  DevBuf<int> newid, cmin, vmap, omap, lab;     // aggregation: ids, the next start partition, level and row maps
  DevBuf<int> head, seg_start, size, first, small;  // pair heads and starts; community sizes and first members
  DevBuf<double> tot, ext, win, sub_tot, sub_ext, dsmall;  // community and sub-community sums
  DevBuf<double> rho, sigma, rsum, rcnt, uw, uwv;  // umap: per-row rho, sigma, distance sums; [N][k] and emitted weights
  DevBuf<int> ucnt, urow, ucol;                 // umap: emitted entries per listed entry, their rows and columns
};

// The scratch of the score calls, shared by them: each runs on h->stream, and a buffer that grows is freed only after
// the device has drained.  Every buffer grows on demand and is kept for the next call.  Buffers that no one call uses
// together are one (DESIGN §9): count, keys, idx, stats and cta_part.
struct ScoreScratch {
  DevBuf<float> rows, query_rows, hx;  // prepared rows [n][KD] of X and of Q (kmeans: of the centres), |x - c|^2 / 2
  DevBuf<double> centre;               // [KNN_MAX_D] column sums of X, or its column means (pcr, kmeans: and n)
  DevBuf<int> part;                    // knn, kbet: [Nq][splits][k] listed candidates
  DevBuf<int32_t> idx;                 // lisi, kbet: [N][k] neighbour lists; kmeans: [2][N] this and the previous labels
  DevBuf<float> dist;                  // lisi: [N][k] the distances when the caller passes none
  DevBuf<int> phi;                     // silhouette, kbet: [N][2] (group, label) levels; kmeans: [N] sort codes
  DevBuf<int> sort_perm, inv_sort;     // the rows sorted by pair (silhouette, kbet) or by code (pcr, kmeans)
  DevBuf<int> pstart;                  // [J + 1] each pair's or segment's first sorted row
  DevBuf<int> count;                   // [J] finite rows of each pair or segment; components: [N] rows per root
  DevBuf<int4> tiles;                  // silhouette, kbet: the sweep's tiles
  DevBuf<unsigned long long> keys;     // run_check: the smallest bad word; kmeans: [2][2 T] race keys
  DevBuf<KbetPair> pairs;              // kbet: [J] each pair's label's k0, rows, degrees of freedom and pair range
  DevBuf<double> seg_sums;             // pcr, kmeans: [J][d] each segment's column sums, then its combined row
  DevBuf<double> chunk_edge;           // pcr, kmeans: [3][chunks][d] the head, tail and total piece of each chunk
  DevBuf<int> chunk_n;                 // pcr, kmeans: [3][chunks] their finite rows; kmeans: per-CTA finite rows
  DevBuf<double> cta_part;             // pcr, kmeans: per-CTA fp64 partials
  DevBuf<double> stats;                // pcr: the covariance, the scatter and n; kmeans: [2][K][d] this and next centres
  DevBuf<unsigned char> finite;        // kmeans: [N] whether each row is finite
  DevBuf<double> d2;                   // kmeans: [N] the seeding's D^2
  DevBuf<int> small;                   // kmeans: the winner, the changed count, [K] counts, [K] seeds
  DevBuf<unsigned long long> seg_codes;  // kmeans: [J] the code of each segment of the sorted rows
  LeidenBufs leiden;                   // umap_graph, leiden
};
ScoreScratch& score_scratch(hb_handle* h) {
  if (!h->scores) h->scores.reset(new ScoreScratch());
  return *h->scores;
}

// work() as the score call timed under `region`: on the handle's device, on h->stream after the work queued on
// `caller` so far and before the work queued there next
template <typename F>
int run_score(hb_handle* h, cudaStream_t caller, const char* region, F&& work) {
  CK(cudaSetDevice(h->device));
  return on_caller_stream(h, caller, [&] {
    RegionScope rs(h, region);
    return work();
  });
}

// *out = *p, read once h->stream has drained
template <typename T>
int read_back(hb_handle* h, const T* p, T* out) {
  CK(cudaMemcpyAsync(out, p, sizeof(T), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}
// A read-only check on h->stream: `check` over `grid` x 256 threads with args and then s.keys, filled with ~0 first,
// where it leaves the smallest bad word it finds.  *bad: that word (~0: none).
template <typename... P, typename... A>
int run_check(hb_handle* h, unsigned long long* bad, void (*check)(P...), dim3 grid, const A&... args) {
  ScoreScratch& s = score_scratch(h);
  CK(s.keys.reserve(1));
  CK(cudaMemsetAsync(s.keys.p, 0xff, sizeof(unsigned long long), h->stream));
  TRY(launch(h, check, grid, dim3(256), 0, args..., s.keys.p));
  return read_back(h, s.keys.p, bad);
}

// Status 2, with the message when there is a handle: the geometry hooks run the shape checks without one
template <typename... A>
int refuse(hb_handle* h, const char* fmt, A... args) { return h ? fail(h, 2, fmt, args...) : 2; }
// The search's shape limits, which the calls on an embedding (`entry`) share: fewer than 2^31 rows to search (n, named
// `what`) and 1 <= d <= KNN_MAX_D
int check_search_shape(hb_handle* h, const char* entry, const char* what, int64_t n, int d) {
  if (n >= (1LL << 31)) return refuse(h, "%s: %s = %lld rows are not supported (%s < 2^31)", entry, what, (long long)n, what);
  if (d < 1 || d > KNN_MAX_D) return refuse(h, "%s: d = %d is not supported (1 <= d <= %d)", entry, d, KNN_MAX_D);
  return 0;
}
// The same for hb_silhouette, hb_kbet and hb_pcr, which also need two rows
int check_score_shape(hb_handle* h, const char* entry, int64_t N, int d) {
  if (N < 2) return refuse(h, "%s: N = %lld rows, at least 2 are needed", entry, (long long)N);
  return check_search_shape(h, entry, "N", N, d);
}

// The eight values of the geometry hooks (hb_debug_knn_geometry, hb_debug_lisi_geometry) for a search of Nq rows
// against Nx
void knn_geometry_record(int d, int k, int64_t Nq, int64_t Nx, int num_sms, int64_t out[8]) {
  const KnnGeometry g = knn_geometry(d, k, Nq, Nx, num_sms);
  const int64_t v[8] = {g.tq, KNN_TN, g.stages, g.splits, (int64_t)g.smem, g.tiles_per_split, g.KD, 2 * g.tq};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
}

// rows -> dst [n][KD] (and hx), centred on `centre` / centre_n or normalised; with perm, row r of dst is row perm[r]
int knn_prepare(hb_handle* h, const DevRows& r, int d, int KD, bool cosine, const double* centre, double centre_n,
                float* dst, float* hx, const int* perm = nullptr) {
  const int grid = grid_for(r.n * 32, 256, h->num_sms * 16);
  with_rows(r, [&](auto p) {
    using T = row_t<decltype(p)>;
    if (perm)
      k_knn_prepare<T, true><<<grid, 256, 0, h->stream>>>(p, r.ld, r.n, d, KD, (int)cosine, centre, centre_n, dst, hx, perm);
    else
      k_knn_prepare<T, false><<<grid, 256, 0, h->stream>>>(p, r.ld, r.n, d, KD, (int)cosine, centre, centre_n, dst, hx, nullptr);
  });
  CKL();
  return 0;
}

// X's rows -> dst (and hx), optionally through perm: centred on X's column means, whose sums go to `centre`
// (Euclidean), or normalised (cosine, centre unused)
int prepare_centred(hb_handle* h, const DevRows& X, int d, int KD, bool cosine, double* centre, float* dst, float* hx,
                    const int* perm = nullptr) {
  if (!cosine) {
    CK(cudaMemsetAsync(centre, 0, sizeof(double) * KNN_MAX_D, h->stream));
    const int grid = grid_for(X.n, 2, h->num_sms * 8);
    with_rows(X, [&](auto x) { k_knn_colsum<<<grid, 256, 0, h->stream>>>(x, X.ld, X.n, d, centre); });
    CKL();
  }
  return knn_prepare(h, X, d, KD, cosine, cosine ? nullptr : centre, (double)X.n, dst, hx, perm);
}

// k_knn_tc over `grid` at the geometry's query tile and list width (E = 2 up to k = 64, else 4); KnnGroupArgs select
// the grouped sweep over a.tiles
template <typename Args>
int launch_knn_tc(hb_handle* h, const KnnGeometry& g, int k, dim3 grid, const Args& a) {
  constexpr bool GROUPED = std::is_same<Args, KnnGroupArgs>::value;
  if (k <= 64) {
    if (g.tq == 128) return launch(h, k_knn_tc<128, 2, GROUPED>, grid, dim3(256), g.smem, a);
    return launch(h, k_knn_tc<64, 2, GROUPED>, grid, dim3(128), g.smem, a);
  }
  if (g.tq == 128) return launch(h, k_knn_tc<128, 4, GROUPED>, grid, dim3(256), g.smem, a);
  return launch(h, k_knn_tc<64, 4, GROUPED>, grid, dim3(128), g.smem, a);
}

// The sweep and the merge of prepared rows, on h->stream: the k nearest of the Nx reference rows Xp (hx their halved
// squared norms) for each of the Nq query rows Qp, into idx / dist [Nq][k].  knn_search and hb_kmeans run it.
int knn_sweep(hb_handle* h, const float* Qp, int64_t Nq, const float* Xp, const float* hx, int64_t Nx, int d, int k,
              bool cosine, bool exclude_self, int32_t* idx, float* dist) {
  ScoreScratch& s = score_scratch(h);
  const KnnGeometry g = knn_geometry(d, k, Nq, Nx, h->num_sms);
  CK(s.part.reserve((size_t)Nq * g.splits * k));
  const KnnArgs a{Qp, Xp, hx, s.part.p, Nq, Nx, g.KD, k, g.stages, exclude_self, g.tiles_per_split};
  TRY(launch_knn_tc(h, g, k, dim3((unsigned)g.qtiles, (unsigned)g.splits), a));
  const int nc = g.splits * k;
  return launch(h, k_knn_merge, dim3((unsigned)((Nq + 3) / 4)), dim3(128), (size_t)4 * 2 * nc * sizeof(float), Qp, Xp,
                (const int*)s.part.p, Nq, g.KD, k, nc, (int)cosine, idx, dist);
}

// The index of the (major, minor) code pairs of X's rows (hb_silhouette: (group, label); hb_kbet: (label, batch)),
// on h->stream: the rows sorted by pair (s.sort_perm) into ti, the pair starts (s.pstart), the rows in sorted order
// centred and prepared into s.rows / s.hx, and the finite rows of each pair (s.count).  names: the major's and the
// minor's in a code's refusal.
int pair_index(hb_handle* h, const DevRows& X, int d, int KD, const int32_t* major, int n_major, const int32_t* minor,
               int n_minor, const char* const names[2], TupleIndex& ti) {
  ScoreScratch& s = score_scratch(h);
  const int64_t N = X.n;
  const cudaStream_t st = h->stream;
  CK(s.phi.reserve(2 * (size_t)N));
  CK(s.rows.reserve((size_t)N * KD));
  CK(s.hx.reserve((size_t)N));
  CK(s.centre.reserve((size_t)KNN_MAX_D));
  k_silhouette_phi<<<grid_for(N, 256, h->num_sms * 8), 256, 0, st>>>(minor, major, N, n_minor, n_major, s.phi.p);
  CKL();
  TupleKeys keys;
  TRY(tuple_keys(h, {n_major, n_minor}, keys));
  TRY(build_tuple_index(h, s.phi.p, N, keys, false, s.sort_perm, s.inv_sort, ti, names));
  const int J = (int)ti.uniq.size();
  CK(s.pstart.reserve((size_t)J + 1));
  CK(s.count.reserve((size_t)J));
  TRY(upload_vector(h, s.pstart, std::vector<int>(ti.tstart.begin(), ti.tstart.end())));
  CK(cudaMemsetAsync(s.count.p, 0, sizeof(int) * J, st));
  TRY(prepare_centred(h, X, d, KD, false, s.centre.p, s.rows.p, s.hx.p, s.sort_perm.p));
  k_silhouette_count<<<grid_for(N, 256, h->num_sms * 8), 256, 0, st>>>(s.hx.p, N, s.pstart.p, J, s.count.p);
  CKL();
  return 0;
}

// The column sums of X's rows in the segments of one code (device [N], codes 0..n_codes - 1; `name` the code's in a
// refusal), on h->stream: the rows sorted by code (s.sort_perm) into ti, the segment starts (s.pstart), then
// k_pcr_sums into s.seg_sums, s.count and the chunk pieces.  `a` holds the arguments for k_pcr_combine / k_kms_means.
int segment_sums(hb_handle* h, const DevRows& X, int d, const int32_t* codes, int n_codes, const char* name,
                 TupleIndex& ti, PcrSumArgs& a) {
  ScoreScratch& s = score_scratch(h);
  const int64_t N = X.n;
  TupleKeys keys;
  TRY(tuple_keys(h, {n_codes}, keys));
  const char* const names[1] = {name};
  TRY(build_tuple_index(h, codes, N, keys, false, s.sort_perm, s.inv_sort, ti, names));
  const int J = (int)ti.uniq.size();
  const int64_t chunks = (N + PCR_CHUNK - 1) / PCR_CHUNK;
  CK(s.pstart.reserve((size_t)J + 1));
  CK(s.count.reserve((size_t)J));
  CK(s.seg_sums.reserve((size_t)J * d));
  CK(s.chunk_edge.reserve((size_t)3 * chunks * d));
  CK(s.chunk_n.reserve((size_t)3 * chunks));
  TRY(upload_vector(h, s.pstart, std::vector<int>(ti.tstart.begin(), ti.tstart.end())));
  a = PcrSumArgs{X.ld, N, d, J, chunks, s.sort_perm.p, s.pstart.p, s.seg_sums.p, s.count.p, s.chunk_edge.p, s.chunk_n.p};
  const dim3 gs((unsigned)((chunks + PCR_WARPS - 1) / PCR_WARPS));
  return with_rows(X, [&](auto x) { return launch(h, k_pcr_sums<row_t<decltype(x)>>, gs, dim3(32 * PCR_WARPS), 0, a, x); });
}

}  // namespace
