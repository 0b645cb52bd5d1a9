// knn_host.cuh — hb_knn (DESIGN §9): the checks, the scratch of the score calls and the launches of knn.cuh.  The
// call needs no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// The scratch of the score calls (hb_knn, hb_lisi, hb_silhouette, hb_graph_components, hb_kbet, hb_pcr, hb_kmeans), shared by them: each runs on h->stream, and a buffer
// that grows is freed only after the device has drained.  Every buffer grows on demand and is kept for the next call.
struct ScoreScratch {
  DevBuf<float> rows, query_rows, hx;  // prepared rows [n][KD] of X and of Q, |x - c|^2 / 2 (or |x|^2 / 2)
  DevBuf<double> centre;               // [KNN_MAX_D] column sums of X; pcr: its column means
  DevBuf<int> part;                    // knn, kbet: [Nq][splits][k] listed candidates
  DevBuf<int32_t> idx;                 // lisi: the neighbour lists when the caller passes no idx / dist; kbet: the lists
  DevBuf<float> dist;
  DevBuf<int> phi;                     // silhouette, kbet: [N][2] (group, label) levels
  DevBuf<int> sort_perm, inv_sort;     // silhouette, kbet: the rows sorted by (group, label); pcr: by batch
  DevBuf<int> pstart, count;           // silhouette, kbet, pcr: [J + 1] pair (batch) starts, [J] finite rows of each
  DevBuf<int4> tiles;                  // silhouette, kbet: the sweep's tiles
  DevBuf<int> sizes;                   // components: [N] rows per root
  DevBuf<unsigned long long> bad;      // components: the range pass's smallest bad entry
  DevBuf<KbetPair> kbet_pairs;         // kbet: [J] each pair's label's k0, rows, degrees of freedom and pair range
  DevBuf<double> pcr_rows;             // pcr: [J][d] each batch's column sums, then its between-batch row
  DevBuf<double> pcr_edge;             // pcr: [3][chunks][d] the head, tail and total piece of each chunk of rows
  DevBuf<int> pcr_edge_n;              // pcr: [3][chunks] their finite rows
  DevBuf<double> pcr_part, pcr_out;    // pcr: the Grams' per-CTA partials; the covariance, the scatter and n
  DevBuf<unsigned char> km_fin;        // kmeans: [N] whether each row is finite
  DevBuf<double> km_d2, km_part;       // kmeans: [N] the seeding's D^2; per-CTA partials
  DevBuf<double> km_centres;           // kmeans: [2][K][d] the current and the next centres
  DevBuf<int32_t> km_labels;           // kmeans: [2][N] this and the previous iteration's labels
  DevBuf<int> km_small;                // kmeans: the winner, the changed count, [K] counts, [K] seeds
  DevBuf<unsigned long long> km_keys;  // kmeans: [2][2 T] the race keys of two rounds
  DevBuf<unsigned long long> km_codes; // kmeans: [J] the label of each segment of the rows sorted by label
};
ScoreScratch& score_scratch(hb_handle* h) {
  if (!h->scores) h->scores.reset(new ScoreScratch());
  return *h->scores;
}

// rows -> dst [n][KD] (and hx), centred on `centre` / centre_n or normalised; with perm, row r of dst is row perm[r]
int knn_prepare(hb_handle* h, const DevRows& r, int d, int KD, bool cosine, const double* centre, double centre_n,
                float* dst, float* hx, const int* perm = nullptr) {
  const int grid = grid_for(r.n * 32, 256, h->num_sms * 16);
  with_rows(r, [&](auto p) {
    using T = std::remove_const_t<std::remove_pointer_t<decltype(p)>>;
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

// Status 2, with the message when there is a handle: the geometry hooks run the shape checks without one
template <typename... A>
int refuse(hb_handle* h, const char* fmt, A... args) { return h ? fail(h, 2, fmt, args...) : 2; }
// The search's shape limits, which hb_knn and hb_lisi (`entry`) share: fewer than 2^31 rows to search (n, named
// `what`) and 1 <= d <= KNN_MAX_D
int check_search_shape(hb_handle* h, const char* entry, const char* what, int64_t n, int d) {
  if (n >= (1LL << 31)) return refuse(h, "%s: %s = %lld rows are not supported (%s < 2^31)", entry, what, (long long)n, what);
  if (d < 1 || d > KNN_MAX_D) return refuse(h, "%s: d = %d is not supported (1 <= d <= %d)", entry, d, KNN_MAX_D);
  return 0;
}

// The eight values of the geometry hooks (hb_debug_knn_geometry, hb_debug_lisi_geometry) for a search of Nq rows
// against Nx
void knn_geometry_record(int d, int k, int64_t Nq, int64_t Nx, int num_sms, int64_t out[8]) {
  const KnnGeometry g = knn_geometry(d, k, Nq, Nx, num_sms);
  const int64_t v[8] = {g.tq, KNN_TN, g.stages, g.splits, (int64_t)g.smem, g.tiles_per_split, g.KD, 2 * g.tq};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
}

// The sweep and the merge of prepared rows, on h->stream: the k nearest of the Nx reference rows Xp (hx their halved
// squared norms) for each of the Nq query rows Qp, into idx / dist [Nq][k].  knn_search and hb_kmeans run it.
int knn_sweep(hb_handle* h, const float* Qp, int64_t Nq, const float* Xp, const float* hx, int64_t Nx, int d, int k,
              bool cosine, bool exclude_self, int32_t* idx, float* dist) {
  ScoreScratch& s = score_scratch(h);
  const KnnGeometry g = knn_geometry(d, k, Nq, Nx, h->num_sms);
  CK(s.part.reserve((size_t)Nq * g.splits * k));
  KnnArgs a;
  a.Qp = Qp;
  a.Xp = Xp;
  a.hx = hx;
  a.part_i = s.part.p;
  a.Nq = Nq;
  a.Nx = Nx;
  a.KD = g.KD;
  a.k = k;
  a.stages = g.stages;
  a.exclude_self = exclude_self;
  a.tiles_per_split = g.tiles_per_split;
  const dim3 grid((unsigned)g.qtiles, (unsigned)g.splits);
  if (k <= 64) {
    if (g.tq == 128)
      TRY(launch(h, k_knn_tc<128, 2>, grid, dim3(256), g.smem, a));
    else
      TRY(launch(h, k_knn_tc<64, 2>, grid, dim3(128), g.smem, a));
  } else {
    if (g.tq == 128)
      TRY(launch(h, k_knn_tc<128, 4>, grid, dim3(256), g.smem, a));
    else
      TRY(launch(h, k_knn_tc<64, 4>, grid, dim3(128), g.smem, a));
  }
  const int nc = g.splits * k;
  return launch(h, k_knn_merge, dim3((unsigned)((Nq + 3) / 4)), dim3(128), (size_t)4 * 2 * nc * sizeof(float), Qp, Xp,
                (const int*)s.part.p, Nq, g.KD, k, nc, (int)cosine, idx, dist);
}

// The search itself, for arguments the caller has checked, on h->stream: column sums (Euclidean), the preparation of X
// (and of Q unless it is X), the sweep and the merge into idx / dist [Nq][k].  hb_knn and hb_lisi run it.
int knn_search(hb_handle* h, const DevRows& Q, const DevRows& X, int d, int k, bool cosine, bool exclude_self,
               int32_t* idx, float* dist) {
  ScoreScratch& s = score_scratch(h);
  const int KD = (d + 7) & ~7;
  const bool shared_rows = Q.p == X.p && Q.dtype == X.dtype && Q.ld == X.ld && Q.n == X.n;  // one prepared copy serves
  CK(s.rows.reserve((size_t)X.n * KD));
  if (!shared_rows) CK(s.query_rows.reserve((size_t)Q.n * KD));
  CK(s.hx.reserve((size_t)X.n));
  CK(s.centre.reserve((size_t)KNN_MAX_D));

  TRY(prepare_centred(h, X, d, KD, cosine, s.centre.p, s.rows.p, s.hx.p));
  const float* Qp = s.rows.p;
  if (!shared_rows) {
    TRY(knn_prepare(h, Q, d, KD, cosine, cosine ? nullptr : s.centre.p, (double)X.n, s.query_rows.p, nullptr));
    Qp = s.query_rows.p;
  }
  return knn_sweep(h, Qp, Q.n, s.rows.p, s.hx.p, X.n, d, k, cosine, exclude_self, idx, dist);
}

int run_knn(hb_handle* h, const DevRows& Q, const DevRows& X, int d, int k, int metric, bool exclude_self, int32_t* idx,
            float* dist, cudaStream_t caller) {
  if (Q.n < 1 || X.n < 1) return fail(h, 2, "hb_knn needs at least one query row and one reference row");
  TRY(check_search_shape(h, "hb_knn", "Nx", X.n, d));
  if (k < 1 || k > KNN_MAX_K) return fail(h, 2, "hb_knn: k = %d is not supported (1 <= k <= %d)", k, KNN_MAX_K);
  if (k > X.n - (exclude_self ? 1 : 0))
    return fail(h, 2, "hb_knn: k = %d exceeds the %lld candidate rows of a query row", k, (long long)(X.n - (exclude_self ? 1 : 0)));
  if (metric != HB_EUCLIDEAN && metric != HB_COSINE) return fail(h, 2, "hb_knn: unknown metric %d", metric);
  TRY(check_rows(h, Q, d, "Q"));
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, idx, "idx"));
  if (dist) TRY(check_device_ptr(h, dist, "dist"));
  CK(cudaSetDevice(h->device));
  return on_caller_stream(h, caller, [&] {
    RegionScope rs(h, "knn");
    return knn_search(h, Q, X, d, k, metric == HB_COSINE, exclude_self, idx, dist);
  });
}

}  // namespace
