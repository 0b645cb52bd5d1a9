// knn_host.cuh — hb_knn (DESIGN §9): the checks and the search, from the preparation and sweep of score_host.cuh.  The
// call needs no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

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
  return run_score(h, caller, "knn",
                   [&] { return knn_search(h, Q, X, d, k, metric == HB_COSINE, exclude_self, idx, dist); });
}

}  // namespace
