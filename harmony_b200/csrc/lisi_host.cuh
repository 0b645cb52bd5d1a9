// lisi_host.cuh — hb_lisi (DESIGN §10): the checks and the launches: knn_search (knn_host.cuh) for each row's
// floor(3 p) - 1 nearest other rows, then k_lisi.  The call needs no setup and touches no state of a Harmony run or a
// mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// The neighbours LISI weighs at perplexity p: floor(3 p) - 1 (the package searches 3 p rows with the cell itself and
// drops the first), 0 for a p that is not finite or below 1, KNN_SWEEP_MAX_K + 1 for any k above the sweep's limit.
int lisi_k(double p) {
  if (!(p >= 1.0) || !std::isfinite(p)) return 0;
  const double k = std::floor(3.0 * p) - 1.0;
  return k > KNN_SWEEP_MAX_K ? KNN_SWEEP_MAX_K + 1 : (int)k;
}

// The refusals hb_lisi and hb_debug_lisi_geometry share; h may be null (no message).
int lisi_check_shape(hb_handle* h, int d, double p, int64_t N, int* k_out) {
  const int k = lisi_k(p);
  if (k == 0) return refuse(h, "hb_lisi: perplexity %g is not supported (a finite p >= 1)", p);
  if (k > KNN_SWEEP_MAX_K) return refuse(h, "hb_lisi: perplexity %g needs more than %d neighbours (p < 43 1/3)", p, KNN_SWEEP_MAX_K);
  if (k > N - 1) return refuse(h, "hb_lisi: perplexity %g needs k = %d neighbours, N = %lld rows have %lld", p, k, (long long)N, (long long)(N - 1));
  TRY(check_search_shape(h, "hb_lisi", "N", N, d));  // N >= 2^31 passes the check above: the refusals keep their order
  *k_out = k;
  return 0;
}

int run_lisi(hb_handle* h, const DevRows& X, int d, const int32_t* labels, int64_t labels_ld, int n_sets, double p,
             double* lisi, int32_t* idx, float* dist, cudaStream_t caller) {
  int k = 0;
  TRY(lisi_check_shape(h, d, p, X.n, &k));
  if (n_sets < 1) return fail(h, 2, "hb_lisi: n_sets = %d, at least one label set is needed", n_sets);
  if (labels_ld < X.n) return fail(h, 2, "hb_lisi: label stride %lld is smaller than N = %lld", (long long)labels_ld, (long long)X.n);
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, labels, "labels"));
  TRY(check_device_ptr(h, lisi, "lisi"));
  if (idx) TRY(check_device_ptr(h, idx, "idx"));
  if (dist) TRY(check_device_ptr(h, dist, "dist"));
  return run_score(h, caller, "lisi", [&] {
    ScoreScratch& s = score_scratch(h);
    if (!idx) {
      CK(s.idx.reserve((size_t)X.n * k));
      idx = s.idx.p;
    }
    if (!dist) {
      CK(s.dist.reserve((size_t)X.n * k));
      dist = s.dist.p;
    }
    TRY(knn_search(h, X, X, d, k, false, true, idx, dist));
    return launch(h, k_lisi, dim3((unsigned)((X.n + LISI_WARPS - 1) / LISI_WARPS)), dim3(32 * LISI_WARPS), 0,
                  (const int32_t*)idx, (const float*)dist, X.n, k, labels, labels_ld, n_sets, std::log(p), lisi);
  });
}

}  // namespace
