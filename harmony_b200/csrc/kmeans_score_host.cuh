// kmeans_score_host.cuh — hb_kmeans (DESIGN §15): the checks and launches of kmeans_score.cuh, the §9 sweep as the
// assignment step, setup's tuple index and hb_pcr's segment sums as the means, and sklearn's Lloyd stopping rule on
// the host.  The call needs no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// candidates per seeding round: sklearn's greedy k-means++, 2 + floor(ln K)
int kmeans_trials(int K) { return 2 + (int)std::floor(std::log((double)K)); }

// contiguous row ranges of k_kms_colsum / k_kms_sqdist: at most 4 CTAs per SM
struct KmsRanges {
  int ctas = 1;
  int64_t rows = 1;
};
KmsRanges kms_ranges(int64_t N, int num_sms) {
  KmsRanges r;
  const int64_t cap = 4 * (int64_t)num_sms;
  r.rows = std::max<int64_t>(KMS_WARPS, (N + cap - 1) / cap);
  r.ctas = (int)std::max<int64_t>(1, (N + r.rows - 1) / r.rows);
  return r;
}

struct KmeansRun {
  hb_handle* h;
  const DevRows& X;
  int d, K, KD, T;
  int64_t N;
  KmsRanges ranges;
  int seed_grid;
  double n_fin = 0.0, tol_abs = 0.0;
};

// sum over CTAs of k_kms_sqdist, in CTA order on the host; with far, also whether a row exceeds KMS_MAX_SQ
int kms_sqdist(KmeansRun& r, const int32_t* labels, const double* centres, double* out, int* far = nullptr) {
  hb_handle* h = r.h;
  ScoreScratch& s = score_scratch(h);
  int* far_d = far ? s.small.p + 1 : nullptr;
  if (far_d) CK(cudaMemsetAsync(far_d, 0, sizeof(int), h->stream));
  TRY(with_rows(r.X, [&](auto x) {
    return launch(h, k_kms_sqdist<row_t<decltype(x)>>, dim3((unsigned)r.ranges.ctas),
                  dim3(32 * KMS_WARPS), 0, x, r.X.ld, r.N, r.d, r.ranges.rows, (const unsigned char*)s.finite.p, labels,
                  centres, s.cta_part.p, far_d);
  }));
  std::vector<double> part(r.ranges.ctas);
  CK(cudaMemcpyAsync(part.data(), s.cta_part.p, sizeof(double) * part.size(), cudaMemcpyDeviceToHost, h->stream));
  if (far) CK(cudaMemcpyAsync(far, far_d, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  double t = 0.0;
  for (double v : part) t += v;
  *out = t;
  return 0;
}

// The column mean of the finite rows into s.centre, their count, the tolerance, and the prepared rows.  Status 3 for
// fewer than K finite rows; status 2 for a finite row too far from the mean for the fp32 assignment.
int kms_prepare(KmeansRun& r, double tol) {
  hb_handle* h = r.h;
  ScoreScratch& s = score_scratch(h);
  const int ctas = r.ranges.ctas;
  CK(s.cta_part.reserve(std::max<size_t>((size_t)ctas * r.d + 1, (size_t)r.seed_grid * KMS_MAX_T)));
  CK(s.chunk_n.reserve((size_t)ctas));
  CK(s.centre.reserve((size_t)KNN_MAX_D + 1));
  TRY(with_rows(r.X, [&](auto x) {
    return launch(h, k_kms_colsum<row_t<decltype(x)>>, dim3((unsigned)ctas),
                  dim3(32 * KMS_WARPS), 0, x, r.X.ld, r.N, r.d, r.ranges.rows, s.cta_part.p, s.chunk_n.p, s.finite.p);
  }));
  double* n_out = s.centre.p + KNN_MAX_D;
  TRY(launch(h, k_pcr_mean, dim3((unsigned)r.d), dim3(256), 0, (const double*)s.cta_part.p, (const int*)s.chunk_n.p,
             (int64_t)ctas, r.d, s.centre.p, n_out));
  CK(cudaMemcpyAsync(&r.n_fin, n_out, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (r.n_fin < r.K)
    return fail(h, 3, "hb_kmeans: %.0f finite rows, fewer than the K = %d clusters", r.n_fin, r.K);
  double total = 0.0;
  int far = 0;
  TRY(kms_sqdist(r, nullptr, s.centre.p, &total, &far));
  if (far)
    return fail(h, 2, "hb_kmeans: a finite row lies beyond |x - m|^2 = 2^124 of the column mean m, outside the fp32 "
                      "range of the assignment");
  r.tol_abs = tol * total / (r.n_fin * r.d);  // sklearn's _tolerance: tol times the mean column variance (ddof 0)
  return knn_prepare(h, r.X, r.d, r.KD, false, s.centre.p, 1.0, s.rows.p, nullptr);
}

// Greedy k-means++ of init `init` into seeds (device [K]); ends with the seeds' caller rows in `centres`
int kms_seed(KmeansRun& r, uint64_t seed, int init, int32_t* seeds, double* centres) {
  hb_handle* h = r.h;
  RegionScope rs(h, "kmeans_seed");
  ScoreScratch& s = score_scratch(h);
  const int T = r.T;
  int* winner = s.small.p;
  unsigned long long* keys[2] = {s.keys.p, s.keys.p + 2 * T};
  const KmsSeedArgs a{s.rows.p, s.finite.p, s.d2.p, r.N, r.KD, T, kmeans_score_key(seed, (uint64_t)init)};
  const dim3 grid((unsigned)r.seed_grid), block(32 * KMS_WARPS);
  CK(cudaMemsetAsync(s.keys.p, 0xff, sizeof(unsigned long long) * 4 * T, h->stream));
  TRY(launch(h, k_kms_update, grid, block, 0, a, (const int*)nullptr, 0, keys[0]));
  for (int round = 0; round < r.K; ++round) {
    unsigned long long* cur = keys[round & 1];
    if (round > 0) TRY(launch(h, k_kms_potential, grid, block, 0, a, (const unsigned long long*)cur, s.cta_part.p));
    TRY(launch(h, k_kms_pick, dim3(1), dim3(32), 0, (const double*)s.cta_part.p, r.seed_grid, T,
               (const unsigned long long*)cur, round, seeds, winner, keys[(round + 1) & 1]));
    if (round + 1 < r.K) TRY(launch(h, k_kms_update, grid, block, 0, a, (const int*)winner, round + 1, keys[(round + 1) & 1]));
  }
  return with_rows(r.X, [&](auto x) {
    return launch(h, k_kms_gather<row_t<decltype(x)>>,
                  dim3((unsigned)grid_for((int64_t)r.K * r.d, 256, h->num_sms * 4)), dim3(256), 0, x, r.X.ld, r.d,
                  (const int32_t*)seeds, r.K, centres);
  });
}

// labels <- the nearest of the centres (device [K][d] fp64) for every finite row, -1 for the others; s.phi <- the
// sort codes; *changed (device) += the rows whose label differs from old
int kms_assign(KmeansRun& r, const double* centres, int32_t* labels, const int32_t* old, int* changed) {
  hb_handle* h = r.h;
  ScoreScratch& s = score_scratch(h);
  const DevRows C{centres, HB_FLOAT64, r.d, r.K};
  TRY(knn_prepare(h, C, r.d, r.KD, false, s.centre.p, 1.0, s.query_rows.p, s.hx.p));
  TRY(knn_sweep(h, s.rows.p, r.N, s.query_rows.p, s.hx.p, r.K, r.d, 1, false, false, labels, nullptr));
  return launch(h, k_kms_labels, dim3((unsigned)grid_for(r.N, 32 * KMS_WARPS, h->num_sms * 4)), dim3(32 * KMS_WARPS), 0,
                labels, old, (const unsigned char*)s.finite.p, r.N, r.K, s.phi.p, changed);
}

// next <- the means of the labels' members (from a copy of cur: an empty cluster keeps its centre)
int kms_means(KmeansRun& r, const double* cur, double* next) {
  hb_handle* h = r.h;
  ScoreScratch& s = score_scratch(h);
  TupleIndex ti;
  PcrSumArgs a;
  TRY(segment_sums(h, r.X, r.d, s.phi.p, r.K + 1, "hb_kmeans: labels", ti, a));
  CK(s.seg_codes.reserve((size_t)a.J));
  TRY(upload_vector(h, s.seg_codes, std::vector<unsigned long long>(ti.uniq.begin(), ti.uniq.end())));
  CK(cudaMemcpyAsync(next, cur, sizeof(double) * r.K * r.d, cudaMemcpyDeviceToDevice, h->stream));
  return launch(h, k_kms_means, dim3((unsigned)((a.J + PCR_WARPS - 1) / PCR_WARPS)), dim3(32 * PCR_WARPS), 0, a,
                (const unsigned long long*)s.seg_codes.p, r.K, next, s.small.p + 2);
}

// One init: seeds, Lloyd, the final assignment; labels and centres into the scratch, inertia and n_iter out
int kms_init(KmeansRun& r, uint64_t seed, int init, int max_iter, int32_t** labels_out, double** centres_out,
             double* inertia, int* n_iter) {
  hb_handle* h = r.h;
  ScoreScratch& s = score_scratch(h);
  const size_t Kd = (size_t)r.K * r.d;
  double* cen[2] = {s.stats.p, s.stats.p + Kd};
  int32_t* lab[2] = {s.idx.p, s.idx.p + r.N};
  int32_t* seeds = s.small.p + 2 + r.K;
  int* changed = s.small.p + 1;
  TRY(kms_seed(r, seed, init, seeds, cen[0]));
  CK(cudaMemsetAsync(lab[1], 0xff, sizeof(int32_t) * r.N, h->stream));  // the previous labels of iteration 1: none
  std::vector<double> c_old(Kd), c_new(Kd);
  CK(cudaMemcpyAsync(c_old.data(), cen[0], sizeof(double) * Kd, cudaMemcpyDeviceToHost, h->stream));
  bool strict = false;
  int it = 0;
  for (int i = 0; i < max_iter; ++i) {
    CK(cudaMemsetAsync(changed, 0, sizeof(int), h->stream));
    TRY(kms_assign(r, cen[0], lab[0], lab[1], changed));
    TRY(kms_means(r, cen[0], cen[1]));
    int ch = 0;
    CK(cudaMemcpyAsync(c_new.data(), cen[1], sizeof(double) * Kd, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&ch, changed, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    double shift = 0.0;
    for (size_t e = 0; e < Kd; ++e) shift += (c_new[e] - c_old[e]) * (c_new[e] - c_old[e]);
    std::swap(cen[0], cen[1]);
    std::swap(c_old, c_new);
    it = i + 1;
    if (ch == 0) {  // the labels did not change: strict convergence
      strict = true;
      break;
    }
    if (shift <= r.tol_abs) break;
    std::swap(lab[0], lab[1]);
  }
  if (!strict) {  // the labels of the final centres
    CK(cudaMemsetAsync(changed, 0, sizeof(int), h->stream));
    TRY(kms_assign(r, cen[0], lab[0], lab[1], changed));
  }
  TRY(kms_sqdist(r, lab[0], cen[0], inertia));
  *n_iter = it;
  *labels_out = lab[0];
  *centres_out = cen[0];
  return 0;
}

// The whole call on h->stream, for arguments the caller has checked
int kmeans_run(hb_handle* h, const DevRows& X, int d, int K, uint64_t seed, int n_init, int max_iter, double tol,
               int32_t* labels, double* centres, double* inertia, int32_t* n_iter, int32_t* seeds) {
  ScoreScratch& s = score_scratch(h);
  KmeansRun r{h, X, d, K, (d + 7) & ~7, kmeans_trials(K), X.n};
  r.ranges = kms_ranges(X.n, h->num_sms);
  r.seed_grid = grid_for(X.n * KMS_GROUP, 32 * KMS_WARPS, h->num_sms * 8);  // KMS_GROUP lanes per row
  CK(s.finite.reserve((size_t)X.n));
  CK(s.rows.reserve((size_t)X.n * r.KD));
  CK(s.query_rows.reserve((size_t)K * r.KD));
  CK(s.hx.reserve((size_t)K));
  CK(s.d2.reserve((size_t)X.n));
  CK(s.stats.reserve((size_t)2 * K * d));
  CK(s.idx.reserve((size_t)2 * X.n));
  CK(s.small.reserve((size_t)2 + 2 * K));
  CK(s.keys.reserve((size_t)4 * KMS_MAX_T));
  CK(s.phi.reserve((size_t)X.n));
  TRY(kms_prepare(r, tol));
  std::vector<double> inertia_h(n_init);
  std::vector<int32_t> n_iter_h(n_init);
  for (int init = 0; init < n_init; ++init) {
    int32_t* lab;
    double* cen;
    TRY(kms_init(r, seed, init, max_iter, &lab, &cen, &inertia_h[init], &n_iter_h[init]));
    if (seeds)
      CK(cudaMemcpyAsync(seeds + (size_t)init * K, s.small.p + 2 + K, sizeof(int32_t) * K, cudaMemcpyDeviceToDevice,
                         h->stream));
    bool best = true;  // the lowest inertia, the earliest init on a tie
    for (int j = 0; j < init; ++j) best &= inertia_h[init] < inertia_h[j];
    if (best) {
      CK(cudaMemcpyAsync(labels, lab, sizeof(int32_t) * X.n, cudaMemcpyDeviceToDevice, h->stream));
      CK(cudaMemcpyAsync(centres, cen, sizeof(double) * K * d, cudaMemcpyDeviceToDevice, h->stream));
    }
  }
  CK(cudaMemcpyAsync(inertia, inertia_h.data(), sizeof(double) * n_init, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(n_iter, n_iter_h.data(), sizeof(int32_t) * n_init, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));  // the host vectors go on return
  return 0;
}

int run_kmeans(hb_handle* h, const DevRows& X, int d, int K, uint64_t seed, int n_init, int max_iter, double tol,
               int32_t* labels, double* centres, double* inertia, int32_t* n_iter, int32_t* seeds, cudaStream_t caller) {
  if (X.n < 1) return fail(h, 2, "hb_kmeans: N = %lld rows, at least 1 is needed", (long long)X.n);
  TRY(check_search_shape(h, "hb_kmeans", "N", X.n, d));
  if (K < 1 || K > KMS_MAX_K || K > X.n)
    return fail(h, 2, "hb_kmeans: K = %d is not supported (1 <= K <= min(N, %d))", K, KMS_MAX_K);
  if (n_init < 1) return fail(h, 2, "hb_kmeans: n_init = %d, at least one init is needed", n_init);
  if (max_iter < 0) return fail(h, 2, "hb_kmeans: max_iter = %d is negative", max_iter);
  if (!(tol >= 0.0) || !std::isfinite(tol)) return fail(h, 2, "hb_kmeans: tol = %g must be finite and >= 0", tol);
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, labels, "labels"));
  TRY(check_device_ptr(h, centres, "centres"));
  TRY(check_device_ptr(h, inertia, "inertia"));
  TRY(check_device_ptr(h, n_iter, "n_iter"));
  if (seeds) TRY(check_device_ptr(h, seeds, "seeds"));
  return run_score(h, caller, "kmeans", [&] {
    return kmeans_run(h, X, d, K, seed, n_init, max_iter, tol, labels, centres, inertia, n_iter, seeds);
  });
}

}  // namespace
