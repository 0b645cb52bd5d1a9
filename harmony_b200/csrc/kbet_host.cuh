// kbet_host.cuh — hb_kbet (DESIGN §13): the checks and the launches: hb_silhouette's (label, batch) index, sorted
// preparation and finite counts (pair_index, score_host.cuh), the k0 of each label on the host, k_knn_tc's grouped sweep
// over the tested labels' tiles, k_knn_merge and k_kbet.  The call needs no setup and touches no state of a Harmony run
// or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// The size of a label's tests from its n finite rows in `present` batches: 0 (not tested) for fewer than 10 rows or
// one batch; else the fixed k0, 0 when it exceeds n; else scib's min(70, max(10, floor(mean / 4))) with the mean n /
// present over the batches with rows, lowered to floor((2^31 - 1) / n) where k0 n would reach 2^31 - 1.
int kbet_k0(int64_t n, int present, int fixed_k0) {
  if (n < 10 || present < 2) return 0;
  if (fixed_k0) return fixed_k0 <= n ? fixed_k0 : 0;
  int64_t k0 = std::min<int64_t>(70, std::max<int64_t>(10, (int64_t)std::floor((double)n / present / 4)));
  const int64_t top = (1LL << 31) - 1;
  if (k0 * n >= top) k0 = top / n;
  return (int)k0;
}

// The whole call on h->stream, for arguments the caller has checked
int kbet_run(hb_handle* h, const DevRows& X, int d, const int32_t* batches, int n_batches, const int32_t* labels,
             int n_labels, int fixed_k0, double* stat, double* pval, int32_t* k0_out, int32_t* idx, int64_t idx_ld) {
  ScoreScratch& s = score_scratch(h);
  const int64_t N = X.n;
  const cudaStream_t st = h->stream;
  const int KD = (d + 7) & ~7;
  // ---- the index of the (label, batch) pairs, the rows in sorted order and the finite rows per pair
  TupleIndex ti;
  static const char* const names[2] = {"hb_kbet: labels", "hb_kbet: batches"};
  TRY(pair_index(h, X, d, KD, labels, n_labels, batches, n_batches, names, ti));
  const int J = (int)ti.uniq.size();
  std::vector<int> count(J);
  CK(cudaMemcpyAsync(count.data(), s.count.p, sizeof(int) * J, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));

  // ---- each label's k0 (pair q is label uniq[q] / n_batches: the label is the most significant level)
  std::vector<int64_t> n(n_labels, 0);
  std::vector<int> present(n_labels, 0), p0(n_labels, -1), p1(n_labels, 0);
  for (int q = 0; q < J; ++q) {
    const int l = (int)(ti.uniq[q] / n_batches);
    if (p0[l] < 0) p0[l] = q;
    p1[l] = q + 1;
    n[l] += count[q];
    present[l] += count[q] > 0;
  }
  std::vector<int32_t> k0(n_labels);
  int kmax = 0;
  for (int l = 0; l < n_labels; ++l) {
    k0[l] = kbet_k0(n[l], present[l], fixed_k0);
    kmax = std::max(kmax, k0[l] - 1);
  }
  if (idx && idx_ld < kmax)
    return fail(h, 2, "hb_kbet: idx_ld = %lld is smaller than the %d neighbours of the largest k0", (long long)idx_ld, kmax);
  if (k0_out) CK(cudaMemcpyAsync(k0_out, k0.data(), sizeof(int32_t) * n_labels, cudaMemcpyHostToDevice, st));
  std::vector<KbetPair> pairs(J);
  for (int q = 0; q < J; ++q) {
    const int l = (int)(ti.uniq[q] / n_batches);
    pairs[q] = KbetPair{k0[l], (int)n[l], present[l] - 1, p0[l], p1[l]};
  }
  CK(s.pairs.reserve((size_t)J));
  TRY(upload_vector(h, s.pairs, pairs));

  // ---- the grouped sweep over the tested labels' tiles, and the merge into sorted-position lists
  if (kmax > 0) {
    const KnnGeometry g = knn_geometry(d, kmax, N, N, h->num_sms);
    std::vector<int4> tiles;
    for (const int4& t : sil_tiles(ti, n_batches, g.tq))
      if (k0[(int)(ti.uniq[t.z] / n_batches)] > 0)
        tiles.push_back(make_int4(t.x, t.y, (int)ti.tstart[t.z], (int)ti.tstart[t.w]));
    CK(s.tiles.reserve(tiles.size()));
    TRY(upload_vector(h, s.tiles, tiles));
    CK(s.part.reserve((size_t)N * kmax));
    CK(s.idx.reserve((size_t)N * kmax));
    CK(cudaMemsetAsync(s.part.p, 0xff, sizeof(int) * (size_t)N * kmax, st));  // rows of untested labels: no candidate
    const KnnGroupArgs a{{s.rows.p, s.rows.p, s.hx.p, s.part.p, N, N, KD, kmax, g.stages, 1, 0}, s.tiles.p};
    TRY(launch_knn_tc(h, g, kmax, dim3((unsigned)tiles.size()), a));
    TRY(launch(h, k_knn_merge, dim3((unsigned)((N + 3) / 4)), dim3(128), (size_t)4 * 2 * kmax * sizeof(float),
               (const float*)s.rows.p, (const float*)s.rows.p, (const int*)s.part.p, N, KD, kmax, kmax, 0, s.idx.p,
               (float*)nullptr));
  }
  KbetArgs k{kmax > 0 ? s.idx.p : nullptr, s.hx.p, s.pstart.p, s.count.p, s.pairs.p, s.sort_perm.p, stat, pval,
             idx, N, idx ? idx_ld : 0, J, kmax};
  return launch(h, k_kbet, dim3((unsigned)((N + KBET_WARPS - 1) / KBET_WARPS)), dim3(32 * KBET_WARPS), 0, k);
}

int run_kbet(hb_handle* h, const DevRows& X, int d, const int32_t* batches, int n_batches, const int32_t* labels,
             int n_labels, int k0, double* stat, double* pval, int32_t* k0_out, int32_t* idx, int64_t idx_ld,
             cudaStream_t caller) {
  TRY(check_score_shape(h, "hb_kbet", X.n, d));
  if (n_batches < 1) return fail(h, 2, "hb_kbet: n_batches = %d, at least one batch is needed", n_batches);
  if (labels && n_labels < 1) return fail(h, 2, "hb_kbet: n_labels = %d, at least one label is needed", n_labels);
  if (!labels) n_labels = 1;
  if (n_batches > X.n || n_labels > X.n)
    return fail(h, 2, "hb_kbet: %d batches and %d labels, more codes than the N = %lld rows", n_batches, n_labels, (long long)X.n);
  if (k0 != 0 && (k0 < 2 || k0 > KBET_MAX_K0))
    return fail(h, 2, "hb_kbet: k0 = %d is not supported (0 for scib's rule, or 2 <= k0 <= %d)", k0, KBET_MAX_K0);
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, batches, "batches"));
  if (labels) TRY(check_device_ptr(h, labels, "labels"));
  TRY(check_device_ptr(h, stat, "stat"));
  TRY(check_device_ptr(h, pval, "pval"));
  if (k0_out) TRY(check_device_ptr(h, k0_out, "k0_out"));
  if (idx) TRY(check_device_ptr(h, idx, "idx"));
  return run_score(h, caller, "kbet", [&] {
    return kbet_run(h, X, d, batches, n_batches, labels, n_labels, k0, stat, pval, k0_out, idx, idx_ld);
  });
}

}  // namespace
