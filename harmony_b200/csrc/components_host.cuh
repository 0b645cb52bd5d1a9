// components_host.cuh — hb_graph_components (DESIGN §12): the checks and the launches of components.cuh.  The call needs
// no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// The whole call on h->stream, for arguments the caller has checked: the range pass (read back once; comp and
// largest stay unwritten when it finds a bad entry), then the union-find into comp and the sizes into largest.
int components_run(hb_handle* h, const int32_t* idx, int64_t idx_ld, int64_t N, int k, const int32_t* labels,
                   int n_labels, int32_t* comp, int32_t* largest) {
  ScoreScratch& s = score_scratch(h);
  const cudaStream_t st = h->stream;
  const int cap = h->num_sms * 8;
  const int64_t k1 = (int64_t)k + 1;  // an entry's place in the bad word: row k1 + m, the label at m = k
  unsigned long long bad = 0;
  TRY(run_check(h, &bad, k_cc_check, dim3(grid_for(N * k1, 256, cap)), idx, idx_ld, N, k, labels, n_labels));
  if (bad != ~0ull) {
    const int64_t row = (int64_t)(bad / k1);
    const int m = (int)(bad % k1);
    int v = 0;
    TRY(read_back(h, m < k ? idx + row * idx_ld + m : labels + row, &v));
    if (m < k)
      return fail(h, 2, "hb_graph_components: idx[%lld][%d] = %d is not -1 or a row in 0..%lld", (long long)row, m, v,
                  (long long)(N - 1));
    return fail(h, 2, "hb_graph_components: labels[%lld] = %d is not a code in 0..%d", (long long)row, v, n_labels - 1);
  }
  const int rows_grid = grid_for(N, 256, cap);
  TRY(launch(h, k_cc_init, dim3(rows_grid), dim3(256), 0, N, (int*)comp));
  TRY(launch(h, k_cc_hook, dim3(grid_for(N * (int64_t)k, 256, cap)), dim3(256), 0, idx, idx_ld, N, k, labels, (int*)comp));
  TRY(launch(h, k_cc_compress, dim3(rows_grid), dim3(256), 0, N, (int*)comp));
  if (!largest) return 0;
  CK(s.count.reserve((size_t)N));
  CK(cudaMemsetAsync(s.count.p, 0, sizeof(int) * N, st));
  CK(cudaMemsetAsync(largest, 0, sizeof(int32_t) * (labels ? n_labels : 1), st));
  TRY(launch(h, k_cc_count, dim3(rows_grid), dim3(256), 0, (const int*)comp, N, s.count.p));
  return launch(h, k_cc_largest, dim3(rows_grid), dim3(256), 0, (const int*)comp, (const int*)s.count.p, labels, N,
                (int*)largest);
}

int run_components(hb_handle* h, const int32_t* idx, int64_t idx_ld, int64_t N, int k, const int32_t* labels,
                   int n_labels, int32_t* comp, int32_t* largest, cudaStream_t caller) {
  if (N < 1) return fail(h, 2, "hb_graph_components: N = %lld rows, at least 1 is needed", (long long)N);
  if (N >= (1LL << 31)) return fail(h, 2, "hb_graph_components: N = %lld rows are not supported (N < 2^31)", (long long)N);
  if (k < 1) return fail(h, 2, "hb_graph_components: k = %d, at least 1 entry per row is needed", k);
  if (idx_ld < k) return fail(h, 2, "hb_graph_components: row stride %lld of idx is smaller than k = %d", (long long)idx_ld, k);
  if (labels && (n_labels < 1 || n_labels > N))
    return fail(h, 2, "hb_graph_components: n_labels = %d is not supported (1 <= n_labels <= N = %lld)", n_labels, (long long)N);
  TRY(check_device_ptr(h, idx, "idx"));
  TRY(check_device_ptr(h, comp, "comp"));
  if (labels) TRY(check_device_ptr(h, labels, "labels"));
  if (largest) TRY(check_device_ptr(h, largest, "largest"));
  return run_score(h, caller, "components",
                   [&] { return components_run(h, idx, idx_ld, N, k, labels, n_labels, comp, largest); });
}

}  // namespace
