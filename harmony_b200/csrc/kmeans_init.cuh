// kmeans_init.cuh — the native kmeans_centers of init_cluster_cpp.  Included by harmony_b200.cu after assign_host.cuh.
#pragma once

namespace {

// Y = kmeans_centers(..) (utils.cpp:10-64) on the cosine-normalised cells, sharded like everything else:
// initialize_centroids' rule (K start cells, then per centroid the winner of an exponential race weighted by the
// distance from its start cell, already-taken cells skipped) with keyed-hash uniforms, then 10 Lloyd iterations
// (10 x arma::kmeans(.., keep_existing, 1): Euclidean assignment, means of the members).
int kmeans_centers(hb_handle* h) {
  const int K = h->K, d = h->d;
  const size_t Kd = (size_t)K * d;
  if (h->N_global >= (1ll << 32)) return fail(h, 2, "native k-means initialisation supports < 2^32 cells; pass Y0");
  DevBuf<float> ysum;
  CK(ysum.alloc(Kd + K));
  const uint64_t seed = hb_mix64(h->seed ^ 0x6b6d65616e73ull);
  DevBuf<int64_t> cells_d;
  DevBuf<unsigned long long> best_d;
  CK(cells_d.alloc(K));
  CK(best_d.alloc(K));
  std::vector<int64_t> cells(K);
  h->kmeans_means.clear();
  auto keep_means = [&]() -> int {  // test hook: Y after the race's gather (step 0) and after each Lloyd step
    if (!h->kmeans_keep_means) return 0;
    const size_t at = h->kmeans_means.size();
    h->kmeans_means.resize(at + Kd);
    CK(cudaMemcpyAsync(h->kmeans_means.data() + at, h->Y.p, sizeof(float) * Kd, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
  };
  auto gather = [&](int only) -> int {  // Y rows <- cells (all, or one centroid), summed over the ranks that own them
    CK(cudaMemcpyAsync(cells_d.p, cells.data(), sizeof(int64_t) * K, cudaMemcpyHostToDevice, h->stream));
    float* dst = (only >= 0) ? h->Y.p + (size_t)only * d : h->Y.p;
    const size_t cnt = (only >= 0) ? (size_t)d : Kd;
    CK(cudaMemsetAsync(dst, 0, sizeof(float) * cnt, h->stream));
    k_kmeans_gather<<<K, 64, 0, h->stream>>>(h->Zc.p, h->inv_sort.p, h->Y.p, cells_d.p, K, d, h->DS, h->cell_offset, h->n, only);
    CKL();
    return allreduce_f(h, dst, cnt);
  };
  // (1) start cells: floor(u (N - 1))  (utils.cpp:12-16)
  for (int k = 0; k < K; ++k)
    cells[k] = (int64_t)std::floor((double)kmeans_uniform(seed, (uint64_t)K, (uint64_t)k) * (double)(h->N_global - 1));
  TRY(gather(-1));
  // (2) the races of all centroids in one pass over the cells (a centroid's race only looks at its own start cell)
  // both steps run from tensor-core logits U = 2 (z . y - 1) (sigma = 1) when select_kernels chose them; else from
  // the FFMA kernels (thread per cell)
  DevBuf<float> ones, yy;
  const KmeansInit km = h->paths.kmeans;
  const int km_nv = sp_nv(h->KS);
  if (km != KmeansInit::Ffma) {
    CK(ones.alloc(K));
    CK(yy.alloc(K));
    k_fill_f<<<1, 256, 0, h->stream>>>(ones.p, (int64_t)K, 1.0f);
    CKL();
  }
  std::vector<unsigned long long> best(K);
  bool logits_of_start = false;  // U holds the logits of the start cells
  auto race = [&](int i0, int i1, const std::vector<int64_t>& taken) -> int {
    DevBuf<int64_t> taken_d;
    if (!taken.empty()) {
      CK(taken_d.alloc(taken.size()));
      CK(cudaMemcpyAsync(taken_d.p, taken.data(), sizeof(int64_t) * taken.size(), cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaMemsetAsync(best_d.p + i0, 0xff, sizeof(unsigned long long) * (i1 - i0), h->stream));
    switch (km) {
      case KmeansInit::Ffma:
        TRY(launch(h, k_kmeans_race, grid_for(h->n, 128, h->num_sms * 4), 128, sizeof(float) * (size_t)(i1 - i0) * d,
                   h->Zc.p, h->sort_perm.p, h->Y.p, best_d.p, taken.empty() ? nullptr : taken_d.p, (int)taken.size(), h->n,
                   K, d, h->DS, h->cell_offset, seed, i0, i1));
        break;
      case KmeansInit::LogitsTc:
      case KmeansInit::LogitsWide: {
        if (!logits_of_start) {
          TRY(launch_logits(h, ones.p, false, km == KmeansInit::LogitsWide));
          logits_of_start = true;
        }
        const int grid_r = grid_for(h->n * 32, 256, h->num_sms * 8);
        TRY(dispatch<1, 2, 4, 8>(h, km_nv, kUnsupportedK, [&](auto nvc) {
          return launch(h, k_kmeans_race_u<decltype(nvc)::value>, grid_r, 256, 0, h->U.p, h->sort_perm.p, best_d.p,
                        taken.empty() ? nullptr : taken_d.p, (int)taken.size(), h->n, K, h->KS, h->cell_offset, seed, i0, i1);
        }));
        break;
      }
    }
    if (h->world > 1) CKN(g_nccl.AllReduce(best_d.p + i0, best_d.p + i0, (size_t)(i1 - i0), ncclUint64, ncclMin, h->comm, h->stream));
    CK(cudaMemcpyAsync(best.data() + i0, best_d.p + i0, sizeof(unsigned long long) * (i1 - i0), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
  };
  TRY(race(0, K, {}));
  // (3) accept in centroid order; a winner that is already taken re-runs that centroid's race without the taken cells
  // (utils.cpp:38-45); the race of centroid i reads its START cell, so Y is only rewritten afterwards
  std::vector<int64_t> taken;
  for (int i = 0; i < K; ++i) {
    if (best[i] != ~0ull && std::find(taken.begin(), taken.end(), (int64_t)(best[i] & 0xffffffffull)) != taken.end())
      TRY(race(i, i + 1, taken));
    if (best[i] == ~0ull) return fail(h, 3, "native k-means initialisation: no free cell for centroid %d", i);
    const int64_t w = (int64_t)(best[i] & 0xffffffffull);
    taken.push_back(w);
    cells[i] = w;
  }
  h->kmeans_cells = cells;
  TRY(gather(-1));
  TRY(keep_means());
  for (int iter = 0; iter < 10; ++iter) {
    switch (km) {
      case KmeansInit::Ffma:
        CK(cudaMemsetAsync(ysum.p, 0, sizeof(float) * (Kd + K), h->stream));
        TRY(launch(h, k_kmeans_assign, grid_for(h->n, 128, h->num_sms * 4), 128, sizeof(float) * Kd, h->Zc.p, h->Y.p, ysum.p,
                   ysum.p + Kd, h->n, K, d, h->DS));
        TRY(allreduce_f(h, ysum.p, Kd + K));
        k_kmeans_update<<<(int)((Kd + 255) / 256), 256, 0, h->stream>>>(h->Y.p, ysum.p, ysum.p + Kd, K, d);
        CKL();
        break;
      case KmeansInit::LogitsTc:
      case KmeansInit::LogitsWide: {
        // Lloyd iteration on the tensor cores: logits -> one-hot rows of R -> members' sums and counts (K3) -> means
        TRY(launch_logits(h, ones.p, false, km == KmeansInit::LogitsWide));
        k_kmeans_norms<<<(K + 127) / 128, 128, 0, h->stream>>>(h->Y.p, yy.p, K, d);
        CKL();
        const int grid_p = grid_for(h->n * 32, 256, h->num_sms * 8);
        TRY(dispatch<1, 2, 4, 8>(h, km_nv, kUnsupportedK, [&](auto nvc) {
          return launch(h, k_kmeans_pick<decltype(nvc)::value>, grid_p, 256, 0, h->U.p, yy.p, h->R.p, h->n, K, h->KS);
        }));
        CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)h->J * K * (d + 1), h->stream));
        TRY(run_stats_tc(h, h->Zc.p));
        TRY(allreduce_f(h, h->S.p, (size_t)h->J * K * (d + 1)));
        k_kmeans_means_from_stats<<<(int)((Kd + 255) / 256), 256, 0, h->stream>>>(h->S.p, h->Y.p, h->J, K, d);
        CKL();
        break;
      }
    }
    TRY(keep_means());
  }
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // namespace
