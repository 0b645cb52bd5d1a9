// map_host.cuh — mapping new cells onto a finished integration without rerunning Harmony (DESIGN §8): the compression
// of a reference into per-cluster statistics, the setup of a query handle, and the single pass that softly assigns the
// query's cells to the reference's clusters and corrects them with one ridge step anchored on the reference.
// Included by harmony_b200.cu after the setup steps it shares with hb_setup.
#pragma once

namespace {

// the reference statistics a mapping handle holds besides Y (= Yref) and sigma
struct MapState {
  DevBuf<float> Nr;    // [K]
  DevBuf<float> Cref;  // [K][d]
};

// hb_reference: Nr, Cref, Yref (d x K column-major host doubles, like getCentroids) and sigma of the integration the
// handle holds, from the Z_corr getZcorr() returns and R.  Null outputs are skipped.
int reference_stats(hb_handle* h, double* centroids, double* Nr, double* Cref, double* sigma) {
  const int K = h->K, d = h->d, J = h->J, D1 = d + 1;
  DevBuf<double> out;  // [K][2d + 1]: Cref | Nr | Yref
  CK(out.alloc((size_t)K * (2 * d + 1)));
  {
    RegionScope rs(h, "reference");
    TRY(normalise_pending_zc(h));
    CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * D1, h->stream));
    TRY(run_stats_tc(h, h->Zc.p));
    k_reference_fold<<<K, 128, sizeof(double) * D1, h->stream>>>(h->S.p, out.p, J, K, d);
    CKL();
  }
  std::vector<double> o(out.n);
  CK(cudaMemcpyAsync(o.data(), out.p, sizeof(double) * o.size(), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < K; ++k) {
    const double* ok = o.data() + (size_t)k * (2 * d + 1);
    if (Cref) std::copy(ok, ok + d, Cref + (size_t)k * d);
    if (Nr) Nr[k] = ok[d];
    if (centroids) std::copy(ok + D1, ok + D1 + d, centroids + (size_t)k * d);
  }
  if (sigma) TRY(download_small(h, h->sigma.p, K, sigma));
  return 0;
}

bool all_finite(const double* v, size_t n) {
  return std::all_of(v, v + n, [](double x) { return std::isfinite(x); });
}

// hb_map_setup / hb_map_setup_device: the reference checks, then the setup steps hb_setup shares (the query's tuple
// index, kernels, buffers, initial state and rows) and the reference's statistics.  No update plan, no update state and
// no block geometry: mapping runs no update_R.
int map_setup(hb_handle* h, const CellInput& in, int d, int64_t N, const int32_t* B_vec, int C, const double* lambda,
              int K, const double* centroids, const double* Nr, const double* Cref, const double* sigma) {
  if (h->world > 1 || (h->shard_set && (h->N_global != N || h->cell_offset != 0)))
    return fail(h, 3, "mapping does not take sharded cells");
  if (!(in.host || in.dev.p) || !in.phi || !B_vec || !lambda || !centroids || !Nr || !Cref || !sigma)
    return fail(h, 2, "null argument");
  TRY(check_dimensions(h, d, N, C, K));
  for (int c = 0; c < C; ++c)
    if (B_vec[c] < 1) return fail(h, 2, "covariate %d has no levels", c);
  const int B = std::accumulate(B_vec, B_vec + C, 0);
  for (int b = 0; b < B; ++b)
    if (!(std::isfinite(lambda[b]) && lambda[b] > 0)) return fail(h, 2, "lambda[%d] = %g: lambda must be finite and positive", b, lambda[b]);
  TRY(check_sigma(h, sigma, K));
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(Nr[k]) && Nr[k] >= 0)) return fail(h, 2, "Nr[%d] = %g: cluster masses must be finite and >= 0", k, Nr[k]);
  if (!all_finite(centroids, (size_t)K * d) || !all_finite(Cref, (size_t)K * d))
    return fail(h, 2, "the reference's centroids and Cref must be finite");
  CK(cudaSetDevice(h->device));
  h->n = h->N_global = N;
  h->cell_offset = 0;
  set_shape(h, d, C, K, B_vec);
  h->lambda_estimation = false;
  HostLap lap(h->stream, "hb_map_setup");
  TupleIndex ti;
  TRY(setup_tuples(h, in, ti));
  lap.mark("tuple index (device)");
  TRY(alloc_common(h, 1));
  h->map.reset(new MapState());
  CK(h->map->Nr.alloc(K));
  CK(h->map->Cref.alloc((size_t)K * d));
  lap.mark("device allocations");
  // Pr_b = 0 (the assignment's E is not used); lambda_0 = 0
  TRY(init_common(h));
  CK(cudaMemsetAsync(h->Pr_b.p, 0, sizeof(float) * B, h->stream));
  std::vector<float> lam(B + 1, 0.f);
  for (int b = 0; b < B; ++b) lam[b + 1] = (float)lambda[b];
  TRY(upload_vector(h, h->lambda, lam));
  set_sigma_scalars(h, sigma);
  TRY(upload_vector(h, h->sigma, std::vector<float>(sigma, sigma + K)));
  TRY(upload_vector(h, h->Y, std::vector<float>(centroids, centroids + (size_t)K * d)));
  TRY(upload_vector(h, h->map->Nr, std::vector<float>(Nr, Nr + K)));
  TRY(upload_vector(h, h->map->Cref, std::vector<float>(Cref, Cref + (size_t)K * d)));
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("memsets + small uploads");
  TRY(upload_z(h, in));
  {
    RegionScope rs(h, "upload");  // Z_corr starts as Z_orig: the assignment normalises it in place
    CK(cudaMemcpyAsync(h->Zc.p, h->Zo.p, sizeof(float) * (size_t)N * h->DS, cudaMemcpyDeviceToDevice, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("Z upload");
  h->ran_setup = true;
  h->mapping = true;
  return 0;
}

// hb_map: R_q = softmax_k(-2 (1 - Yref_k . z_i / |z_i|) / sigma_k) in natural order, the query's statistics, the solve
// against the reference (k_map_solve) and Z_corr = Z_orig - sum_k R_k V[q][k].  Repeatable: a second call first puts
// Z_orig back into Z_corr.
int run_map(hb_handle* h) {
  const int K = h->K, d = h->d, J = h->J;
  CK(cudaSetDevice(h->device));
  if (h->ran_map)
    CK(cudaMemcpyAsync(h->Zc.p, h->Zo.p, sizeof(float) * (size_t)h->n * h->DS, cudaMemcpyDeviceToDevice, h->stream));
  TRY(run_assign(h, true, false));
  {
    RegionScope rs(h, "ridge_stats");
    CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * (d + 1), h->stream));
    TRY(run_stats_tc(h, h->Zo.p));
  }
  {
    RegionScope rs(h, "ridge_solve");
    MapSolveArgs a;
    a.S = h->S.p;
    a.Nr = h->map->Nr.p;
    a.Cref = h->map->Cref.p;
    a.lambda = h->lambda.p;
    a.tuple_levels = h->tuple_levels.p;
    a.V = h->V.p;
    a.Wfull = h->Wfull.p;
    a.scratch = h->scratch.p;
    a.err_flag = h->err_flag.p;
    a.J = J;
    a.K = K;
    a.B = h->B;
    a.C = h->C;
    a.d = d;
    k_map_solve<<<K, 256, 0, h->stream>>>(a);
    CKL();
  }
  TRY(run_apply(h));
  h->ran_map = true;
  return h->C > 1 ? check_err_flag(h) : 0;
}

}  // namespace
