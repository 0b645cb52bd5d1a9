// map_host.cuh — mapping new cells onto a finished integration without rerunning Harmony (DESIGN §8): the compression
// of a reference into per-cluster statistics, the setup of a query handle, and the single pass that softly assigns the
// query's cells to the reference's clusters and corrects them with one ridge step anchored on the reference.
// Included by harmony_b200.cu after the setup steps it shares with hb_setup (setup_tuples, ZInput).
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

// hb_map_setup / hb_map_setup_device: the query's tuple index and rows, the reference's statistics and the buffers the
// mapping reads.  No update plan, no update state and no block geometry: mapping runs no update_R.
int map_setup(hb_handle* h, const ZInput& Z, int d, int64_t N, const int32_t* phi_i, bool phi_on_device,
              const int32_t* B_vec, int C, const double* lambda, int K, const double* centroids, const double* Nr,
              const double* Cref, const double* sigma) {
  if (h->ran_setup) return fail(h, 3, "setup was already run on this object");
  if (h->world > 1 || (h->shard_set && (h->N_global != N || h->cell_offset != 0)))
    return fail(h, 3, "mapping does not take sharded cells");
  if (!(Z.host || Z.dev) || !phi_i || !B_vec || !lambda || !centroids || !Nr || !Cref || !sigma)
    return fail(h, 2, "null argument");
  if (d < 1 || N < 1 || C < 1 || K < 1) return fail(h, 2, "bad dimensions");
  if (K > 1024) return fail(h, 2, "K = %d is not supported (K <= 1024)", K);
  if (N > 2000000000LL) return fail(h, 2, "more than 2e9 cells per GPU are not supported");
  for (int c = 0; c < C; ++c)
    if (B_vec[c] < 1) return fail(h, 2, "covariate %d has no levels", c);
  const int B = std::accumulate(B_vec, B_vec + C, 0);
  for (int b = 0; b < B; ++b)
    if (!(std::isfinite(lambda[b]) && lambda[b] > 0)) return fail(h, 2, "lambda[%d] = %g: lambda must be finite and positive", b, lambda[b]);
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(sigma[k]) && (float)sigma[k] > 0.f))
      return fail(h, 2, "sigma[%d] = %g: sigma must be finite and positive", k, sigma[k]);
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(Nr[k]) && Nr[k] >= 0)) return fail(h, 2, "Nr[%d] = %g: cluster masses must be finite and >= 0", k, Nr[k]);
  if (!all_finite(centroids, (size_t)K * d) || !all_finite(Cref, (size_t)K * d))
    return fail(h, 2, "the reference's centroids and Cref must be finite");
  CK(cudaSetDevice(h->device));
  h->n = h->N_global = N;
  h->cell_offset = 0;
  h->d = d;
  h->C = C;
  h->K = K;
  h->KS = (K + 3) & ~3;
  h->DS = (d + 3) & ~3;
  h->B_vec.assign(B_vec, B_vec + C);
  h->B = B;
  h->lambda_estimation = false;
  HostLap lap(h->stream, "hb_map_setup");
  TupleIndex ti;
  TRY(setup_tuples(h, phi_i, phi_on_device, Z.stream, ti));
  lap.mark("tuple index (device)");
  // ---- the buffers the assignment, the statistics, the solve and the apply read
  const int J = h->J, KS = h->KS, M = B + 1;
  const size_t nK = (size_t)N * KS, nd = (size_t)N * h->DS, BK = (size_t)B * KS;
  h->coop_grid = h->num_sms;
  h->paths = select_kernels(K, d, J, N, 1, h->coop_grid, h->kernel_set);
  h->map.reset(new MapState());
  for (DevBuf<float>* b : {&h->Zo, &h->Zc}) CK(b->alloc(nd));
  for (DevBuf<float>* b : {&h->U, &h->R}) CK(b->alloc(nK));
  for (DevBuf<float>* b : {&h->O, &h->E}) CK(b->alloc(BK));
  CK(h->Pr_b.alloc(B));
  CK(h->Y.alloc((size_t)K * d));
  CK(h->sigma.alloc(K));
  CK(h->lambda.alloc(M));
  CK(h->tmpT.alloc((size_t)B * K));
  CK(h->Oacc.alloc(BK + KS));
  CK(h->S.alloc((size_t)J * K * (d + 1)));
  CK(h->V.alloc((size_t)J * K * d));
  CK(h->scratch.alloc((size_t)K * (2 * (size_t)M * M + 2 * (size_t)M * d)));
  CK(h->err_flag.alloc(1));
  CK(h->obj_acc.alloc(2));
  CK(h->stage.alloc((size_t)8 << 20));
  CK(h->tuple_levels.alloc((size_t)J * C));
  CK(h->map->Nr.alloc(K));
  CK(h->map->Cref.alloc((size_t)K * d));
  TRY(build_tiles(h, h->tiles, h->tuple_start_h, TM));
  TRY(build_tiles(h, h->tc_tiles, h->tuple_start_h, TC_TM));
  lap.mark("device allocations");
  // ---- initial state and the small uploads; Pr_b = 0 (the assignment's E is not used)
  CK(cudaMemsetAsync(h->err_flag.p, 0, sizeof(int), h->stream));
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  for (float* t : {h->O.p, h->E.p}) CK(cudaMemsetAsync(t, 0, sizeof(float) * BK, h->stream));
  CK(cudaMemsetAsync(h->Pr_b.p, 0, sizeof(float) * B, h->stream));
  CK(cudaMemsetAsync(h->R.p, 0, sizeof(float) * nK, h->stream));
  for (float* z : {h->Zo.p, h->Zc.p}) CK(cudaMemsetAsync(z, 0, sizeof(float) * nd, h->stream));
  k_fill_f<<<grid_for((int64_t)nK, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->U.p, (int64_t)nK, U_PAD);
  CKL();
  auto up = [&](auto& buf, const auto& v) {
    return cudaMemcpyAsync(buf.p, v.data(), sizeof(v[0]) * v.size(), cudaMemcpyHostToDevice, h->stream);
  };
  CK(up(h->tuple_levels, h->tuple_levels_h));
  std::vector<float> lam(M, 0.f);
  for (int b = 0; b < B; ++b) lam[b + 1] = (float)lambda[b];
  CK(up(h->lambda, lam));
  set_sigma_scalars(h, sigma);
  CK(up(h->sigma, std::vector<float>(sigma, sigma + K)));
  CK(up(h->Y, std::vector<float>(centroids, centroids + (size_t)K * d)));
  CK(up(h->map->Nr, std::vector<float>(Nr, Nr + K)));
  CK(up(h->map->Cref, std::vector<float>(Cref, Cref + (size_t)K * d)));
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("memsets + small uploads");
  if (Z.dev)
    TRY(upload_rows_device(h, Z.dev, Z.dtype, Z.ld, Z.stream));
  else
    TRY(upload_rows(h, Z.host, d, h->DS, h->Zo.p));
  {
    RegionScope rs(h, "upload");  // Z_corr starts as Z_orig: the assignment normalises it in place
    CK(cudaMemcpyAsync(h->Zc.p, h->Zo.p, sizeof(float) * nd, cudaMemcpyDeviceToDevice, h->stream));
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
