// correct_host.cuh — moe_correct_ridge_cpp (harmony.cpp:345-638): the ridge statistics, the solve and the apply.
#pragma once

namespace {

// S[q][k][:] += R_q^T [Z_q | 1] on the tensor cores (stats_tc3.cuh): one launch per 128 clusters x 64 or 128 columns
// of [Z | 1] (K = 100, d = 50: one launch).  The caller zeroes S.
int run_stats_tc(hb_handle* h, const float* Zsrc) {
  const int K = h->K, D1 = h->d + 1;
  StatsTcArgs t;
  t.R = h->R.p;
  t.Zo = Zsrc;
  t.S = h->S.p;
  t.d = h->d;
  t.K = K;
  t.KS = h->KS;
  t.DS = h->DS;
  const int grid_tc = h->tiles.deal(t, h->num_sms);
  const int nb = D1 > 64 ? 128 : 64;
  for (t.k_off = 0; t.k_off < K; t.k_off += 128)
    for (t.c_off = 0; t.c_off < D1; t.c_off += nb) {
      const size_t smem = stats_tc_smem_bytes(stats_tc_rk(h->KS, t.k_off), stats_tc_rc(h->DS, t.c_off, nb), nb);
      TRY(launch(h, nb == 64 ? k_stats_tc<1> : k_stats_tc<2>, grid_tc, ST_THREADS, smem, t));
    }
  return 0;
}

// Zc = Zo - sum_k R_k V[q][k] for the per-tuple corrections V a solve wrote (moe_correct_ridge_cpp, and the mapping of
// a query in map_host.cuh)
int run_apply(hb_handle* h) {
  const int K = h->K, d = h->d;
  RegionScope rs(h, "ridge_apply");
  switch (h->paths.apply) {
    case Apply::Tc:
    case Apply::TcCols: {
      // Tc: one range of all columns; TcCols (d > 256, or K x d beyond the FFMA apply): ranges of <= 128 columns.
      // Each column range runs in cluster ranges of at most AP_MAXK clusters, equal sizes, multiples of 8, and small
      // enough for two raw stages of shared memory: the first launch subtracts its share from Zo, the following ones
      // from the partial result in Zc
      const bool cols = h->paths.apply == Apply::TcCols;
      ApplyTcArgs a;
      a.R = h->R.p;
      a.V = h->V.p;
      a.Zc = h->Zc.p;
      a.d = d;
      a.K = K;
      a.KS = h->KS;
      a.DS = h->DS;
      const int grid = h->tiles.deal(a, h->num_sms);
      const int DC = cols ? 128 : h->DS;
      auto kernel = cols ? k_apply_tc_cols : d <= 64 ? k_apply_tc<1> : k_apply_tc<2>;
      for (a.c_off = 0; a.c_off < h->DS; a.c_off += DC) {
        a.DC = std::min(DC, h->DS - a.c_off);
        auto stages = [&](int RS) { return cols ? apply_cols_stages(RS, a.DC) : apply_tc_stages(RS, d, h->DS); };
        int npass = (K + AP_MAXK - 1) / AP_MAXK, Kpass = 0;
        for (;; ++npass) {
          Kpass = (((K + npass - 1) / npass) + 7) & ~7;
          if (stages(apply_tc_rs(Kpass, h->KS, 0)) >= 2) break;
        }
        for (int k_off = 0; k_off < K; k_off += Kpass) {
          a.k_off = k_off;
          a.Kp = std::min(Kpass, K - k_off);
          a.KD = (a.Kp + 7) & ~7;
          a.minuend = (k_off == 0) ? h->Zo.p : h->Zc.p;
          const int RS = apply_tc_rs(a.KD, h->KS, k_off);
          TRY(launch(h, kernel, grid, AP_THREADS, cols ? apply_cols_smem_bytes(RS, a.DC) : apply_tc_smem_bytes(RS, d, h->DS), a));
        }
      }
      break;
    }
    case Apply::Ffma: {
      ApplyArgs a;
      a.R = h->R.p;
      a.Zo = h->Zo.p;
      a.V = h->V.p;
      a.Zc = h->Zc.p;
      a.d = d;
      a.K = K;
      a.ldR = h->KS;
      a.ldZ = h->DS;
      const int grid = h->tiles.deal(a, h->num_sms * 4);
      TRY(launch(h, k_ridge_apply, grid, dim3((d + 3) / 4, TM / 4), apply_ffma_smem_bytes(K, d), a));
      break;
    }
  }
  return 0;
}

int run_correct(hb_handle* h) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, C = h->C;
  const int D1 = d + 1;
  {
    RegionScope rs(h, "ridge_stats");
    CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * D1, h->stream));
    TRY(run_stats_tc(h, h->Zo.p));
    TRY(allreduce_f(h, h->S.p, (size_t)J * K * D1));
  }
  {
    RegionScope rs(h, "ridge_solve");
    SolveArgs a;
    a.S = h->S.p;
    a.O = h->O.p;
    a.E = h->E.p;
    a.N_b = h->N_b.p;
    a.lambda = h->lambda_estimation ? nullptr : h->lambda.p;
    a.tuple_levels = h->tuple_levels.p;
    a.cov_of = h->cov_of_d.p;
    a.Y = h->Y.p;
    a.V = h->V.p;
    a.Wfull = h->Wfull.p;
    a.skipped = h->skipped.p;
    a.scratch = h->scratch.p;
    a.iscratch = h->iscratch.p;
    a.err_flag = h->err_flag.p;
    a.J = J;
    a.K = K;
    a.B = B;
    a.C = C;
    a.d = d;
    a.KS = h->KS;
    a.alpha = h->alpha;
    a.cutoff = h->cutoff;
    k_ridge_solve<<<K, 256, sizeof(int) * (size_t)(B + C), h->stream>>>(a);
    CKL();
  }
  return run_apply(h);
}

}  // namespace
