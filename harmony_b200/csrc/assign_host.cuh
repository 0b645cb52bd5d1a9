// assign_host.cuh — logits, the natural-order and plan-order assignments and the legacy centroid step built on them.
#pragma once

namespace {

// buffers the assignment grows on first use
struct AssignState {
  DevBuf<float> Ypad;          // Y padded for k_logits_wide
  DevBuf<float> Rkeep, OEkeep;  // R / O,E saved around the distance-only assignment of the legacy centroid step
  DevBuf<double> objkeep;
};

// the fields both logits kernels take
template <typename A>
A logits_args(hb_handle* h, const float* sigma, bool normalise) {
  A t{};
  t.Zc = h->Zc.p;
  t.sigma = sigma;
  t.U = h->U.p;
  t.n = h->n;
  t.d = h->d;
  t.K = h->K;
  t.DS = h->DS;
  t.KS = h->KS;
  t.normalise = normalise ? 1 : 0;
  return t;
}

// U[i][k] = (2 / sigma_k) (z_i . y_k / |z_i| - 1) for all clusters on the tensor cores, 128 clusters per launch and d
// in chunks (logits_wide.cuh), after one pass that pads Y
int launch_logits_wide(hb_handle* h, const float* sigma, bool normalise) {
  const int KDc = (h->d + LW_DC - 1) / LW_DC * LW_DC, rows = (h->K + LW_NP - 1) / LW_NP * LW_NP;
  DevBuf<float>& Ypad = h->asg->Ypad;
  CK(Ypad.reserve((size_t)rows * KDc));
  k_pad_rows<<<grid_for((int64_t)rows * KDc, 256, h->num_sms * 4), 256, 0, h->stream>>>(h->Y.p, Ypad.p, h->K, h->d, rows, KDc);
  CKL();
  LogitsWideArgs t = logits_args<LogitsWideArgs>(h, sigma, normalise);
  t.Ypad = Ypad.p;
  t.KDc = KDc;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((h->n + LW_TM - 1) / LW_TM, h->num_sms));
  for (t.n_off = 0; t.n_off < h->K; t.n_off += LW_NP) TRY(launch(h, k_logits_wide, grid, LW_THREADS, logits_wide_smem_bytes(), t));
  return 0;
}

// U[i][k] = (2 / sigma_k) (z_i . y_k / |z_i| - 1) for all clusters on the tensor cores, 64 clusters per launch
// (logits_tc.cuh), or from launch_logits_wide when `wide`; `sigma`: device array of K values
int launch_logits(hb_handle* h, const float* sigma, bool normalise, bool wide) {
  if (wide) return launch_logits_wide(h, sigma, normalise);
  LogitsArgs t = logits_args<LogitsArgs>(h, sigma, normalise);
  t.Y = h->Y.p;
  t.KD = (h->d + 7) & ~7;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((h->n + LG_TM - 1) / LG_TM, h->num_sms));
  for (t.n_off = 0; t.n_off < h->K; t.n_off += LG_NP) TRY(launch(h, k_logits_tc, grid, LG_THREADS, logits_smem_bytes(t.KD), t));
  return 0;
}

// the fused kernel (assign_tc3.cuh) over the tiles, R / Z_corr outputs and accumulators the caller set in t
int launch_assign_tc3(hb_handle* h, Assign3Args& t, int grid, bool normalise, bool want_obj) {
  t.Zc = h->Zc.p;
  t.Y = h->Y.p;
  t.sigma = h->sigma.p;
  t.U = h->U.p;
  t.tuple_levels = h->tuple_levels.p;
  t.obj_acc = h->obj_acc.p;
  t.d = h->d;
  t.K = h->K;
  t.C = h->C;
  t.B = h->B;
  t.DS = h->DS;
  t.KS = h->KS;
  t.KD = (h->d + 7) & ~7;
  t.NP = (h->K + 15) & ~15;
  t.SS = assign3_stage_stride(h->KS);
  t.ns = h->paths.k1_stages;
  t.normalise = normalise ? 1 : 0;
  t.want_obj = want_obj ? 1 : 0;
  return launch(h, want_obj ? k_assign_tc3<true> : k_assign_tc3<false>, grid, A3_THREADS,
                assign3_smem_bytes(t.ns, t.KD, t.NP, t.KS), t);
}

// natural order: R, the per-tile sums of O and of the row sums, then O and E; want_obj: objective sums (init)
int run_assign(hb_handle* h, bool normalise, bool want_obj) {
  RegionScope rs(h, "assign");
  const int K = h->K, d = h->d, B = h->B, KS = h->KS;
  float* O_acc = h->Oacc.p;
  float* rs_acc = h->Oacc.p + (size_t)B * KS;
  CK(cudaMemsetAsync(h->Oacc.p, 0, sizeof(float) * ((size_t)B * KS + KS), h->stream));
  const Tiles& tl = h->tiles;
  switch (h->paths.assign) {
    case Assign::FusedTc: {
      Assign3Args t{};
      t.R = h->R.p;
      t.tile_p0 = h->tc_tiles.cell0.p;
      t.tile_len = h->tc_tiles.len.p;
      t.tile_tuple = h->tc_tiles.tuple.p;
      t.ntiles = h->tc_tiles.count;
      t.O_acc = O_acc;
      t.rs_acc = rs_acc;
      t.Zc_out = normalise ? h->Zc.p : nullptr;  // the compatibility paths read the normalised embedding back
      TRY(launch_assign_tc3(h, t, std::max(1, std::min(h->tc_tiles.count, h->num_sms)), normalise, want_obj));
      break;
    }
    case Assign::LogitsTc:
    case Assign::LogitsWide: {
      // shapes whose FFMA k_assign does not fit: logits on the tensor cores, then the softmax over the natural-order tiles
      TRY(launch_logits(h, h->sigma.p, normalise, h->paths.assign == Assign::LogitsWide));
      const int nv = sp_nv(KS);
      const size_t smem_sm = sizeof(float) * 8 * 128 * (size_t)nv;
      const int grid = std::max(1, std::min(tl.count, h->num_sms * 8));
      TRY(dispatch<1, 2, 4, 8>(h, nv, kUnsupportedK, [&](auto nvc) {
        return launch(h, k_softmax_tiles<decltype(nvc)::value>, grid, 256, smem_sm, h->U.p, h->R.p, h->sigma.p, tl.cell0.p,
                      tl.len.p, tl.tuple.p, h->tuple_levels.p, O_acc, rs_acc, h->obj_acc.p, tl.count, K, KS, h->C, want_obj ? 1 : 0);
      }));
      if (normalise) {  // the cold start leaves the normalised embedding in Z_corr (harmony.cpp:220)
        k_normalise_rows<<<grid_for((int64_t)h->n * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zc.p, h->Zc.p, h->n, d, h->DS);
        CKL();
      }
      break;
    }
    case Assign::Ffma: {
      AssignArgs a;
      a.Zc = h->Zc.p;
      a.Y = h->Y.p;
      a.sigma = h->sigma.p;
      a.U = h->U.p;
      a.R = h->R.p;
      a.tile_cell0 = tl.cell0.p;
      a.tile_len = tl.len.p;
      a.tile_tuple = tl.tuple.p;
      a.tuple_levels = h->tuple_levels.p;
      a.O_acc = O_acc;
      a.rs_acc = rs_acc;
      a.obj_acc = h->obj_acc.p;
      a.ntiles = tl.count;
      a.d = d;
      a.K = K;
      a.C = h->C;
      a.KP = (K + 63) & ~63;
      a.DS = h->DS;
      a.KS = KS;
      a.normalise = normalise ? 1 : 0;
      const size_t smem = assign_ffma_smem_bytes(K, d);
      TRY(dispatch<1, 2, 4, 8, 16, 32>(h, kq_for(K), kUnsupportedK, [&](auto kq) -> int {
        constexpr int KQ = decltype(kq)::value;
        // the occupancy query needs the shared-memory limit raised
        CK(cudaFuncSetAttribute(k_assign<KQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 1;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_assign<KQ>, ASSIGN_THREADS, smem));
        if (occ < 1) occ = 1;
        return launch(h, k_assign<KQ>, std::max(1, std::min(tl.count, h->num_sms * occ)), ASSIGN_THREADS, smem, a);
      }));
      break;
    }
  }
  h->R_user_set = false;
  TRY(allreduce_f(h, h->Oacc.p, (size_t)B * KS + KS));
  k_assign_finalize<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(O_acc, rs_acc, h->Pr_b.p, h->O.p, h->E.p, B, K, KS);
  CKL();
  if (!want_obj) CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));  // the cold start does not evaluate the objective
  return 0;
}

// cold start in the order of round 0 of the coming cluster_cpp call, where call_path chose that order
// (paths.cold != None): a tile's column sums are a share of its block's removal sums and go to the update kernel's
// accumulator slots; R is not stored and the objective is not evaluated
int run_assign_plan_order(hb_handle* h, bool normalise) {
  RegionScope rs(h, "assign");
  const UpdateState& u = *h->upd;
  const int K = h->K, B = h->B, KS = h->KS;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  switch (h->paths.cold) {
    case ColdStart::FusedTc: {
      Assign3Args t{};
      t.row_index = r.order;
      t.tile_p0 = r.tile_p0;
      t.tile_len = r.tile_len;
      t.tile_tuple = r.tile_tuple;
      t.tile_blk = r.tile_blk;
      t.ntiles_ptr = r.tile_count;
      t.acc = u.acc2.p;
      TRY(launch_assign_tc3(h, t, h->num_sms, normalise, false));
      break;
    }
    case ColdStart::LogitsTc:
    case ColdStart::LogitsWide: {
      // shapes the fused kernel cannot hold (d > 64 or K > 128): logits on the tensor cores, then one gather pass over
      // U in the order of round 0 for the softmax + the blocks' removal sums (harmony.cpp:312-313)
      TRY(launch_logits(h, h->sigma.p, normalise, h->paths.cold == ColdStart::LogitsWide));
      const int nv = sp_nv(KS);
      const size_t smem_sm = sizeof(float) * 8 * 128 * (size_t)nv;
      TRY(dispatch<1, 2>(h, nv, kUnsupportedUpdateK, [&](auto nvc) {
        return launch(h, k_softmax_block_sums<decltype(nvc)::value>, dim3(h->coop_grid, h->nb), 256, smem_sm, h->U.p, r.order,
                      r.ranges, h->tuple_levels.p, u.acc2.p, h->coop_grid, K, KS, h->C, B);
      }));
      break;
    }
  }
  h->R_user_set = false;
  // O, E of the assignment = the sums of the blocks' removal terms (harmony.cpp:226-227)
  // sharded cells: the rem halves of slots 1 .. nb in ONE all-reduce (their add halves are still zero here)
  if (h->world > 1) TRY(allreduce_f(h, u.slot(1), u.slot_floats() * (size_t)h->nb));
  k_assign_finalize_plan<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(u.acc2.p, h->nb, h->Pr_b.p, h->O.p, h->E.p, B, K, KS);
  CKL();
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));  // the cold start does not evaluate the objective
  h->zc_pending_norm = normalise;  // the normalised embedding (harmony.cpp:220) is materialised on demand
  return 0;
}

// STEP 1 of harmony::cluster_cpp as it ran before 2.0.4 (harmony.cpp:235-238):
//   Y = arma::normalise(Z_corr * R.t(), 2, 0);   dist_mat = 2 * (1 - Y.t() * Z_corr);
// built from the kernels of the ridge statistics (R^T [Z_corr | 1] per tuple) and of the assignment.  The
// assignment kernels also rewrite R, O, E and the objective sums, which this step must leave alone: they are
// saved and restored around the call (compatibility path, not a fast one).
int legacy_centroid_step(hb_handle* h) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, KS = h->KS;
  const int D1 = d + 1;
  const size_t nK = (size_t)h->n * KS, BK = (size_t)B * KS;
  AssignState& keep = *h->asg;
  CK(cudaMemsetAsync(h->S.p, 0, sizeof(float) * (size_t)J * K * D1, h->stream));
  TRY(run_stats_tc(h, h->Zc.p));  // the statistics of the corrected, normalised embedding
  TRY(allreduce_f(h, h->S.p, (size_t)J * K * D1));
  k_centroids_from_stats<<<K, 64, sizeof(float) * (size_t)d, h->stream>>>(h->S.p, h->Y.p, J, K, d);
  CKL();
  // distances to the new centroids -> U; everything else the assignment writes is put back
  CK(keep.Rkeep.reserve(nK));
  CK(keep.OEkeep.reserve(2 * BK));
  CK(keep.objkeep.reserve(2));
  CK(cudaMemcpyAsync(keep.Rkeep.p, h->R.p, sizeof(float) * nK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(keep.OEkeep.p, h->O.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(keep.OEkeep.p + BK, h->E.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(keep.objkeep.p, h->obj_acc.p, 2 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  TRY(run_assign(h, false, true));
  CK(cudaMemcpyAsync(h->R.p, keep.Rkeep.p, sizeof(float) * nK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->O.p, keep.OEkeep.p, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->E.p, keep.OEkeep.p + BK, sizeof(float) * BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(h->obj_acc.p, keep.objkeep.p, 2 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

}  // namespace
