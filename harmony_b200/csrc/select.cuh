// select.cuh — kernel selection: one kernel per stage for a shape, and the update path of a cluster_cpp call (host only).
#pragma once

namespace {

using namespace hb;

// One kernel per stage, chosen by select_kernels.  The values of UpdatePath are hb_debug_kernel_paths' numbers, those
// of Assign, ColdStart and Apply hb_debug_wide_paths'.
enum class UpdatePath { PerStep = 0, TwoPass = 1, SinglePass = 2 };
// assignment in natural order (init, legacy centroid step, cold start of the calls that do not run it in plan order):
// fused wgmma (assign_tc3.cuh), FFMA k_assign, or logits (logits_tc.cuh / logits_wide.cuh) + k_softmax_tiles
enum class Assign { FusedTc = 1, Ffma = 2, LogitsTc = 3, LogitsWide = 4 };
// cold-start assignment in the order of round 0 of the plan: fused wgmma, or logits + k_softmax_block_sums;
// None: no kernel for the shape, the cold start runs in natural order
enum class ColdStart { None = 0, FusedTc = 1, LogitsTc = 2, LogitsWide = 3 };
// ridge apply: wgmma k_apply_tc (one column range), FFMA k_ridge_apply, or k_apply_tc_cols over 128-column ranges
enum class Apply { Tc = 1, Ffma = 2, TcCols = 3 };
// native k-means initialisation: FFMA race and Lloyd steps, or both from logits with sigma = 1
enum class KmeansInit { Ffma, LogitsTc, LogitsWide };

struct KernelPaths {
  UpdatePath update = UpdatePath::PerStep;
  bool tuple_ranges = false;  // 2 J <= #SMs: the plan gives every CTA a slice of a block inside one tuple
  int k1_stages = 0;          // operand stages (1, 2) of the fused assignment kernel; 0: not fused
  Assign assign = Assign::Ffma;
  ColdStart cold = ColdStart::None;
  Apply apply = Apply::Ffma;
  KmeansInit kmeans = KmeansInit::Ffma;
};

int two_pass_nv(int KS) {
  int nv = 1;
  while (4 * UPD_LPR * nv < KS) nv <<= 1;
  return nv;
}
size_t two_pass_smem_bytes(int KS, int nb, int J) {
  const size_t tabn = (size_t)std::max(2, nb) * KS;
  const int nv = two_pass_nv(KS);
  const size_t rowbuf = (size_t)UPD_GWARPS * (upd_depth_upd(nv) + upd_depth_look(nv)) * UPD_RPW * KS;
  return sizeof(float) * ((size_t)KS + 2 * (tabn + (size_t)UPD_GWARPS * KS + 2 * (size_t)UPD_STAGE + (size_t)((J + 8) & ~3)) + rowbuf);
}

// The kernels of a shape (n: local cells, nb: update blocks); kernel_set: the HB_KS_* bits of the test hook.
// update_R runs the single-pass persistent kernel (update_single_pass.cuh) when every CTA's slice of a block can lie
// inside one covariate tuple (2 J <= #SMs), its ring fits shared memory and n KS < 2^32; else the two-pass
// persistent kernel (update_two_pass.cuh) when KS <= 256, J <= 8192 and its buffers fit shared memory; else three
// launches per block step (update_per_step.cuh).
// The other stages take their wgmma kernel where it fits, else their FFMA kernel where it fits (assign_ffma_fits,
// apply_ffma_fits, kmeans_ffma_fits), else the kernel of the wide shapes.  HB_KS_FFMA_CONTRACTIONS rules out the
// wgmma kernels, HB_KS_WIDE the wgmma and FFMA ones.  A stage that runs from logits takes k_logits_tc where it fits
// (not under HB_KS_WIDE), else the d-chunked k_logits_wide.  The plan-order cold start has no FFMA kernel: it runs
// from logits where k_logits_tc is among the wgmma kernels or the natural-order assignment runs from logits.
KernelPaths select_kernels(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set) {
  const int KS = (K + 3) & ~3, KD = (d + 7) & ~7, NP = (K + 15) & ~15;
  KernelPaths p;
  p.tuple_ranges = 2 * J <= num_sms;
  if (kernel_set & HB_KS_UPDATE_PER_STEP)
    p.update = UpdatePath::PerStep;
  else if (!(kernel_set & HB_KS_UPDATE_TWO_PASS) && p.tuple_ranges && sp_ring_rows(KS, SMEM_LIMIT) > 0 &&
           (uint64_t)n * (uint64_t)KS < (1ull << 32))
    p.update = UpdatePath::SinglePass;
  else if (KS <= 256 && J <= 8192 && two_pass_smem_bytes(KS, nb, J) <= SMEM_LIMIT)
    p.update = UpdatePath::TwoPass;
  const bool wide = kernel_set & HB_KS_WIDE;
  const bool tc = !(kernel_set & (HB_KS_FFMA_CONTRACTIONS | HB_KS_WIDE));
  const bool logits_tc = !wide && logits_tc_fits(d);
  if (tc) {
    const int ns = assign3_smem_bytes(2, KD, NP, KS) <= SMEM_LIMIT ? 2 : 1;
    if (d <= 64 && K <= 128 && assign3_smem_bytes(ns, KD, NP, KS) <= SMEM_LIMIT) p.k1_stages = ns;
  }
  if (p.k1_stages) {
    p.assign = Assign::FusedTc;
    p.cold = ColdStart::FusedTc;
  } else {
    if (wide || !assign_ffma_fits(K, d)) p.assign = logits_tc ? Assign::LogitsTc : Assign::LogitsWide;
    if ((tc && logits_tc) || p.assign != Assign::Ffma) p.cold = logits_tc ? ColdStart::LogitsTc : ColdStart::LogitsWide;
  }
  if (tc && apply_tc_fits(d))
    p.apply = Apply::Tc;  // cluster ranges of <= AP_MAXK per launch
  else if (wide || !apply_ffma_fits(K, d))
    p.apply = Apply::TcCols;
  if (tc && logits_tc && KS <= 256)
    p.kmeans = KmeansInit::LogitsTc;
  else if (wide || !kmeans_ffma_fits(K, d))
    p.kmeans = logits_tc ? KmeansInit::LogitsTc : KmeansInit::LogitsWide;
  return p;
}

// The update_R path of a cluster_cpp call of T rounds, and whether a cold-start assignment runs in the order of round
// 0 of the plan (and hands that round's removal sums to the single-pass kernel) instead of in natural order.  The
// two-pass kernel keeps its R-store rounds in a 32-bit mask: longer calls run per step, like every call with the
// legacy centroid step.
struct CallPath {
  UpdatePath update;
  bool plan_order_assign;
};
CallPath call_path(const KernelPaths& p, unsigned T, bool legacy_centroid) {
  CallPath c{p.update, false};
  if (legacy_centroid || (p.update == UpdatePath::TwoPass && T > 31)) c.update = UpdatePath::PerStep;
  c.plan_order_assign = c.update == UpdatePath::SinglePass && p.cold != ColdStart::None && T > 0;
  return c;
}

// ---- the sweep (knn.cuh): hb_knn, hb_lisi, hb_kbet, hb_silhouette -----------------------------------------------------
// Query rows per CTA (tq) and operand stages of the reference tiles (KNN_TN rows each) of a sweep whose kernel keeps
// row_bytes of shared memory per query row past the pipeline, and the CTA's bytes.  The first of (128, 2), (128, 1),
// (64, 2), (64, 1) that fits: the query tile and whatever the kernel keeps per row stay for the CTA's life, so wide rows
// and long lists take the memory from the second reference stage first and from the query tile last (a 64-row tile
// halves the flop per reference byte and runs one warpgroup).
struct SweepShape {
  int tq = 0, stages = 0;
  size_t smem = 0;
};
SweepShape sweep_shape(int KD, size_t row_bytes) {
  SweepShape g;
  static const int shapes[4][2] = {{128, 2}, {128, 1}, {64, 2}, {64, 1}};
  for (const auto& s : shapes)
    if (sweep_smem_bytes(s[0], s[1], KD) + s[0] * row_bytes <= SMEM_LIMIT) {
      g.tq = s[0], g.stages = s[1];
      break;
    }
  g.smem = sweep_smem_bytes(g.tq, g.stages, KD) + g.tq * row_bytes;
  return g;
}

// Launch geometry of the k-nearest-neighbour sweep: sweep_shape for k_knn_tc's lists, and reference splits.  (64, 2)
// holds d = 128, k = 64; (64, 1), reached only by hb_lisi's k > 64, holds d = 128, k = KNN_SWEEP_MAX_K.  With fewer
// query tiles than SMs the reference is split over grid.y so that the GPU is full, as far as k_knn_merge's candidate
// limit and the reference's tiles allow.
struct KnnGeometry {
  int tq = 0, stages = 0, splits = 0, KD = 0;
  size_t smem = 0;
  int64_t qtiles = 0, tiles_per_split = 0;
};
bool knn_fits(int d, int k) { return d >= 1 && d <= KNN_MAX_D && k >= 1 && k <= KNN_MAX_K; }
KnnGeometry knn_geometry(int d, int k, int64_t Nq, int64_t Nx, int num_sms) {
  KnnGeometry g;
  g.KD = (d + 7) & ~7;
  const SweepShape s = sweep_shape(g.KD, knn_row_bytes(k));
  g.tq = s.tq, g.stages = s.stages, g.smem = s.smem;
  g.qtiles = (Nq + g.tq - 1) / g.tq;
  const int64_t xtiles = (Nx + KNN_TN - 1) / KNN_TN;
  int64_t splits = 1;
  if (g.qtiles < num_sms) splits = std::max<int64_t>(1, std::min<int64_t>({num_sms / g.qtiles, xtiles, KNN_MERGE_MAX / k}));
  g.tiles_per_split = (xtiles + splits - 1) / splits;
  g.splits = (int)((xtiles + g.tiles_per_split - 1) / g.tiles_per_split);  // no empty split
  return g;
}

}  // namespace
