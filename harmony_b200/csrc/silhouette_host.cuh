// silhouette_host.cuh — hb_silhouette (DESIGN §11): the checks and the launches of silhouette.cuh: the (group, label)
// index, sorted preparation and finite counts (pair_index, score_host.cuh), the tile list and the sweep.  The call needs
// no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// Launch geometry of k_silhouette_tc: sweep_shape (select.cuh) of the pipeline alone, which is (128, 2) for every
// d <= 128
struct SilGeometry {
  int tq = 0, stages = 0, KD = 0;
  size_t smem = 0;
};
SilGeometry sil_geometry(int d) {
  SilGeometry g;
  g.KD = (d + 7) & ~7;
  const SweepShape s = sweep_shape(g.KD, 0);
  g.tq = s.tq, g.stages = s.stages, g.smem = s.smem;
  return g;
}

// The eight values of hb_debug_silhouette_geometry
void sil_geometry_record(int d, int64_t N, int num_sms, int64_t out[8]) {
  const SilGeometry g = sil_geometry(d);
  const int64_t tiles = (N + g.tq - 1) / g.tq;
  const int64_t v[8] = {g.tq, KNN_TN, g.stages, (int64_t)g.smem, g.KD, 2 * g.tq, tiles, (tiles + num_sms - 1) / num_sms};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
}

// The tiles of <= tq sorted rows, none across a group, largest group first: {first row, end row, first pair, end
// pair of the group}.  Pair q belongs to group uniq[q] / n_labels (group most significant in the key).
std::vector<int4> sil_tiles(const TupleIndex& ti, int n_labels, int tq) {
  struct Group {
    int p0, p1;
    int64_t rows;
  };
  std::vector<Group> gs;
  const int J = (int)ti.uniq.size();
  for (int q = 0; q < J;) {
    int e = q + 1;
    while (e < J && ti.uniq[e] / n_labels == ti.uniq[q] / n_labels) ++e;
    gs.push_back({q, e, ti.tstart[e] - ti.tstart[q]});
    q = e;
  }
  std::stable_sort(gs.begin(), gs.end(), [](const Group& a, const Group& b) { return a.rows > b.rows; });
  std::vector<int4> tiles;
  for (const Group& g : gs)
    for (int64_t r = ti.tstart[g.p0]; r < ti.tstart[g.p1]; r += tq)
      tiles.push_back(make_int4((int)r, (int)std::min<int64_t>(r + tq, ti.tstart[g.p1]), g.p0, g.p1));
  return tiles;
}

// The whole call on h->stream, for arguments the caller has checked
int silhouette_run(hb_handle* h, const DevRows& X, int d, const int32_t* labels, int n_labels, const int32_t* groups,
                   int n_groups, double* s_out) {
  ScoreScratch& s = score_scratch(h);
  const SilGeometry g = sil_geometry(d);
  TupleIndex ti;
  static const char* const names[2] = {"hb_silhouette: groups", "hb_silhouette: labels"};
  TRY(pair_index(h, X, d, g.KD, groups, n_groups, labels, n_labels, names, ti));
  // ---- the sweep
  const std::vector<int4> tiles = sil_tiles(ti, n_labels, g.tq);
  CK(s.tiles.reserve(tiles.size()));
  TRY(upload_vector(h, s.tiles, tiles));
  SilArgs a{s.rows.p, s.hx.p, s.pstart.p, s.count.p, s.tiles.p, s.sort_perm.p, s_out, g.KD, g.stages};
  const dim3 grid((unsigned)tiles.size());
  if (g.tq == 128) return launch(h, k_silhouette_tc<128>, grid, dim3(256), g.smem, a);
  return launch(h, k_silhouette_tc<64>, grid, dim3(128), g.smem, a);
}

int run_silhouette(hb_handle* h, const DevRows& X, int d, const int32_t* labels, int n_labels, const int32_t* groups,
                   int n_groups, double* s, cudaStream_t caller) {
  TRY(check_score_shape(h, "hb_silhouette", X.n, d));
  if (n_labels < 1) return fail(h, 2, "hb_silhouette: n_labels = %d, at least one label is needed", n_labels);
  if (groups && n_groups < 1) return fail(h, 2, "hb_silhouette: n_groups = %d, at least one group is needed", n_groups);
  if (!groups) n_groups = 1;
  if (n_labels > X.n || n_groups > X.n)
    return fail(h, 2, "hb_silhouette: %d labels and %d groups, more codes than the N = %lld rows", n_labels, n_groups, (long long)X.n);
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, labels, "labels"));
  if (groups) TRY(check_device_ptr(h, groups, "groups"));
  TRY(check_device_ptr(h, s, "s"));
  return run_score(h, caller, "silhouette",
                   [&] { return silhouette_run(h, X, d, labels, n_labels, groups, n_groups, s); });
}

}  // namespace
