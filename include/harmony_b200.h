/* harmony_b200.h — C ABI of libharmony_b200.so: the H100 (sm_90a) implementation of the Harmony
 * hot loop.  One opaque handle == one instance of the reference's C++ class `harmony`
 * (/root/reference/src/harmony.h:20-70); every entry point below replaces the like-named method /
 * field that the reference exposes to R through its Rcpp module (`RCPP_MODULE(harmony_module)`,
 * /root/reference/src/harmony.cpp:672-709).  INTEGRATION.md shows the Rcpp shim that binds them.
 *
 * Conventions
 *   - plain C types only; the library never throws.  Functions returning `int` give 0 on success,
 *     >0 on error (message via hb_last_error), and hb_cluster additionally -1 for "aborted by
 *     user" exactly like harmony::cluster_cpp (/root/reference/src/harmony.cpp:233-234).
 *   - matrices cross the boundary in the reference's layout: column-major with cells as columns
 *     (Z is d x N, R is K x N, Y is d x K, O/E are K x B, lambda matrix is K x (B+1)), doubles,
 *     i.e. exactly the memory of the R numeric matrices the reference takes and returns.
 *   - the sparse design matrix Phi (B x N dgCMatrix, /root/reference/R/ui.R:210-213) is passed as its
 *     row-index slot: every column has exactly C non-zeros (one level per covariate), so
 *     phi_i[n*C + c] is the (global, 0-based) row of the c-th non-zero of column n.
 *   - all buffers are caller-owned host memory; inputs are copied during the call
 *     (like harmony::setup, harmony.cpp:41,44), outputs are written into caller-allocated arrays.
 *     The exceptions are hb_setup_device and hb_get_field_device, which take the per-cell matrices
 *     (and, for hb_setup_device, optionally the labels phi_i) in the caller's device memory (fp32 or
 *     fp64, any row stride) and order themselves on a caller's CUDA stream.
 *   - a handle must be driven from one host thread at a time (the reference is single-threaded).
 */
#ifndef HARMONY_B200_H
#define HARMONY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hb_handle hb_handle;

/* ---- lifetime: `new(harmony)` (R/ui.R:269) / the external-pointer finaliser ------------------- */
/* device < 0 selects the current CUDA device. */
int hb_create(hb_handle** out, int device);
void hb_destroy(hb_handle* h);
/* Last error text of this handle ("" if none); valid until the next call on the handle. */
const char* hb_last_error(const hb_handle* h);
/* Pops one pending warning (e.g. "Too few cells. Setting block_size to 0.2", harmony.cpp:86-88) into
 * buf; returns 1 if a warning was written, 0 if none is pending.  The shim turns it into Rcpp::warning. */
int hb_pop_warning(hb_handle* h, char* buf, size_t cap);
/* Library/ABI version: major*10000 + minor*100 + patch (0.3.0: labels in device memory; 0.4.0: mapping a query onto
 * a reference, hb_reference / hb_map_setup / hb_map).  hb_knn, hb_debug_knn_geometry, hb_lisi,
 * hb_debug_lisi_geometry, hb_silhouette, hb_debug_silhouette_geometry, hb_graph_components, hb_kbet,
 * hb_debug_chi2_sf, hb_pcr, hb_debug_sym_eig, hb_kmeans, hb_umap_graph and hb_leiden were added without moving the
 * number. */
int hb_version(void);

/* ---- multi-GPU (one process per GPU; cells sharded contiguously; SURVEY §8e) ------------------- */
/* Size of the opaque communicator id (an ncclUniqueId). */
#define HB_COMM_ID_BYTES 128
/* Rank 0 creates the id and ships it to the other ranks by any host-side means (the Python host uses
 * torch.distributed); every rank then calls hb_comm_init BEFORE hb_setup. */
int hb_comm_unique_id(char id[HB_COMM_ID_BYTES]);
int hb_comm_init(hb_handle* h, int rank, int world_size, const char id[HB_COMM_ID_BYTES]);
/* The communicator stays alive for the life of the process; a later handle of the same (device, rank,
 * world_size) may pass id == NULL to share it instead of paying the ~1 s NCCL set-up again. */
/* Declares that this handle holds cells [cell_offset, cell_offset + n_local) of an N_global-cell
 * problem.  Must precede hb_setup; without it the handle owns all cells. */
int hb_set_shard(hb_handle* h, int64_t N_global, int64_t cell_offset);

/* ---- harmony::setup (harmony.h:25-30, harmony.cpp:29-111; called at R/ui.R:271-275) ---------- */
/* Z: d x N(local) column-major doubles.  lambda: B+1 values, or NULL / lambda[0] == -1 for the
 * reference's automatic estimation (harmony.cpp:75-76).  Errors: N < 6 -> status 1 with the
 * reference's message (harmony.cpp:83-85); 6 <= N < 40 -> warning + block_size 0.2 (:86-88).
 * phi_i must be host (or managed) memory: there is no stream to order a device read against; a device
 * pointer -> status 2 before any launch.  The covariate-tuple index (cells stably sorted by their tuple
 * of levels) is built on the device from either. */
int hb_setup(hb_handle* h, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
             const double* sigma, const double* theta, const double* lambda, double alpha, int max_iter_kmeans,
             double epsilon_kmeans, double epsilon_harmony, int K, double block_size,
             double batch_proportion_cutoff, int verbose);

/* Element types of device-memory matrices (hb_setup_device, hb_get_field_device). */
enum hb_dtype { HB_FLOAT32 = 0, HB_FLOAT64 = 1 };

/* hb_setup with Z in device memory: N(local) rows of d values of z_dtype, row stride z_ld >= d elements (the bytes of a
 * d x N column-major matrix when z_ld == d), in device or managed memory of the handle's device.  phi_i may lie in
 * host memory or in device or managed memory of the handle's device; every other argument is hb_setup's, on the host.
 * Z and a device phi_i are read after the work already queued on `stream` (a cudaStream_t; NULL: the legacy default
 * stream) and the call returns once they have been copied.  Status 2 before any launch for a NULL, host or
 * other-device Z, an other-device phi_i, an unknown dtype or z_ld < d. */
int hb_setup_device(hb_handle* h, const void* Z, int z_dtype, int64_t z_ld, void* stream, int d, int64_t N,
                    const int32_t* phi_i, const int32_t* B_vec, int C, const double* sigma, const double* theta,
                    const double* lambda, double alpha, int max_iter_kmeans, double epsilon_kmeans,
                    double epsilon_harmony, int K, double block_size, double batch_proportion_cutoff, int verbose);

/* Seed of the native generators (k-means initialisation, per-round update orders).  The reference
 * draws both from R's RNG (utils.cpp:10-64, harmony.cpp:272-273); the shim may instead inject them. */
int hb_set_seed(hb_handle* h, uint64_t seed);
/* Polled between clustering rounds like Progress::check_abort() (harmony.cpp:233); non-zero -> -1. */
int hb_set_abort_callback(hb_handle* h, int (*cb)(void*), void* user);

/* ---- harmony::init_cluster_cpp (harmony.cpp:131-156) ------------------------------------------ */
/* Y0: d x K column-major initial centroids (what kmeans_centers returns, harmony.cpp:133), or NULL to
 * run the native GPU k-means initialisation. */
int hb_init_cluster(hb_handle* h, const double* Y0);

/* ---- harmony::cluster_cpp (harmony.cpp:208-262) incl. update_R (:269-342) --------------------- */
/* update_orders: max_iter_kmeans x N_global int64 — row t is the `update_order` that
 * arma::shuffle would produce for the t-th update_R call (harmony.cpp:272-273) — or NULL to draw the
 * orders natively on the device.  Returns 0, -1 (aborted) or >0 (error). */
int hb_cluster(hb_handle* h, const int64_t* update_orders);

/* ---- harmony::moe_correct_ridge_cpp (harmony.cpp:345-638) -------------------------------------- */
int hb_moe_correct_ridge(hb_handle* h);

/* ---- harmony::check_convergence (harmony.cpp:173-205): 1 = converged, 0 = not, <0 = error ----- */
int hb_check_convergence(hb_handle* h, int type);

/* ---- harmony::compute_objective (harmony.cpp:158-170): appends to the four objective traces --- */
int hb_compute_objective(hb_handle* h);

/* ---- mapping a query onto a finished integration (DESIGN.md §8) -------------------------------- */
/* The compression of the integration the handle holds (any state after hb_init_cluster), per cluster k, from the
 * Z_corr getZcorr() returns and R: Nr[k] = sum_n R[k,n], Cref[:,k] = sum_n R[k,n] Z_corr[:,n], centroids[:,k] =
 * Cref[:,k] / |Cref[:,k]| (a zero column stays zero), and sigma.  centroids and Cref are d x K column-major, Nr and
 * sigma K values; NULL outputs are skipped.  Status 3 before hb_init_cluster, on a sharded handle (world > 1) and on a
 * mapping handle.  Region "reference". */
int hb_reference(hb_handle* h, double* centroids, double* Nr, double* Cref, double* sigma);
/* Sets a handle up to map Nq query cells onto a reference, instead of hb_setup.  Z: d x Nq column-major doubles in the
 * reference's PC space; phi_i / B_vec / C: the query's own covariates (hb_setup's form, B_q = sum(B_vec) levels);
 * lambda: B_q ridge penalties, one per query level, finite and > 0; K, centroids, Nr, Cref, sigma: hb_reference's
 * output.  Any Nq >= 1.  Status 2 for a NULL argument, bad dimensions, lambda <= 0 or non-finite, sigma non-finite or
 * <= 0, Nr < 0, non-finite centroids or Cref, or labels outside their covariate's levels; status 3 if the handle already
 * ran a setup or is sharded (hb_comm_init with world > 1, or hb_set_shard).  HB_KERNEL_SET is read here as in hb_setup.
 * phi_i must be host or managed memory. */
int hb_map_setup(hb_handle* h, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
                 const double* lambda, int K, const double* centroids, const double* Nr, const double* Cref,
                 const double* sigma);
/* hb_map_setup with Z (and optionally phi_i) in device memory, with hb_setup_device's dtype, row stride, stream and
 * pointer conventions and checks. */
int hb_map_setup_device(hb_handle* h, const void* Z, int z_dtype, int64_t z_ld, void* stream, int d, int64_t N,
                        const int32_t* phi_i, const int32_t* B_vec, int C, const double* lambda, int K,
                        const double* centroids, const double* Nr, const double* Cref, const double* sigma);
/* Maps the query of a handle set up by hb_map_setup*: R_q = softmax_k(-2 (1 - Yref_k . z_n / |z_n|) / sigma_k), then
 * one ridge correction per cluster in which Nr_k and Cref_k anchor the intercept and only the query's level terms are
 * fitted (no level filter, fixed lambda, the centroids unchanged).  Afterwards HB_Z_CORR is the mapped embedding
 * (hb_get_field and hb_get_field_device), HB_Z_ORIG the input, HB_R R_q, HB_Y the reference's centroids and HB_SIGMA
 * its sigma.  Repeatable.  Status 3 on a handle set up by hb_setup.  On a mapping handle hb_init_cluster, hb_cluster,
 * hb_moe_correct_ridge, hb_compute_objective, hb_check_convergence, hb_set_field and the fields HB_W, HB_THETA and
 * HB_LAMBDA return status 3.  Regions "assign", "ridge_stats", "ridge_solve", "ridge_apply". */
int hb_map(hb_handle* h);

/* ---- exact k nearest neighbours in an embedding (DESIGN.md §9) ---------------------------------- */
enum hb_metric { HB_EUCLIDEAN = 0, HB_COSINE = 1 };
/* For every one of the Nq rows of Q the k rows of X at the smallest distance, by brute force over all pairs:
 * idx[Nq][k] (0-based rows of X) and, unless NULL, dist[Nq][k], each row by ascending distance.  Q and X: rows of d values
 * of q_dtype / x_dtype (hb_dtype) with row strides q_ld, x_ld >= d elements; Q, X, idx and dist in device or managed
 * memory of the handle's device.  fp64 values are rounded to fp32 after centring (Euclidean) and before normalising.
 * metric: HB_EUCLIDEAN (dist is the distance, not its square) or HB_COSINE (dist = 1 - cos; a zero row divides by 1 and
 * so lies at distance 1 from every row).  exclude_self: row i of X is no candidate for row i of Q (a search of an
 * embedding against itself).  The candidates are selected on 3xTF32 scores and the winners' distances recomputed directly
 * in fp32, so dist is accurate per pair and only the membership of rows within a narrow band of the k-th distance is
 * subject to rounding (DESIGN.md §9 gives the band); among exact duplicates any may be returned, no row twice.  A pair
 * whose fp32 distance is NaN or infinite is never returned; a query row with fewer than k returnable rows ends with
 * idx = -1, dist = +inf.
 * Limits, status 2 with a message before any launch: 1 <= k <= 64, k <= Nx (Nx - 1 with exclude_self), 1 <= d <= 128,
 * Nq >= 1, Nx < 2^31, an unknown metric or dtype, a row stride < d, a NULL, host or other-device pointer.
 * Q and X are read after the work queued on `stream` (a cudaStream_t; NULL: the legacy default stream) and work queued on
 * `stream` afterwards sees idx and dist; the host is not blocked.  Needs no setup: it runs on a fresh handle, on one that
 * is running Harmony and on a mapping handle, whose state it leaves untouched; its scratch stays with the handle.  On a
 * sharded handle it is a local call.  Region "knn". */
int hb_knn(hb_handle* h, const void* Q, int q_dtype, int64_t q_ld, int64_t Nq, const void* X, int x_dtype, int64_t x_ld,
           int64_t Nx, int d, int k, int metric, int exclude_self, int32_t* idx, float* dist, void* stream);
/* Test hook (host only): the launch geometry hb_knn picks for (d, k, Nq, Nx) on num_sms SMs: out = {query rows per CTA,
 * reference rows per tile, reference operand stages, reference splits (grid.y; > 1 when the query tiles alone would not
 * fill the GPU), shared-memory bytes, reference tiles per split, padded row length in floats, threads per CTA}.
 * Returns 0, or 2 with out untouched for a d or k hb_knn refuses. */
int hb_debug_knn_geometry(int d, int k, int64_t Nq, int64_t Nx, int num_sms, int64_t out[8]);
/* LISI, the Local Inverse Simpson's Index (DESIGN.md §10), of every row of X [N, d] for n_sets label sets: with the
 * k = floor(3 perplexity) - 1 nearest other rows by Euclidean distance D_j (hb_knn's search with exclude_self), weights
 * P_j ~ exp(-beta D_j) with beta bisected in fp64 until the entropy is within 1e-5 of ln(perplexity) (at most 50
 * evaluations), and lisi[i][s] = 1 / sum over the labels of set s of (sum of P_j over the neighbours with that label)^2:
 * the effective number of labels around row i.  -1 for a row whose final entropy is exactly 0; NaN for a row without a
 * neighbour (every row with a non-finite value).  labels: n_sets rows of labels_ld >= N int32 codes, set s of row j at
 * labels[s * labels_ld + j]; codes are arbitrary, only equality counts.  lisi [N][n_sets] fp64; idx [N][k] and dist
 * [N][k] (as hb_knn returns them) when not NULL.  X of x_dtype (hb_dtype) with row stride x_ld >= d.
 * Limits, status 2 with a message before any launch: a finite perplexity >= 1, k <= 128 (perplexity < 43 1/3),
 * k <= N - 1, N < 2^31, 1 <= d <= 128, n_sets >= 1, labels_ld >= N, an unknown dtype, a row stride < d, a NULL (X,
 * labels, lisi), host or other-device pointer.  Ordered on `stream` like hb_knn; needs no setup and leaves a Harmony or
 * mapping handle's state untouched.  Region "lisi". */
int hb_lisi(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* labels,
            int64_t labels_ld, int n_sets, double perplexity, double* lisi, int32_t* idx, float* dist, void* stream);
/* Test hook (host only): hb_debug_knn_geometry's eight values for hb_lisi's search of N rows at this perplexity on
 * num_sms SMs.  Returns 0, or 2 with out untouched for a d, perplexity or N hb_lisi refuses. */
int hb_debug_lisi_geometry(int d, double perplexity, int64_t N, int num_sms, int64_t out[8]);
/* Silhouette widths (DESIGN.md §11) of every row of X [N, d] with labels[i] in 0..n_labels-1 and, when groups is not
 * NULL, groups[i] in 0..n_groups-1 (int32 device arrays of N codes; no groups: one group).  Only rows of one group
 * interact, and only finite rows take part (a row with a NaN or an infinity, or whose centred |x - c|^2 overflows fp32,
 * gets NaN and is nobody's neighbour).  With D the Euclidean distance and n the finite rows of row i's (group, label):
 * a = sum of D to the other rows of its (group, label) / (n - 1), b = the smallest mean of D to the rows of another
 * label of its group that has a finite row, s[i] = (b - a) / max(a, b) (0 when that is 0); 0 when n = 1, NaN when its
 * group has no other such label.  Without groups this is sklearn.metrics.silhouette_samples.  s [N] fp64 in the
 * caller's order.  X of x_dtype (hb_dtype) with row stride x_ld >= d.  Limits, status 2 with a message before any
 * launch: 2 <= N < 2^31, 1 <= d <= 128, n_labels >= 1, n_groups >= 1 when groups are given, n_labels and n_groups
 * <= N, an unknown dtype, a row stride < d, a NULL (X, labels, s), host or other-device pointer; a code out of range
 * is status 2 naming the cell, found before the sweep.  Ordered on `stream` like hb_knn; needs no setup and leaves a
 * Harmony or mapping handle's state untouched; on a sharded handle the call is local.  Region "silhouette". */
int hb_silhouette(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* labels,
                  int n_labels, const int32_t* groups, int n_groups, double* s, void* stream);
/* Test hook (host only): the launch geometry of hb_silhouette's sweep for (d, N) on num_sms SMs: out = {rows per query
 * tile, reference rows per tile, operand stages, shared-memory bytes, padded row length in floats, threads per CTA,
 * query tiles of N rows in one group, waves of those tiles}.  Returns 0, or 2 with out untouched for a d or N
 * hb_silhouette refuses. */
int hb_debug_silhouette_geometry(int d, int64_t N, int num_sms, int64_t out[8]);
/* Connected components of a neighbour graph (DESIGN.md §12).  idx [N][k] int32 with row stride idx_ld >= k: entry j of
 * row i is the undirected edge {i, j}, -1 is no neighbour (hb_knn's fill); self and repeated entries add nothing.  With
 * labels (int32 [N], codes 0..n_labels-1) an edge is kept only between rows of one label, so components never cross
 * labels; labels NULL keeps every edge and ignores n_labels.  comp [N]: the smallest row of each row's component (the
 * same whatever order the union-find runs in).  largest (NULL: not computed): [n_labels] (one entry without labels), the
 * size of the largest component among the rows of each label, 0 for a code no row has.  All pointers in device or
 * managed memory of the handle's device.  Limits, status 2 with a message before any launch: 1 <= N < 2^31, k >= 1,
 * idx_ld >= k, 1 <= n_labels <= N when labels are given, a NULL (idx, comp), host or other-device pointer.  An entry
 * outside -1..N-1 or a code outside 0..n_labels-1 is status 2 naming the row and the entry, found by a read-only pass
 * before comp and largest are written.  Ordered on `stream` like hb_knn; needs no setup and leaves a Harmony or mapping
 * handle's state untouched; on a sharded handle the call is local.  Region "components". */
int hb_graph_components(hb_handle* h, const int32_t* idx, int64_t idx_ld, int64_t N, int k, const int32_t* labels,
                        int n_labels, int32_t* comp, int32_t* largest, void* stream);
/* kBET (DESIGN.md §13): for every row of X [N, d], a chi-square test of the batches among the row and its k0 - 1 nearest
 * other rows of its label against the label's batch frequencies.  batches: int32 codes 0..n_batches-1; labels (NULL:
 * one label): int32 codes 0..n_labels-1; both device arrays of N codes.  Only finite rows take part, as in
 * hb_silhouette.  Per label l with n_l finite rows, n_{l,b} of them in batch b and B_l batches with n_{l,b} > 0: not
 * tested when n_l < 10, B_l = 1 or (fixed k0) n_l < k0; else k0_l = k0, or for k0 = 0 scib's rule min(70, max(10,
 * floor(n_l / B_l / 4))), lowered to floor((2^31 - 1) / n_l) where k0_l n_l would reach 2^31 - 1.  For a finite row i of
 * a tested label: the row and its k0_l - 1 nearest other finite rows of its label by Euclidean distance (hb_knn's search
 * and band), o_b their batch counts, stat[i] = sum_b (o_b - k0_l p_b)^2 / (k0_l p_b) with p_b = n_{l,b} / n_l, and
 * pval[i] = Q((B_l - 1) / 2, stat[i] / 2), the chi-square upper tail with B_l - 1 degrees of freedom, in fp64.  Other
 * rows get NaN.  stat and pval [N] fp64 in the caller's order; k0_out (NULL: skipped) [n_labels] (1 without labels),
 * 0 for a label not tested; idx (NULL: skipped) [N][idx_ld] int32: a tested row's k0_l - 1 neighbours (caller's rows)
 * by ascending distance, -1 after them and for every other row.  X of x_dtype (hb_dtype) with row stride x_ld >= d.
 * Limits, status 2 with a message before any launch: 2 <= N < 2^31, 1 <= d <= 128, n_batches >= 1, n_labels >= 1 when
 * labels are given, n_batches and n_labels <= N, k0 = 0 or 2 <= k0 <= 129, an unknown dtype, a row stride < d, a NULL
 * (X, batches, stat, pval), host or other-device pointer.  Status 2 after the index pass, before any output is written:
 * a code out of range (naming the cell), more than 1e6 (label, batch) pairs, idx_ld below the largest k0_l - 1.
 * Ordered on `stream` like hb_knn; needs no setup and leaves a Harmony or mapping handle's state untouched; on a
 * sharded handle the call is local; two calls give bit-identical results.  Region "kbet". */
int hb_kbet(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* batches,
            int n_batches, const int32_t* labels, int n_labels, int k0, double* stat, double* pval, int32_t* k0_out,
            int32_t* idx, int64_t idx_ld, void* stream);
/* Test hook (host only): the p-value function of hb_kbet, the chi-square upper tail of x with dof degrees of freedom,
 * into *out.  Returns 0, or 2 with out untouched for dof < 1. */
int hb_debug_chi2_sf(double x, int dof, double* out);
/* Principal component regression (DESIGN.md §14): the share of X's variance that its batches explain, scib's pcr.
 * X [N, d] of x_dtype (hb_dtype) with row stride x_ld >= d; batches: int32 device codes 0..n_batches-1, one per row.
 * Only finite rows take part (n of them, n_b in batch b).  With m the column mean over finite rows and
 * C = sum (x - m)(x - m)^T, the components are C's m_c = min(n_comps, N, d) leading eigenpairs (lambda_j, v_j) in
 * descending order, v_j's entry of largest magnitude positive (the first on a tie); var[j] = lambda_j / (n - 1),
 * components[j][.] = v_j, and r2[j] = sum_b (S_b . v_j)^2 / n_b / lambda_j clamped to [0, 1] with
 * S_b = sum over batch b of (x - m): the R^2 of regressing PC j on the one-hot batches.  r2[j] = 0 when
 * lambda_j <= d eps lambda_1 or fewer than two batches have finite rows.  score = sum_j r2[j] lambda_j / sum_j lambda_j.
 * n < 2: var, r2 and score are NaN; sum_j lambda_j = 0: score is NaN.  Outputs are fp64 device arrays: var and r2
 * [m_c], components [m_c][d] (NULL: skipped), score [1].  Limits, status 2 with a message before any launch:
 * 2 <= N < 2^31, 1 <= d <= 128, 1 <= n_batches <= N, n_comps >= 1, an unknown dtype, a row stride < d, a NULL (X,
 * batches, var, r2, score), host or other-device pointer.  Status 2 after the index pass, before any output is
 * written: a batch code out of range (naming the cell).  Ordered on `stream` like hb_knn; needs no setup and leaves a
 * Harmony or mapping handle's state untouched; on a sharded handle the call is local; two calls give bit-identical
 * results.  Region "pcr". */
int hb_pcr(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* batches,
           int n_batches, int n_comps, double* var, double* r2, double* components, double* score, void* stream);
/* Test hook (host only): hb_pcr's eigensolver on the symmetric n x n host matrix A (row-major, upper triangle read):
 * the eigenvalues in descending order into w [n] and V [n][n] row-major with column j the unit eigenvector of w[j],
 * signed as hb_pcr's components.  Returns 0, or 2 with the outputs untouched for n outside 1..128. */
int hb_debug_sym_eig(int n, const double* A, double* w, double* V);

/* k-means of an embedding (DESIGN.md §15), the clustering behind the NMI / ARI scores: K clusters of the finite rows of
 * X [N, d] (x_dtype, row stride x_ld >= d; a row with a NaN or an infinity takes no part and gets label -1).  n_init
 * inits; each is seeded by greedy k-means++ (2 + floor(ln K) candidates per round, drawn with probability ~ D^2 by
 * keyed-hash exponential races under `seed`; the candidate of the smallest potential is kept) and iterated by Lloyd's
 * rule as sklearn's algorithm="lloyd" runs it: assign (the nearest centre by hb_knn's search, the lower index on an exact
 * tie), means of the members in fp64 (an empty cluster keeps its centre), stop when the labels repeat or when the
 * squared centre shift is <= tol times the mean column variance of the finite rows; after max_iter iterations without
 * repeated labels the rows are assigned once more.  max_iter = 0: the seeds' assignment.  Of the inits, the one of the
 * lowest inertia (sum of |x - c_label|^2 over finite rows, fp64), the earliest on a tie, gives labels [N] int32 and
 * centres [K][d] fp64; inertia [n_init] fp64 and n_iter [n_init] int32 are per init; seeds (NULL: skipped)
 * [n_init][K] int32 the seed rows.  All outputs in device memory.  Limits, status 2 with a message before any launch:
 * 1 <= N < 2^31, 1 <= d <= 128, 1 <= K <= min(N, 1024), n_init >= 1, max_iter >= 0, tol finite and >= 0, an unknown
 * dtype, a row stride < d, a NULL (X, labels, centres, inertia, n_iter), host or other-device pointer.  Status 3 with
 * the outputs untouched: fewer than K finite rows.  Status 2 after the first passes, the outputs untouched: a finite
 * row with |x - m|^2 > 2^124 for m the column mean (the assignment's fp32 scores would overflow).  Ordered on `stream` like hb_knn; needs no setup and leaves a
 * Harmony or mapping handle's state untouched; on a sharded handle the call is local; two calls give bit-identical
 * results.  Regions "kmeans" and, within it, "kmeans_seed". */
int hb_kmeans(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, int K, uint64_t seed,
              int n_init, int max_iter, double tol, int32_t* labels, double* centres, double* inertia, int32_t* n_iter,
              int32_t* seeds, void* stream);

/* scanpy's UMAP connectivities (umap-learn's fuzzy_simplicial_set, local_connectivity 1, set_op_mix_ratio 1; DESIGN
 * §16) of neighbour lists idx / dist [N][k] (hb_knn's with exclude_self: -1 / +inf fill, rows contiguous, idx_ld =
 * dist_ld = k <= 128) in device memory.  n_neighbors counts the cell itself (scanpy's, k + 1).  rho, sigma and the
 * weights in fp64; the symmetric union P = W + W^T - W o W^T as a CSR in the caller's device buffers: indptr int64
 * [N + 1], indices int32 (ascending within a row) and data fp32, each of at least 2 N k entries; *nnz (host) gets the
 * entries written.  No diagonal and no explicit zero.  Ordered on `stream`; needs no setup and touches no handle state;
 * two calls give bit-identical results.  Region "umap_graph". */
int hb_umap_graph(hb_handle* h, const int32_t* idx, int64_t idx_ld, const float* dist, int64_t dist_ld, int64_t N, int k,
                  int n_neighbors, int64_t* indptr, int32_t* indices, float* data, int64_t* nnz, void* stream);

/* Deterministic Leiden (DESIGN §16) of the symmetric CSR graph indptr int64 [N + 1] / indices int32 / data (dtype
 * HB_FLOAT32 or HB_FLOAT64, finite and > 0) in device memory, rows strictly ascending and no diagonal, for modularity
 * with resolution gamma (RBConfigurationVertexPartition).  A graph that breaks these is refused with status 2, naming
 * the row and entry, before any output is written.  labels int32 [N] (device): communities numbered by decreasing
 * size, ties by the smallest member row.  Host outputs: *n_communities, *quality (Q in fp64), *iterations; stats (NULL
 * or host int64 [3]): levels, local-moving sweeps and refinement rounds run.  n_iterations -1 repeats iterations until
 * no label changes (at most 64), else runs that many.  A reached cap leaves a warning (hb_pop_warning).  Ordered on
 * `stream`; needs no setup and touches no handle state; two calls give bit-identical results.  Regions "leiden" and,
 * within it, "leiden_move", "leiden_refine" and "leiden_aggregate". */
int hb_leiden(hb_handle* h, const int64_t* indptr, const int32_t* indices, const void* data, int dtype, int64_t N,
              int64_t nnz, double resolution, int n_iterations, int32_t* labels, int32_t* n_communities, double* quality,
              int32_t* iterations, int64_t* stats, void* stream);

/* ---- fields / getters (harmony.cpp:640-669, 675-696) ------------------------------------------- */
enum hb_field {
  HB_Z_CORR = 0, /* getZcorr(): d x N  */
  HB_Z_ORIG = 1, /* getZorig(): d x N  */
  HB_R = 2,      /* R / getR(): K x N  */
  HB_Y = 3,      /* Y / getCentroids(): d x K */
  HB_O = 4,      /* O: K x B */
  HB_E = 5,      /* E: K x B */
  HB_W = 6,      /* W: (B+1) x d, betas of the last corrected cluster (rows of dropped levels are 0) */
  HB_PR_B = 7,   /* Pr_b: B */
  HB_THETA = 8,  /* theta: B */
  HB_SIGMA = 9,  /* sigma: K */
  HB_LAMBDA = 10,    /* getLambda(): K x (B+1) */
  HB_LAMBDA_VEC = 11 /* lambda field: B+1 (only when not estimating) */
};
/* Number of doubles hb_get_field writes for `field` (0 for an unknown field). */
int64_t hb_field_size(const hb_handle* h, int field);
/* Device -> host copy-out with float -> double conversion (conv_to<RMAT>::from, harmony.cpp:640-650).
 * With a sharded handle the per-cell fields return the local shard. */
int hb_get_field(hb_handle* h, int field, double* out);
/* Device-memory hb_get_field for HB_Z_CORR, HB_Z_ORIG and HB_R: writes the N_local rows (cells in the caller's order) of
 * d or K values of `dtype` with row stride ld >= cols elements into `out`, device or managed memory of the handle's
 * device.  Does not block the host: the copy runs after the work queued on `stream` so far, and work queued on
 * `stream` afterwards sees the result.  Status 2 before any launch for a NULL, host or other-device `out`, another
 * field, an unknown dtype or ld < cols. */
int hb_get_field_device(hb_handle* h, int field, void* out, int dtype, int64_t ld, void* stream);
/* Writable fields (the Rcpp module's .field() members are read-write): HB_Y, HB_R, HB_O, HB_E,
 * HB_THETA, HB_SIGMA, HB_LAMBDA_VEC, HB_Z_CORR.  `in` holds hb_field_size(h, field) values.
 * A written HB_SIGMA takes effect at the next update_R and compute_objective, as in the reference, which keeps the
 * distances and divides by the current sigma (harmony.cpp:158-162, 318-319): the distances of the last assignment are
 * kept, divided by the new sigma.  Status 2 if a sigma value is not finite or not positive. */
int hb_set_field(hb_handle* h, int field, const double* in);

enum hb_scalar { HB_N = 0, HB_B = 1, HB_K = 2, HB_D = 3, HB_C = 4, HB_ALPHA = 5, HB_MAX_ITER_KMEANS = 6,
                 HB_BLOCK_SIZE = 7, HB_EPSILON_KMEANS = 8, HB_EPSILON_HARMONY = 9, HB_N_LOCAL = 10,
                 HB_LAMBDA_ESTIMATION = 11, HB_WINDOW_SIZE = 12, HB_LEGACY_CENTROID_STEP = 13, HB_KERNEL_SET = 14,
                 HB_DEVICE = 15 /* CUDA device of the handle (read-only) */ };
/* HB_KERNEL_SET (test hook, default 0, read by the next hb_setup): the library picks its kernels from the problem's
 * shape alone; these bits force the kernels that serve shapes outside the default ones' limits onto ANY shape so that
 * the parity suite can hold them to the same bar (tests/test_gpu_parity.py::test_fallback_kernels_match_oracle). */
enum hb_kernel_set { HB_KS_FFMA_CONTRACTIONS = 1, /* fp32 FFMA assignment / apply / k-means initialisation instead of wgmma */
                     HB_KS_UPDATE_PER_STEP = 2,   /* update_R in three launches per block step */
                     HB_KS_UPDATE_TWO_PASS = 4,   /* update_R in the two-pass persistent kernel (look-ahead + update groups) */
                     HB_KS_NO_PEER_EXCHANGE = 8,  /* sharded cells: one NCCL all-reduce per block step */
                     HB_KS_WIDE = 16              /* the kernels of the shapes past the FFMA kernels' shared-memory limits:
                                                     d-chunked logits + softmax passes for the assignment, column-range
                                                     ridge apply, k-means initialisation from those logits */ };
int hb_get_scalar(const hb_handle* h, int which, double* out);
/* Settable: HB_ALPHA, HB_MAX_ITER_KMEANS (vignettes/detailedWalkthrough.Rmd:364), HB_EPSILON_*, HB_KERNEL_SET and
 * HB_LEGACY_CENTROID_STEP (0/1): run STEP 1 of harmony::cluster_cpp — Y = normalise(Z_corr * R.t()),
 * dist_mat = 2 (1 - Y.t() Z_corr), harmony.cpp:235-238, commented out in 2.0.4 — at the top of every clustering
 * round, as the package version that rendered the reference's vignette did.  Compatibility path: one
 * statistics + assignment pass per round on top of the per-step update kernels. */
int hb_set_scalar(hb_handle* h, int which, double value);
/* B_vec field (harmony.cpp:683): writes C ints. */
int hb_get_B_vec(const hb_handle* h, int32_t* out);

enum hb_trace_id { HB_OBJECTIVE_KMEANS = 0, HB_OBJECTIVE_KMEANS_DIST = 1, HB_OBJECTIVE_KMEANS_ENTROPY = 2,
                   HB_OBJECTIVE_KMEANS_CROSS = 3, HB_OBJECTIVE_HARMONY = 4, HB_KMEANS_ROUNDS = 5 };
/* Trace vectors (harmony.h:55-56).  Returns the trace length; writes min(length, cap) values if out. */
int64_t hb_trace(const hb_handle* h, int trace, double* out, int64_t cap);

/* ---- instrumentation (src/timer.h regions -> CUDA-event timers) -------------------------------- */
/* Number of kernels this library has launched on the handle since creation. */
int64_t hb_kernel_launches(const hb_handle* h);
/* CUDA stream (cudaStream_t) all work of this handle is ordered on, for callers that time with events. */
void* hb_stream(const hb_handle* h);
/* Blocks until all queued work of the handle has finished; returns the sticky CUDA status as 0/>0. */
int hb_synchronize(hb_handle* h);
/* Accumulated device time (ms) and launch count of a named region ("assign", "update_R",
 * "ridge_stats", "ridge_solve", "ridge_apply", "plan", "upload" / "download": the per-cell row transfers of setup,
 * the getters and hb_set_field, host copies included, and "tuple_index": setup's covariate-tuple index, the upload
 * of host labels and the host's O(J) part included); returns 0 if the region exists. */
int hb_region_time(hb_handle* h, const char* region, double* ms, int64_t* launches);
/* Enables per-region CUDA-event timing (adds synchronisation; off by default). */
int hb_enable_timing(hb_handle* h, int on);
/* Test hook (host only, no GPU needed): position of cell i (inverse = 0) or the cell at position i
 * (inverse = 1) in the keyed pseudo-random order of n cells that replaces arma::shuffle (harmony.cpp:272-273)
 * when no update order is injected.  Returns ~0 for i >= n. */
uint64_t hb_debug_permute(uint64_t i, uint64_t n, uint64_t key, int inverse);
/* Test hook (host only): the host worker pool of the download path (hb_get_field) widens n floats to
 * doubles; `threads` sizes the pool on first use (<= 0: HB_HOST_THREADS or the core count).  Returns the pool size. */
int hb_debug_widen(double* out, const float* in, int64_t n, int threads);
/* Test hooks of the native kmeans_centers (hb_init_cluster(h, NULL); utils.cpp:10-64): the keyed-hash uniform that
 * stands in for arma::randu at (centroid i, global cell g) — i = K addresses the K start-cell draws — and the global
 * cells initialize_centroids chose (returns their number, 0 if the native initialisation has not run). */
double hb_debug_kmeans_uniform(const hb_handle* h, uint64_t i, uint64_t g);
int hb_debug_kmeans_cells(const hb_handle* h, int64_t* out);
/* Test hook: with on != 0, the native initialisations that follow record Y (K x d row-major floats) after the race's
 * gather (step 0) and after each of the 10 Lloyd steps (steps 1..10); each native initialisation clears the record
 * first, hb_init_cluster with Y0 records nothing.  hb_debug_kmeans_means copies the record (11 K d floats) and
 * returns its length, 0 if there is none.  Off by default. */
int hb_debug_kmeans_keep_means(hb_handle* h, int on);
int64_t hb_debug_kmeans_means(const hb_handle* h, float* out);
/* Test hook: the covariate-tuple index hb_setup built.  Returns J (the number of tuples; -1 before setup) and writes
 * the non-null outputs: sort_perm (N_local values: the caller's cell at each tuple-sorted position), tuple_levels
 * (J x C global levels, tuples in ascending mixed-radix order with covariate 0 most significant) and tuple_start
 * (J + 1 values: the first sorted position of each tuple, then N_local). */
int hb_debug_tuple_index(const hb_handle* h, int32_t* sort_perm, int32_t* tuple_levels, int64_t* tuple_start);
/* Test hook (host only): ring geometry of the persistent update_R kernel for rows of KS floats:
 * out = {float4 per lane, row groups per warp ring (a power of two), rows per group, shared-memory bytes, warps per
 * CTA, 0, 0, 0, 0}.  Returns 1 if the shape is supported, 0 if the library would use the other update kernels. */
int hb_debug_update_geometry(int KS, int nb, int64_t out[9]);
/* Test hook (host only): the kernels hb_setup picks for K clusters, d dimensions, J covariate tuples, n local cells,
 * nb update blocks on num_sms SMs under the HB_KERNEL_SET bits kernel_set:
 * out = {update_R path (0 per step, 1 two-pass, 2 single-pass), operand stages of the fused tensor-core assignment
 * (0: not fused), tensor-core logits for the plan-order assignment, tensor-core ridge apply, tensor-core k-means
 * initialisation, cold-start assignment of a 20-round cluster_cpp call in the plan's order, update_R path of a
 * 40-round call, update_R path of a call with HB_LEGACY_CENTROID_STEP}.  Returns 0. */
int hb_debug_kernel_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[8]);
/* Test hook (host only): the kernel of each stage whose FFMA kernel stops at a shared-memory limit, for the same
 * arguments: out = {natural-order assignment (1 fused wgmma, 2 FFMA, 3 wgmma logits + softmax pass, 4 d-chunked wgmma
 * logits + softmax pass), plan-order cold start of a 20-round call (0 natural order, 1 fused wgmma, 2 wgmma logits +
 * block sums, 3 d-chunked logits + block sums), ridge apply (1 wgmma, 2 FFMA, 3 wgmma over column ranges), native k-means
 * initialisation (1 FFMA, 2 wgmma logits with KS <= 256, 3 wgmma logits, 4 d-chunked logits)}.  Returns 0. */
int hb_debug_wide_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[4]);

#ifdef __cplusplus
}
#endif
#endif /* HARMONY_B200_H */
