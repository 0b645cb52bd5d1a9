// harmony_b200.cu — the C ABI of include/harmony_b200.h (libharmony_b200.so).  One hb_handle == one instance of the
// reference's `harmony` class (/root/reference/src/harmony.h:20-70).  sm_90a (H100) only; there is no CPU path.
// The library is this one translation unit: the kernels, then the host modules, each included once what it uses
// exists.
#include "../../include/harmony_b200.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <numeric>
#include <string>
#include <tuple>
#include <vector>

#include "kernels.cuh"
#include "io.cuh"
#include "update_per_step.cuh"
#include "update_two_pass.cuh"
#include "update_single_pass.cuh"
#include "assign_tc3.cuh"
#include "logits_tc.cuh"
#include "logits_wide.cuh"
#include "apply_tc3.cuh"
#include "stats_tc3.cuh"
#include "knn.cuh"
#include "lisi.cuh"
#include "silhouette.cuh"
#include "components.cuh"
#include "kbet.cuh"
#include "pcr.cuh"
#include "kmeans_score.cuh"
#include "leiden.cuh"

#include "select.cuh"
#include "handle.cuh"
#include "comm.cuh"
#include "trace.cuh"
#include "transfer.cuh"
#include "sort.cuh"
#include "plan.cuh"
#include "tuples.cuh"
#include "update_host.cuh"
#include "correct_host.cuh"
#include "assign_host.cuh"
#include "kmeans_init.cuh"

namespace {

// utils.cpp:102-108
int my_ceil(float num) {
  int inum = (int)num;
  if (num == (float)inum) return inum;
  return inum + 1;
}

int check_err_flag(hb_handle* h) {
  int flag = 0;
  CK(cudaMemcpyAsync(&flag, h->err_flag.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (flag) {
    int z = 0;
    cudaMemcpyAsync(h->err_flag.p, &z, sizeof(int), cudaMemcpyHostToDevice, h->stream);
    if (flag == 1) return fail(h, 4, "update order holds an index outside [0, N)");
    if (flag == 2) return fail(h, 5, "inv(): matrix is singular");
    if (flag == 3) return fail(h, 4, "update order is not a permutation of the cells");
    return fail(h, 6, "device error flag %d", flag);
  }
  return 0;
}

// the K values of sigma must be finite and positive as floats
int check_sigma(hb_handle* h, const double* sigma, int K) {
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(sigma[k]) && (float)sigma[k] > 0.f))
      return fail(h, 2, "sigma[%d] = %g: sigma must be finite and positive", k, sigma[k]);
  return 0;
}

// sigma0 and sigma_uniform (the update kernels' scalar-sigma form) of the K values of sigma, as floats
void set_sigma_scalars(hb_handle* h, const double* sigma) {
  h->sigma0 = (float)sigma[0];
  h->sigma_uniform = std::all_of(sigma + 1, sigma + h->K, [&](double s) { return (float)s == h->sigma0; });
}

// The plan and the update state for calls of up to T rounds (a prebuilt plan is dropped: its buffers go)
int reserve_rounds(hb_handle* h, int T) {
  if (T <= h->plan->rounds) return 0;
  TRY(plan_discard(h));
  CK(cudaStreamSynchronize(h->stream));
  TRY(plan_alloc_rounds(h, T));
  return update_reserve(h, T);
}

// ---- the setup steps of both kinds of handle: hb_setup* (Harmony) and hb_map_setup* (map_host.cuh) ------------------
// The cells given to setup: Z as host doubles (d per row, dense) or device rows, and the labels phi, read on the
// library stream after the work queued on `stream`
struct CellInput {
  const double* host = nullptr;
  DevRows dev{};  // dev.p null: host Z
  cudaStream_t stream = nullptr;
  const int32_t* phi = nullptr;
  bool phi_on_device = false;  // else one copy to the device first
};

// The checks of the cell arguments of setup entry point `entry`, whose Z lies in host memory (`host`) or is the device
// rows *dev.  A host entry point refuses device labels and copies managed ones; a device entry point reads them in place.
int setup_inputs(hb_handle* h, const char* entry, const double* host, const DevRows* dev, void* stream, int d,
                 const int32_t* phi_i, CellInput* in) {
  if (h->ran_setup) return fail(h, 3, "setup was already run on this object");
  if (dev) TRY(check_rows(h, *dev, d, "Z"));
  cudaMemoryType phi_type;
  TRY(phi_location(h, phi_i, &phi_type));
  if (!dev && phi_type == cudaMemoryTypeDevice)
    return fail(h, 2, "phi_i is device memory: %s takes host labels (device labels go through %s_device)", entry, entry);
  *in = CellInput{host, dev ? *dev : DevRows{}, (cudaStream_t)stream, phi_i, dev && phi_type != cudaMemoryTypeHost};
  return 0;
}

int check_dimensions(hb_handle* h, int d, int64_t N, int C, int K) {
  if (d < 1 || N < 1 || C < 1 || K < 1) return fail(h, 2, "bad dimensions");
  if (K > 1024) return fail(h, 2, "K = %d is not supported (K <= 1024)", K);
  if (N > 2000000000LL) return fail(h, 2, "more than 2e9 cells per GPU are not supported");
  return 0;
}

void set_shape(hb_handle* h, int d, int C, int K, const int32_t* B_vec) {
  h->d = d;
  h->C = C;
  h->K = K;
  h->KS = (K + 3) & ~3;
  h->DS = (d + 3) & ~3;
  h->B_vec.assign(B_vec, B_vec + C);
  h->B = std::accumulate(h->B_vec.begin(), h->B_vec.end(), 0);
}

// the kernels of the shape, for update_R in nb blocks, and the device buffers both kinds of handle use, with the tiles
int alloc_common(hb_handle* h, int nb) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, KS = h->KS;
  const size_t nK = (size_t)h->n * KS, nd = (size_t)h->n * h->DS, BK = (size_t)B * KS;
  h->coop_grid = h->num_sms;  // one persistent CTA per SM
  h->paths = select_kernels(K, d, J, h->n, nb, h->coop_grid, h->kernel_set);
  for (DevBuf<float>* b : {&h->Zo, &h->Zc}) CK(b->alloc(nd));
  for (DevBuf<float>* b : {&h->U, &h->R}) CK(b->alloc(nK));
  for (DevBuf<float>* b : {&h->O, &h->E}) CK(b->alloc(BK));
  CK(h->Pr_b.alloc(B));
  CK(h->Y.alloc((size_t)K * d));
  CK(h->sigma.alloc(K));
  CK(h->lambda.alloc(B + 1));
  CK(h->tmpT.alloc((size_t)B * K));
  CK(h->Oacc.alloc(BK + KS));
  CK(h->S.alloc((size_t)J * K * (d + 1)));
  CK(h->V.alloc((size_t)J * K * d));
  CK(h->Wfull.alloc((size_t)K * (B + 1) * d));
  CK(h->scratch.alloc((size_t)K * (2 * (size_t)(B + 1) * (B + 1) + (size_t)(B + 1) * d)));  // the ridge solves'
  CK(h->err_flag.alloc(1));
  CK(h->obj_acc.alloc(2));
  CK(h->stage.alloc((size_t)8 << 20));  // 64 MiB of doubles
  CK(h->tuple_levels.alloc((size_t)J * h->C));
  TRY(build_tiles(h, h->tiles, h->tuple_start_h, TM));
  return build_tiles(h, h->tc_tiles, h->tuple_start_h, TC_TM);
}

// the initial state both kinds of handle start from: no assignment (R = 0, U = padding), empty O / E and rows, and the
// tuples' levels
int init_common(hb_handle* h) {
  const size_t nK = (size_t)h->n * h->KS, nd = (size_t)h->n * h->DS, BK = (size_t)h->B * h->KS;
  CK(cudaMemsetAsync(h->err_flag.p, 0, sizeof(int), h->stream));
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  for (float* t : {h->O.p, h->E.p}) CK(cudaMemsetAsync(t, 0, sizeof(float) * BK, h->stream));
  CK(cudaMemsetAsync(h->R.p, 0, sizeof(float) * nK, h->stream));
  for (float* z : {h->Zo.p, h->Zc.p}) CK(cudaMemsetAsync(z, 0, sizeof(float) * nd, h->stream));
  k_fill_f<<<grid_for((int64_t)nK, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->U.p, (int64_t)nK, U_PAD);
  CKL();
  return upload_vector(h, h->tuple_levels, h->tuple_levels_h);
}

// Z into Zo, in tuple-sorted order (double -> float for host Z)
int upload_z(hb_handle* h, const CellInput& in) {
  if (in.dev.p) return upload_rows_device(h, in.dev, in.stream);
  return upload_rows(h, in.host, h->d, h->DS, h->Zo.p);
}

// ---- hb_setup and hb_setup_device: checks and scalars, the tuple index, the allocations, the uploads ----------------
int setup_scalars(hb_handle* h, int d, int64_t N, const int32_t* B_vec, int C, const double* lambda, int max_iter_kmeans,
                  double epsilon_kmeans, double epsilon_harmony, double alpha, int K, double block_size,
                  double batch_proportion_cutoff, int verbose) {
  TRY(check_dimensions(h, d, N, C, K));
  CK(cudaSetDevice(h->device));
  h->n = N;
  if (!h->shard_set) {
    if (h->world > 1) return fail(h, 3, "hb_set_shard is required when world_size > 1");
    h->N_global = N;
    h->cell_offset = 0;
  }
  const int64_t NG = h->N_global;
  set_shape(h, d, C, K, B_vec);
  h->cov_of.resize(h->B);
  {
    int b = 0;
    for (int c = 0; c < C; ++c)
      for (int l = 0; l < B_vec[c]; ++l) h->cov_of[b++] = c;
  }
  // harmony.cpp:83-91
  if (NG < 6) return fail(h, 1, "Refusing to run with less than 6 cells");
  if (NG < 40) {
    h->warnings.push_back("Too few cells. Setting block_size to 0.2");
    h->block_size = 0.2f;
  } else {
    h->block_size = (float)block_size;
  }
  h->epsilon_kmeans = (float)epsilon_kmeans;
  h->epsilon_harmony = (float)epsilon_harmony;
  h->alpha = (float)alpha;
  h->cutoff = (float)batch_proportion_cutoff;
  h->max_iter_kmeans = (unsigned)max_iter_kmeans;
  h->verbose = verbose;
  h->lambda_estimation = (lambda == nullptr) || (lambda[0] == -1);  // harmony.cpp:75
  // update_R block geometry, harmony.cpp:280-281 (float arithmetic on the GLOBAL cell count)
  h->nb = my_ceil(1.0f / h->block_size);
  h->cpb = (uint32_t)((float)NG * h->block_size);
  if (h->cpb == 0) return fail(h, 2, "block_size * N < 1");
  {
    int bits = 1;
    while ((1ull << bits) < (uint64_t)NG) bits++;
    h->half_bits = (bits + 1) / 2;
  }
  return 0;
}

// joint covariate tuples; cells get sorted by tuple (stable), on the device (tuples.cuh)
int setup_tuples(hb_handle* h, const CellInput& in, TupleIndex& ti) {
  const int C = h->C;
  const int64_t N = h->n;
  TupleKeys keys;
  TRY(tuple_keys(h, h->B_vec, keys));
  const std::vector<int>& base = keys.base;
  const std::vector<uint64_t>& radix = keys.radix;
  {
    RegionScope rs(h, "tuple_index");
    DevBuf<int> phi_up;  // host labels: one upload, then the same kernels
    const int* phi_d = in.phi;
    if (in.phi_on_device) {
      TRY(stream_after(h, h->stream, in.stream));  // read after the caller's work, like Z
    } else {
      CK(phi_up.alloc((size_t)N * C));
      CK(cudaMemcpyAsync(phi_up.p, in.phi, sizeof(int) * (size_t)N * C, cudaMemcpyDefault, h->stream));
      phi_d = phi_up.p;
    }
    TRY(build_tuple_index(h, phi_d, N, keys, true, h->sort_perm, h->inv_sort, ti));
  }
  const int J = (int)ti.uniq.size();
  h->J = J;
  h->tuple_levels_h.resize((size_t)J * C);
  for (int q = 0; q < J; ++q) {
    uint64_t kk = ti.uniq[q];
    for (int c = 0; c < C; ++c) {
      h->tuple_levels_h[(size_t)q * C + c] = base[c] + (int)(kk / radix[c]);
      kk %= radix[c];
    }
  }
  h->tuple_start_h = ti.tstart;
  return 0;
}

// the kernels of the shape and every device buffer, with the tiles and the plan's static tables
int setup_alloc(hb_handle* h) {
  const int K = h->K, B = h->B, J = h->J;
  const int Tplan = std::max(1, (int)h->max_iter_kmeans);
  TRY(alloc_common(h, h->nb));
  for (DevBuf<float>* b : {&h->theta, &h->N_b}) CK(b->alloc(B));
  CK(h->iscratch.alloc((size_t)K * (2 * (size_t)B + J)));
  CK(h->skipped.alloc(K));
  CK(h->cov_of_d.alloc(B));
  TRY(plan_setup(h, h->tuple_start_h, Tplan));
  return reserve_rounds(h, Tplan);
}

// the initial device state, the tables of the tuples and the run parameters, then Z: double -> float, into
// tuple-sorted order (harmony.cpp:41); Z_corr = normalise(Z_orig) (:42)
int setup_uploads(hb_handle* h, const CellInput& in, const double* sigma, const double* theta, const double* lambda,
                  const std::vector<int64_t>& lvl_count, HostLap& lap) {
  const int K = h->K, d = h->d, B = h->B, J = h->J, C = h->C;
  TRY(init_common(h));
  CK(cudaMemsetAsync(h->Wfull.p, 0, sizeof(float) * (size_t)K * (B + 1) * d, h->stream));
  CK(cudaMemsetAsync(h->skipped.p, 0, sizeof(int) * K, h->stream));
  CK(cudaMemsetAsync(h->Y.p, 0, sizeof(float) * (size_t)K * d, h->stream));
  // CSR level -> tuples containing it, ascending tuple order; trailing word: the number of levels of covariate 0
  std::vector<int> lvl_ptr_h(B + 2, 0), lvl_tup_h((size_t)J * C);
  for (size_t i = 0; i < h->tuple_levels_h.size(); ++i) lvl_ptr_h[h->tuple_levels_h[i] + 1]++;
  for (int b = 0; b < B; ++b) lvl_ptr_h[b + 1] += lvl_ptr_h[b];
  std::vector<int> fill(lvl_ptr_h.begin(), lvl_ptr_h.begin() + B);
  for (int q = 0; q < J; ++q)
    for (int c = 0; c < C; ++c) lvl_tup_h[fill[h->tuple_levels_h[(size_t)q * C + c]]++] = q;
  lvl_ptr_h[B + 1] = h->B_vec[0];
  UpdateState& u = *h->upd;
  CK(u.lvl_ptr.alloc(B + 2));
  CK(u.lvl_tup.alloc(std::max<size_t>(1, lvl_tup_h.size())));
  TRY(upload_vector(h, u.lvl_ptr, lvl_ptr_h));
  TRY(upload_vector(h, u.lvl_tup, lvl_tup_h));
  TRY(upload_vector(h, h->cov_of_d, h->cov_of));
  std::vector<float> nbv(B), prb(B);
  for (int b = 0; b < B; ++b) {
    nbv[b] = (float)lvl_count[b];
    prb[b] = (float)lvl_count[b] / (float)h->N_global;  // harmony.cpp:67
  }
  TRY(upload_vector(h, h->N_b, nbv));
  TRY(upload_vector(h, h->Pr_b, prb));
  set_sigma_scalars(h, sigma);
  TRY(upload_vector(h, h->sigma, std::vector<float>(sigma, sigma + K)));
  TRY(upload_vector(h, h->theta, std::vector<float>(theta, theta + B)));
  TRY(upload_vector(h, h->lambda, h->lambda_estimation ? std::vector<float>(B + 1, 0.f) : std::vector<float>(lambda, lambda + B + 1)));
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("memsets + small uploads");
  TRY(upload_z(h, in));
  k_normalise_rows<<<grid_for(h->n * 32, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->Zo.p, h->Zc.p, h->n, d, h->DS);
  CKL();
  CK(cudaStreamSynchronize(h->stream));
  lap.mark("Z upload + normalise");
  return 0;
}

int setup_common(hb_handle* h, const CellInput& in, int d, int64_t N, const int32_t* B_vec, int C, const double* sigma,
                 const double* theta, const double* lambda, double alpha, int max_iter_kmeans, double epsilon_kmeans,
                 double epsilon_harmony, int K, double block_size, double batch_proportion_cutoff, int verbose) {
  if (!(in.host || in.dev.p) || !in.phi || !B_vec || !sigma || !theta) return fail(h, 2, "null argument");
  TRY(setup_scalars(h, d, N, B_vec, C, lambda, max_iter_kmeans, epsilon_kmeans, epsilon_harmony, alpha, K, block_size,
                    batch_proportion_cutoff, verbose));
  HostLap lap(h->stream, "hb_setup");
  TupleIndex ti;
  TRY(setup_tuples(h, in, ti));
  lap.mark("tuple index (device)");
  TRY(setup_alloc(h));
  lap.mark("device allocations");
  TRY(setup_uploads(h, in, sigma, theta, lambda, ti.lvl_count, lap));
  h->ran_setup = true;
  return 0;
}

// the Harmony steps a mapping handle refuses
int refuse_mapping(hb_handle* h, const char* what) {
  return fail(h, 3, "%s: this object maps a query (hb_map_setup), it does not run Harmony", what);
}
// The guard of the Harmony step `what`: a mapping handle refuses it, and it needs init_cluster_cpp (or, for
// init_cluster_cpp itself, setup) to have run
int harmony_step(hb_handle* h, const char* what, bool needs_init = true) {
  if (h->mapping) return refuse_mapping(h, what);
  if (needs_init && !h->ran_init) return fail(h, 3, "init_cluster_cpp has not been run");
  if (!needs_init && !h->ran_setup) return fail(h, 3, "setup has not been run");
  return 0;
}

}  // namespace

#include "map_host.cuh"
#include "score_host.cuh"
#include "knn_host.cuh"
#include "lisi_host.cuh"
#include "silhouette_host.cuh"
#include "components_host.cuh"
#include "kbet_host.cuh"
#include "pcr_host.cuh"
#include "kmeans_score_host.cuh"
#include "leiden_host.cuh"

// =================================================================================================
extern "C" {

int hb_version(void) { return 400; }

int hb_create(hb_handle** out, int device) {
  if (!out) return 1;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return 10;  // no CUDA device: there is no CPU path
  hb_handle* h = new hb_handle();
  if (device < 0) cudaGetDevice(&device);
  h->device = device;
  if (cudaSetDevice(device) != cudaSuccess) {
    delete h;
    return 10;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->num_sms = prop.multiProcessorCount;
  cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  h->plan.reset(new Plan());
  h->upd.reset(new UpdateState());
  h->asg.reset(new AssignState());
  ensure_pinned_staging();  // process-wide; the first handle pays for it, not the first download
  keep_pool_memory(device);
  widen_pool();
  *out = h;
  return 0;
}

void hb_destroy(hb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  release_peer_exchange(h);
  cudaStream_t s = h->stream;
  delete h;  // frees device buffers
  if (s) cudaStreamDestroy(s);
}

const char* hb_last_error(const hb_handle* h) { return h ? h->err.c_str() : "null handle"; }

int hb_pop_warning(hb_handle* h, char* buf, size_t cap) {
  if (!h || h->warnings.empty()) return 0;
  if (buf && cap) {
    strncpy(buf, h->warnings.front().c_str(), cap - 1);
    buf[cap - 1] = 0;
  }
  h->warnings.pop_front();
  return 1;
}

int hb_comm_unique_id(char id[HB_COMM_ID_BYTES]) {
  static_assert(sizeof(ncclUniqueId) <= HB_COMM_ID_BYTES, "id size");
  std::string why;
  if (!load_nccl(&why)) return 11;
  ncclUniqueId uid;
  if (g_nccl.GetUniqueId(&uid) != ncclSuccess) return 11;
  memset(id, 0, HB_COMM_ID_BYTES);
  memcpy(id, &uid, sizeof(uid));
  return 0;
}

int hb_comm_init(hb_handle* h, int rank, int world_size, const char id[HB_COMM_ID_BYTES]) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "hb_comm_init must precede hb_setup");
  if (world_size < 1 || rank < 0 || rank >= world_size) return fail(h, 2, "bad rank/world_size");
  h->rank = rank;
  h->world = world_size;
  if (world_size == 1) return 0;
  std::string why;
  if (!load_nccl(&why)) return fail(h, 11, "%s", why.c_str());
  CK(cudaSetDevice(h->device));
  const CommKey key{h->device, rank, world_size};
  if (!id) {  // reuse the process-wide communicator created by an earlier handle
    auto it = g_comms.find(key);
    if (it == g_comms.end()) return fail(h, 3, "hb_comm_init(NULL id): no communicator has been created yet for this rank/world");
    h->comm = it->second;
    return 0;
  }
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  CKN(g_nccl.CommInitRank(&h->comm, world_size, uid, rank));
  g_comms[key] = h->comm;  // kept until process exit
  return 0;
}

int hb_set_shard(hb_handle* h, int64_t N_global, int64_t cell_offset) {
  if (!h) return 1;
  if (h->ran_setup) return fail(h, 3, "hb_set_shard must precede hb_setup");
  h->N_global = N_global;
  h->cell_offset = cell_offset;
  h->shard_set = true;
  return 0;
}

int hb_set_seed(hb_handle* h, uint64_t seed) {
  if (!h) return 1;
  TRY(plan_discard(h));
  h->seed = seed;
  h->plan->round_counter = 0;
  return 0;
}

int hb_set_abort_callback(hb_handle* h, int (*cb)(void*), void* user) {
  if (!h) return 1;
  h->abort_cb = cb;
  h->abort_user = user;
  return 0;
}

int hb_setup(hb_handle* h, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
             const double* sigma, const double* theta, const double* lambda, double alpha, int max_iter_kmeans,
             double epsilon_kmeans, double epsilon_harmony, int K, double block_size,
             double batch_proportion_cutoff, int verbose) {
  if (!h) return 1;
  CellInput in;
  TRY(setup_inputs(h, "hb_setup", Z, nullptr, nullptr, d, phi_i, &in));
  return setup_common(h, in, d, N, B_vec, C, sigma, theta, lambda, alpha, max_iter_kmeans, epsilon_kmeans,
                      epsilon_harmony, K, block_size, batch_proportion_cutoff, verbose);
}

int hb_setup_device(hb_handle* h, const void* Z, int z_dtype, int64_t z_ld, void* stream, int d, int64_t N,
                    const int32_t* phi_i, const int32_t* B_vec, int C, const double* sigma, const double* theta,
                    const double* lambda, double alpha, int max_iter_kmeans, double epsilon_kmeans,
                    double epsilon_harmony, int K, double block_size, double batch_proportion_cutoff, int verbose) {
  if (!h) return 1;
  CellInput in;
  const DevRows z{Z, z_dtype, z_ld, N};
  TRY(setup_inputs(h, "hb_setup_device", nullptr, &z, stream, d, phi_i, &in));
  return setup_common(h, in, d, N, B_vec, C, sigma, theta, lambda, alpha, max_iter_kmeans, epsilon_kmeans,
                      epsilon_harmony, K, block_size, batch_proportion_cutoff, verbose);
}

int hb_reference(hb_handle* h, double* centroids, double* Nr, double* Cref, double* sigma) {
  if (!h) return 1;
  TRY(harmony_step(h, "hb_reference"));
  if (h->world > 1) return fail(h, 3, "hb_reference does not take a sharded integration");
  CK(cudaSetDevice(h->device));
  return reference_stats(h, centroids, Nr, Cref, sigma);
}

int hb_map_setup(hb_handle* h, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
                 const double* lambda, int K, const double* centroids, const double* Nr, const double* Cref,
                 const double* sigma) {
  if (!h) return 1;
  CellInput in;
  TRY(setup_inputs(h, "hb_map_setup", Z, nullptr, nullptr, d, phi_i, &in));
  return map_setup(h, in, d, N, B_vec, C, lambda, K, centroids, Nr, Cref, sigma);
}

int hb_map_setup_device(hb_handle* h, const void* Z, int z_dtype, int64_t z_ld, void* stream, int d, int64_t N,
                        const int32_t* phi_i, const int32_t* B_vec, int C, const double* lambda, int K,
                        const double* centroids, const double* Nr, const double* Cref, const double* sigma) {
  if (!h) return 1;
  CellInput in;
  const DevRows z{Z, z_dtype, z_ld, N};
  TRY(setup_inputs(h, "hb_map_setup_device", nullptr, &z, stream, d, phi_i, &in));
  return map_setup(h, in, d, N, B_vec, C, lambda, K, centroids, Nr, Cref, sigma);
}

int hb_map(hb_handle* h) {
  if (!h) return 1;
  if (!h->mapping) return fail(h, 3, "hb_map needs an object set up by hb_map_setup");
  return run_map(h);
}

int hb_knn(hb_handle* h, const void* Q, int q_dtype, int64_t q_ld, int64_t Nq, const void* X, int x_dtype, int64_t x_ld,
           int64_t Nx, int d, int k, int metric, int exclude_self, int32_t* idx, float* dist, void* stream) {
  if (!h) return 1;
  return run_knn(h, DevRows{Q, q_dtype, q_ld, Nq}, DevRows{X, x_dtype, x_ld, Nx}, d, k, metric, exclude_self != 0, idx, dist,
                 (cudaStream_t)stream);
}

int hb_lisi(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* labels,
            int64_t labels_ld, int n_sets, double perplexity, double* lisi, int32_t* idx, float* dist, void* stream) {
  if (!h) return 1;
  return run_lisi(h, DevRows{X, x_dtype, x_ld, N}, d, labels, labels_ld, n_sets, perplexity, lisi, idx, dist,
                  (cudaStream_t)stream);
}

int hb_silhouette(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* labels,
                  int n_labels, const int32_t* groups, int n_groups, double* s, void* stream) {
  if (!h) return 1;
  return run_silhouette(h, DevRows{X, x_dtype, x_ld, N}, d, labels, n_labels, groups, n_groups, s, (cudaStream_t)stream);
}

int hb_graph_components(hb_handle* h, const int32_t* idx, int64_t idx_ld, int64_t N, int k, const int32_t* labels,
                        int n_labels, int32_t* comp, int32_t* largest, void* stream) {
  if (!h) return 1;
  return run_components(h, idx, idx_ld, N, k, labels, n_labels, comp, largest, (cudaStream_t)stream);
}

int hb_kbet(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* batches,
            int n_batches, const int32_t* labels, int n_labels, int k0, double* stat, double* pval, int32_t* k0_out,
            int32_t* idx, int64_t idx_ld, void* stream) {
  if (!h) return 1;
  return run_kbet(h, DevRows{X, x_dtype, x_ld, N}, d, batches, n_batches, labels, n_labels, k0, stat, pval, k0_out, idx,
                  idx_ld, (cudaStream_t)stream);
}

int hb_pcr(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, const int32_t* batches,
           int n_batches, int n_comps, double* var, double* r2, double* components, double* score, void* stream) {
  if (!h) return 1;
  return run_pcr(h, DevRows{X, x_dtype, x_ld, N}, d, batches, n_batches, n_comps, var, r2, components, score,
                 (cudaStream_t)stream);
}

int hb_kmeans(hb_handle* h, const void* X, int x_dtype, int64_t x_ld, int64_t N, int d, int K, uint64_t seed,
              int n_init, int max_iter, double tol, int32_t* labels, double* centres, double* inertia, int32_t* n_iter,
              int32_t* seeds, void* stream) {
  if (!h) return 1;
  return run_kmeans(h, DevRows{X, x_dtype, x_ld, N}, d, K, seed, n_init, max_iter, tol, labels, centres, inertia, n_iter,
                    seeds, (cudaStream_t)stream);
}

int hb_umap_graph(hb_handle* h, const int32_t* idx, int64_t idx_ld, const float* dist, int64_t dist_ld, int64_t N, int k,
                  int n_neighbors, int64_t* indptr, int32_t* indices, float* data, int64_t* nnz, void* stream) {
  if (!h) return 1;
  return run_umap_graph(h, idx, idx_ld, dist, dist_ld, N, k, n_neighbors, indptr, indices, data, nnz,
                        (cudaStream_t)stream);
}

int hb_leiden(hb_handle* h, const int64_t* indptr, const int32_t* indices, const void* data, int dtype, int64_t N,
              int64_t nnz, double resolution, int n_iterations, int32_t* labels, int32_t* n_communities, double* quality,
              int32_t* iterations, int64_t* stats, void* stream) {
  if (!h) return 1;
  return run_leiden(h, indptr, indices, data, dtype, N, nnz, resolution, n_iterations, labels, n_communities, quality,
                    iterations, stats, (cudaStream_t)stream);
}

int hb_init_cluster(hb_handle* h, const double* Y0) {
  if (!h) return 1;
  TRY(harmony_step(h, "init_cluster_cpp", false));
  CK(cudaSetDevice(h->device));
  HostLap lap(h->stream, "hb_init_cluster");
  if (Y0)  // Y = normalise(kmeans_centers(..)) (harmony.cpp:133-136), centroids injected by the caller
    TRY(upload_small(h, Y0, (size_t)h->K * h->d, h->Y.p));
  else
    TRY(kmeans_centers(h));
  // Y = arma::normalise(Y, 2, 0)  (harmony.cpp:136)
  lap.mark("centroids (Y0 / native k-means)");
  k_normalise_rows<<<grid_for((int64_t)h->K * 32, 256, 64), 256, 0, h->stream>>>(h->Y.p, h->Y.p, h->K, h->d, h->d);
  CKL();
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  TRY(run_assign(h, false, true));
  TRY(push_objective(h));                       // compute_objective() (:152)
  lap.mark("assignment + objective");
  h->harmony_slots.push_back(h->obj_count - 1);  // objective_harmony.push_back (:153)
  h->ran_init = true;
  return 0;
}

int hb_cluster(hb_handle* h, const int64_t* update_orders) {
  if (!h) return 1;
  TRY(harmony_step(h, "cluster_cpp"));
  CK(cudaSetDevice(h->device));
  const unsigned T = h->max_iter_kmeans;
  const bool cold = h->harmony_slots.size() != 1;  // harmony.cpp:214-228 cold start
  TRY(reserve_rounds(h, (int)std::max(1u, T)));
  const CallPath call = call_path(h->paths, T, h->legacy_centroid);
  const bool plan_assign = cold && call.plan_order_assign;
  if (cold && !plan_assign) TRY(run_assign(h, true, false));
  if (update_orders && T > 0) {
    size_t cnt = (size_t)T * (size_t)h->N_global;
    CK(h->perms_d.reserve(cnt));
    CK(cudaMemcpyAsync(h->perms_d.p, update_orders, sizeof(int64_t) * cnt, cudaMemcpyHostToDevice, h->stream));
  }
  if (h->abort_cb && h->abort_cb(h->abort_user)) return -1;  // Progress::check_abort (:233)
  // the call's first native round: a prebuilt plan drew its rounds from here on
  const uint64_t first_round = h->plan->round_counter - (h->plan->next_ready ? (uint64_t)h->plan->next_T : 0);
  unsigned iter = 0;
  if (call.update == UpdatePath::PerStep) {
    TRY(plan_discard(h));  // a plan prebuilt by an earlier call is not used here
    for (iter = 0; iter < T; iter++) {
      if (iter > 0 && h->abort_cb && h->abort_cb(h->abort_user)) return -1;
      if (h->legacy_centroid) TRY(legacy_centroid_step(h));  // :235-238
      TRY(build_plans(h, 1, update_orders ? h->perms_d.p + (size_t)iter * (size_t)h->N_global : nullptr, 0, h->stream, true));
      TRY(run_update_per_step(h));  // :241
      TRY(push_objective(h));          // :248
      if (iter > h->window_size) {  // :250-256
        int conv = 0;
        TRY(check_convergence_host(h, 0, &conv));
        if (conv) {
          iter++;
          break;
        }
      }
    }
  } else {
    // all T update orders are drawn up front (they do not depend on the data), then the rounds run in
    // chunks: [0, window_size + 2) in one launch, afterwards one round per launch (convergence checks)
    TRY(plan_acquire(h, (int)T, update_orders ? h->perms_d.p : nullptr));
    TRY(update_begin(h, (int)T, [&] { return plan_assign ? run_assign_plan_order(h, true) : 0; }));
    unsigned t0 = 0;
    while (t0 < T) {
      unsigned t1 = (t0 == 0) ? std::min(T, h->window_size + 2) : t0 + 1;
      unsigned mask = 0;
      for (unsigned t = t0; t < t1; ++t)
        if (t < 32 && (t == T - 1 || t > h->window_size)) mask |= 1u << t;  // rounds after which cluster_cpp may stop
      if (t0 > 0 && h->abort_cb && h->abort_cb(h->abort_user)) return -1;
      if (call.update == UpdatePath::SinglePass)
        TRY(run_update_single_pass(h, (int)T, (int)t0, (int)t1, plan_assign));
      else
        TRY(run_update_two_pass(h, (int)T, (int)t0, (int)t1, mask));
      iter = t1;
      if (t1 - 1 > h->window_size) {  // :250-256
        int conv = 0;
        TRY(check_convergence_host(h, 0, &conv));
        if (conv) break;
      }
      t0 = t1;
    }
  }
  // the reference draws one shuffle per executed update_R (:268): rounds drawn but not run, after an early stop or in
  // an adopted plan longer than the call, go back to the counter, so the orders do not depend on the update path
  if (!update_orders) h->plan->round_counter = first_round + iter;
  if (call.update != UpdatePath::PerStep && !update_orders && T > 0 && !h->timing)
    TRY(plan_prebuild(h, (int)T));  // the next call's plan, while this call's correction and the next assignment run
  if (T > 0) h->R_user_set = false;
  if (update_orders) TRY(check_err_flag(h));
  h->kmeans_rounds.push_back((int)iter);         // :259
  h->harmony_slots.push_back(h->obj_count - 1);  // :260
  return 0;
}

int hb_moe_correct_ridge(hb_handle* h) {
  if (!h) return 1;
  TRY(harmony_step(h, "moe_correct_ridge_cpp"));
  CK(cudaSetDevice(h->device));
  TRY(run_correct(h));
  h->zc_pending_norm = false;  // Z_corr was rebuilt from Z_orig
  if (h->C > 1) TRY(check_err_flag(h));
  return 0;
}

int hb_check_convergence(hb_handle* h, int type) {
  if (!h) return -1;
  if (h->mapping) return -refuse_mapping(h, "check_convergence");
  int out = 1;
  int st = check_convergence_host(h, type, &out);
  if (st != 0) return -st;
  return out;
}

int hb_compute_objective(hb_handle* h) {
  if (!h) return 1;
  TRY(harmony_step(h, "compute_objective"));
  CK(cudaSetDevice(h->device));
  CK(cudaMemsetAsync(h->obj_acc.p, 0, 2 * sizeof(double), h->stream));
  k_objective_cells<<<grid_for(h->n * 32, ROW_THREADS, h->num_sms * 8), ROW_THREADS, 0, h->stream>>>(
      h->R.p, h->U.p, h->sigma.p, h->n, h->K, h->KS, h->obj_acc.p);
  CKL();
  return push_objective(h);
}

int64_t hb_field_size(const hb_handle* h, int field) {
  if (!h || !h->ran_setup) return 0;
  switch (field) {
    case HB_Z_CORR:
    case HB_Z_ORIG: return (int64_t)h->n * h->d;
    case HB_R: return (int64_t)h->n * h->K;
    case HB_Y: return (int64_t)h->K * h->d;
    case HB_O:
    case HB_E: return (int64_t)h->K * h->B;
    case HB_W: return (int64_t)(h->B + 1) * h->d;
    case HB_PR_B:
    case HB_THETA: return h->B;
    case HB_SIGMA: return h->K;
    case HB_LAMBDA: return (int64_t)h->K * (h->B + 1);
    case HB_LAMBDA_VEC: return h->B + 1;
  }
  return 0;
}

int hb_get_field(hb_handle* h, int field, double* out) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  if (!out) return fail(h, 2, "null output");
  if (h->mapping && (field == HB_W || field == HB_THETA || field == HB_LAMBDA))
    return fail(h, 3, "field %d belongs to a Harmony run, not to a mapped query", field);
  CK(cudaSetDevice(h->device));
  const int K = h->K, B = h->B, d = h->d;
  const RowField f = row_field(h, field);
  if (f.buf) {
    HostLap lap(h->stream, "hb_get_field");
    if (field == HB_Z_CORR) TRY(normalise_pending_zc(h));
    const int rc = download_rows(h, f.buf, f.cols, f.ld, out);
    if (field == HB_Z_CORR) lap.mark("Z_corr download");
    return rc;
  }
  switch (field) {
    case HB_Y: return download_small(h, h->Y.p, (size_t)K * d, out);
    case HB_O: return download_table(h, h->O.p, out);
    case HB_E: return download_table(h, h->E.p, out);
    case HB_PR_B: return download_small(h, h->Pr_b.p, B, out);
    case HB_THETA: return download_small(h, h->theta.p, B, out);
    case HB_SIGMA: return download_small(h, h->sigma.p, K, out);
    case HB_LAMBDA_VEC: return download_small(h, h->lambda.p, B + 1, out);
    case HB_LAMBDA: {  // getLambda, harmony.cpp:657-669: K x (B+1) column-major
      std::vector<double> E((size_t)K * B), lam(B + 1);
      TRY(download_table(h, h->E.p, E.data()));
      TRY(download_small(h, h->lambda.p, B + 1, lam.data()));
      for (int k = 0; k < K; ++k) {
        out[k] = h->lambda_estimation ? 0.0 : lam[0];
        for (int b = 0; b < B; ++b)
          out[(size_t)(b + 1) * K + k] =
              h->lambda_estimation ? (double)((float)E[(size_t)b * K + k] * h->alpha) : lam[b + 1];
      }
      return 0;
    }
    case HB_W: {  // (B+1) x d column-major; betas of the last cluster that was corrected
      std::vector<int> sk(K);
      CK(cudaMemcpyAsync(sk.data(), h->skipped.p, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      int last = -1;
      for (int k = 0; k < K; ++k)
        if (!sk[k]) last = k;
      std::vector<double> w((size_t)(B + 1) * d, 0.0);
      if (last >= 0) TRY(download_small(h, h->Wfull.p + (size_t)last * (B + 1) * d, (size_t)(B + 1) * d, w.data()));
      for (int b = 0; b <= B; ++b)
        for (int c = 0; c < d; ++c) out[(size_t)c * (B + 1) + b] = w[(size_t)b * d + c];
      return 0;
    }
  }
  return fail(h, 2, "unknown field %d", field);
}

int hb_get_field_device(hb_handle* h, int field, void* out, int dtype, int64_t ld, void* stream) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  const RowField f = row_field(h, field);
  if (!f.buf) return fail(h, 2, "field %d has no device getter (HB_Z_CORR, HB_Z_ORIG, HB_R)", field);
  const DevRows rows{out, dtype, ld, h->n};
  TRY(check_rows(h, rows, f.cols, "out"));
  CK(cudaSetDevice(h->device));
  return on_caller_stream(h, (cudaStream_t)stream, [&] {
    if (field == HB_Z_CORR) TRY(normalise_pending_zc(h));
    RegionScope rs(h, "download");
    with_rows(rows, [&](auto o) {  // `out` is the caller's writable array
      using T = row_t<decltype(o)>;
      copy_rows(f.buf, f.ld, const_cast<T*>(o), ld, h->inv_sort.p, 0, false, h->n, f.cols, h->num_sms, h->stream);
    });
    CKL();
    return 0;
  });
}

int hb_set_field(hb_handle* h, int field, const double* in) {
  if (!h) return 1;
  if (!h->ran_setup) return fail(h, 3, "setup has not been run");
  if (!in) return fail(h, 2, "null input");
  if (h->mapping) return fail(h, 3, "the fields of a mapped query are read-only");
  CK(cudaSetDevice(h->device));
  const int K = h->K, B = h->B, d = h->d;
  if (field == HB_Z_CORR || field == HB_R) {
    const RowField f = row_field(h, field);
    if (field == HB_R)
      h->R_user_set = true;
    else
      h->zc_pending_norm = false;
    return upload_rows(h, in, f.cols, f.ld, f.buf);
  }
  switch (field) {
    case HB_Y: return upload_small(h, in, (size_t)K * d, h->Y.p);
    case HB_O: return upload_table(h, in, h->O.p);
    case HB_E: return upload_table(h, in, h->E.p);
    case HB_THETA: return upload_small(h, in, B, h->theta.p);
    case HB_SIGMA: {
      TRY(check_sigma(h, in, K));
      if (h->ran_init) {
        // U holds -dist / sigma_old (the reference keeps dist_mat and divides by the current sigma in every update_R and
        // compute_objective, harmony.cpp:158-162, 318-319): rescale column k by sigma_old[k] / sigma_new[k]
        std::vector<double> old(K);
        TRY(download_small(h, h->sigma.p, K, old.data()));
        std::vector<double> ratio(K);
        for (int k = 0; k < K; ++k) ratio[k] = old[k] / (double)(float)in[k];
        DevBuf<float> s;
        CK(s.alloc(K));
        TRY(upload_small(h, ratio.data(), K, s.p));
        k_scale_cols<<<grid_for(h->n * K, 256, h->num_sms * 8), 256, 0, h->stream>>>(h->U.p, s.p, h->n, K, h->KS);
        CKL();
        CK(cudaStreamSynchronize(h->stream));
      }
      set_sigma_scalars(h, in);
      return upload_small(h, in, K, h->sigma.p);
    }
    case HB_LAMBDA_VEC:
      h->lambda_estimation = false;
      return upload_small(h, in, B + 1, h->lambda.p);
  }
  return fail(h, 2, "field %d is not writable", field);
}

int hb_get_scalar(const hb_handle* h, int which, double* out) {
  if (!h || !out) return 1;
  switch (which) {
    case HB_N: *out = (double)h->N_global; return 0;
    case HB_N_LOCAL: *out = (double)h->n; return 0;
    case HB_B: *out = h->B; return 0;
    case HB_K: *out = h->K; return 0;
    case HB_D: *out = h->d; return 0;
    case HB_C: *out = h->C; return 0;
    case HB_ALPHA: *out = h->alpha; return 0;
    case HB_MAX_ITER_KMEANS: *out = h->max_iter_kmeans; return 0;
    case HB_BLOCK_SIZE: *out = h->block_size; return 0;
    case HB_EPSILON_KMEANS: *out = h->epsilon_kmeans; return 0;
    case HB_EPSILON_HARMONY: *out = h->epsilon_harmony; return 0;
    case HB_LAMBDA_ESTIMATION: *out = h->lambda_estimation ? 1 : 0; return 0;
    case HB_WINDOW_SIZE: *out = h->window_size; return 0;
    case HB_LEGACY_CENTROID_STEP: *out = h->legacy_centroid ? 1 : 0; return 0;
    case HB_KERNEL_SET: *out = h->kernel_set; return 0;
    case HB_DEVICE: *out = h->device; return 0;
  }
  return 2;
}

int hb_set_scalar(hb_handle* h, int which, double value) {
  if (!h) return 1;
  switch (which) {
    case HB_ALPHA: h->alpha = (float)value; return 0;
    case HB_MAX_ITER_KMEANS:
      if (value < 0) return fail(h, 2, "max_iter_kmeans must be >= 0");
      h->max_iter_kmeans = (unsigned)value;
      return 0;
    case HB_EPSILON_KMEANS: h->epsilon_kmeans = (float)value; return 0;
    case HB_EPSILON_HARMONY: h->epsilon_harmony = (float)value; return 0;
    case HB_LEGACY_CENTROID_STEP: h->legacy_centroid = value != 0.0; return 0;
    case HB_KERNEL_SET: h->kernel_set = (int)value; return 0;  // takes effect at the next hb_setup
  }
  return fail(h, 2, "scalar %d is not writable", which);
}

int hb_get_B_vec(const hb_handle* h, int32_t* out) {
  if (!h || !out) return 1;
  for (int c = 0; c < h->C; ++c) out[c] = h->B_vec[c];
  return 0;
}

int64_t hb_trace(const hb_handle* hc, int trace, double* out, int64_t cap) {
  hb_handle* h = const_cast<hb_handle*>(hc);
  if (!h) return -1;
  if (trace == HB_KMEANS_ROUNDS) {
    if (out)
      for (int64_t i = 0; i < (int64_t)h->kmeans_rounds.size() && i < cap; ++i) out[i] = h->kmeans_rounds[i];
    return (int64_t)h->kmeans_rounds.size();
  }
  if (sync_traces(h) != 0) return -1;
  if (trace >= HB_OBJECTIVE_KMEANS && trace <= HB_OBJECTIVE_KMEANS_CROSS) {
    if (out)
      for (int64_t i = 0; i < h->obj_count && i < cap; ++i) out[i] = h->obj_vals[4 * (size_t)i + trace];
    return h->obj_count;
  }
  if (trace == HB_OBJECTIVE_HARMONY) {
    if (out)
      for (int64_t i = 0; i < (int64_t)h->harmony_slots.size() && i < cap; ++i)
        out[i] = h->obj_vals[4 * (size_t)h->harmony_slots[i]];
    return (int64_t)h->harmony_slots.size();
  }
  return -1;
}

int64_t hb_kernel_launches(const hb_handle* h) { return h ? h->launches : 0; }
void* hb_stream(const hb_handle* h) { return h ? (void*)h->stream : nullptr; }

int hb_synchronize(hb_handle* h) {
  if (!h) return 1;
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

int hb_region_time(hb_handle* h, const char* region, double* ms, int64_t* launches) {
  if (!h || !region) return 1;
  auto it = h->regions.find(region);
  if (it == h->regions.end()) return 2;
  if (ms) *ms = it->second.ms;
  if (launches) *launches = it->second.launches;
  return 0;
}

// Host evaluation of the keyed cell-order permutation used for the native update orders (test hook; the
// same __host__ __device__ code runs in k_plan_block_native / k_kmeans_seed).
uint64_t hb_debug_permute(uint64_t i, uint64_t n, uint64_t key, int inverse) {
  if (n == 0 || i >= n) return ~0ull;
  int bits = 1;
  while ((1ull << bits) < n) bits++;
  const int half_bits = (bits + 1) / 2;
  return inverse ? hb_permute_inv(i, n, half_bits, key) : hb_permute(i, n, half_bits, key);
}

// Host worker pool (test hook, host only): out[i] = (double) in[i] with `threads` threads (first call fixes the
// pool size for the process).  Returns the number of threads of the pool.
int hb_debug_widen(double* out, const float* in, int64_t n, int threads) {
  WidenPool* p = widen_pool(threads);
  if (n > 0) p->widen(out, in, (size_t)n);
  return p->threads();
}

// Ring geometry of the persistent update kernel for rows of KS floats (test hook, host only):
// out = {float4 per lane, groups per warp ring, rows per group, shared-memory bytes, warps}; 0 if the kernel cannot run the shape.
int hb_debug_update_geometry(int KS, int nb, int64_t out[9]) {
  (void)nb;
  if (KS <= 0 || (KS & 3)) return 0;
  const int D = sp_ring_rows(KS, SMEM_LIMIT);
  if (D <= 0) return 0;
  const int nv = sp_nv(KS), ru = sp_ru(nv);
  const int64_t v[9] = {nv, D / ru, ru, (int64_t)sp_smem_bytes(nv, D, KS), SP_NW, 0, 0, 0, 0};
  for (int i = 0; i < 9; ++i) out[i] = v[i];
  return 1;
}

// Kernels hb_setup picks for a shape, and the update path of a cluster_cpp call (test hook, host only).
// Fields 2 and 4 are derived from the stage choices: "wgmma logits" is a k_logits_tc cold start without
// HB_KS_FFMA_CONTRACTIONS (with it, only shapes past FFMA k_assign take that cold start), "tensor-core k-means" a
// k_logits_tc initialisation at KS <= 256.
int hb_debug_kernel_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[8]) {
  const KernelPaths p = select_kernels(K, d, J, n, nb, num_sms, kernel_set);
  const bool cold_logits_tc = p.cold == ColdStart::LogitsTc && !(kernel_set & HB_KS_FFMA_CONTRACTIONS);
  const bool kmeans_tc = p.kmeans == KmeansInit::LogitsTc && ((K + 3) & ~3) <= 256;
  const int64_t v[8] = {(int64_t)p.update, p.k1_stages, cold_logits_tc, p.apply == Apply::Tc, kmeans_tc,
                        call_path(p, 20, false).plan_order_assign, (int64_t)call_path(p, 40, false).update,
                        (int64_t)call_path(p, 20, true).update};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
  return 0;
}

// The kernels of the stages whose FFMA kernels stop at a shared-memory limit, and the kernels that take those shapes
// instead (test hook, host only).  out = {natural-order assignment: 1 fused wgmma, 2 FFMA k_assign, 3 k_logits_tc +
// softmax pass, 4 k_logits_wide + softmax pass; plan-order cold start of a 20-round call: 0 none (natural order),
// 1 fused wgmma, 2 k_logits_tc + block sums, 3 k_logits_wide + block sums; ridge apply: 1 wgmma, 2 FFMA, 3 column
// ranges; native k-means initialisation: 1 FFMA, 2 k_logits_tc logits (KS <= 256), 3 k_logits_tc logits, 4
// k_logits_wide logits}.  The k-means values 2 and 3 run the same kernels; they tell KS <= 256 from KS > 256.
int hb_debug_wide_paths(int K, int d, int J, int64_t n, int nb, int num_sms, int kernel_set, int64_t out[4]) {
  const KernelPaths p = select_kernels(K, d, J, n, nb, num_sms, kernel_set);
  out[0] = (int64_t)p.assign;
  out[1] = call_path(p, 20, false).plan_order_assign ? (int64_t)p.cold : 0;
  out[2] = (int64_t)p.apply;
  out[3] = p.kmeans == KmeansInit::Ffma ? 1 : p.kmeans == KmeansInit::LogitsWide ? 4 : ((K + 3) & ~3) <= 256 ? 2 : 3;
  return 0;
}

// The launch geometry hb_knn picks (test hook, host only): out = {query rows per CTA, reference rows per tile, reference
// operand stages, reference splits, shared-memory bytes, reference tiles per split, padded row length, threads per CTA}.
// Status 2 (out untouched) for a d or k hb_knn refuses.
int hb_debug_knn_geometry(int d, int k, int64_t Nq, int64_t Nx, int num_sms, int64_t out[8]) {
  if (!knn_fits(d, k) || Nq < 1 || Nx < 1 || num_sms < 1) return 2;
  knn_geometry_record(d, k, Nq, Nx, num_sms, out);
  return 0;
}

// The launch geometry of hb_lisi's neighbour search (test hook, host only): hb_debug_knn_geometry's eight values for a
// self-search of N rows with k = floor(3 perplexity) - 1.  Status 2 (out untouched) for a d, perplexity or N hb_lisi
// refuses.
int hb_debug_lisi_geometry(int d, double perplexity, int64_t N, int num_sms, int64_t out[8]) {
  int k = 0;
  if (lisi_check_shape(nullptr, d, perplexity, N, &k) != 0 || num_sms < 1) return 2;
  knn_geometry_record(d, k, N, N, num_sms, out);
  return 0;
}

// The launch geometry of hb_silhouette's sweep (test hook, host only): out = {rows per query tile, reference rows per
// tile, operand stages, shared-memory bytes, padded row length, threads per CTA, query tiles of N rows in one group,
// waves of those tiles on num_sms SMs}.  Status 2 (out untouched) for a d or N hb_silhouette refuses.
int hb_debug_silhouette_geometry(int d, int64_t N, int num_sms, int64_t out[8]) {
  if (check_score_shape(nullptr, "hb_silhouette", N, d) != 0 || num_sms < 1) return 2;
  sil_geometry_record(d, N, num_sms, out);
  return 0;
}

// kBET's p-value function (test hook, host only): the chi2_sf k_kbet runs.  Status 2 (out untouched) for dof < 1.
int hb_debug_chi2_sf(double x, int dof, double* out) {
  if (dof < 1 || !out) return 2;
  *out = chi2_sf(x, dof);
  return 0;
}

// hb_pcr's eigensolver (test hook, host only) on the symmetric n x n matrix A.  Status 2 (outputs untouched) for n
// outside 1..128 or a null pointer.
int hb_debug_sym_eig(int n, const double* A, double* w, double* V) {
  if (n < 1 || n > KNN_MAX_D || !A || !w || !V) return 2;
  sym_eig(n, A, w, V);
  return 0;
}

// The covariate-tuple index setup built (test hook): J, and the non-null ones of sort_perm (N_local cells, sorted
// position -> caller's cell), tuple_levels (J x C global levels) and tuple_start (J + 1 first sorted positions).
int hb_debug_tuple_index(const hb_handle* h, int32_t* sort_perm, int32_t* tuple_levels, int64_t* tuple_start) {
  if (!h || !h->ran_setup) return -1;
  if (sort_perm &&
      (cudaSetDevice(h->device) != cudaSuccess ||
       cudaMemcpy(sort_perm, h->sort_perm.p, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToHost) != cudaSuccess))
    return -1;
  if (tuple_levels) std::copy(h->tuple_levels_h.begin(), h->tuple_levels_h.end(), tuple_levels);
  if (tuple_start) std::copy(h->tuple_start_h.begin(), h->tuple_start_h.end(), tuple_start);
  return h->J;
}

// Test hooks of the native kmeans_centers: the uniform of (centroid i, global cell g) under the handle's seed, and
// the cells initialize_centroids chose (K values; 0 if the native initialisation has not run).
double hb_debug_kmeans_uniform(const hb_handle* h, uint64_t i, uint64_t g) {
  return (double)kmeans_uniform(hb_mix64(h->seed ^ 0x6b6d65616e73ull), i, g);
}
int hb_debug_kmeans_cells(const hb_handle* h, int64_t* out) {
  if (!h || h->kmeans_cells.empty()) return 0;
  for (size_t i = 0; i < h->kmeans_cells.size(); ++i) out[i] = h->kmeans_cells[i];
  return (int)h->kmeans_cells.size();
}
// ... and the means of every step of the native initialisations that run while `on` is set (off by default: the
// record costs a copy and a synchronisation per step).
int hb_debug_kmeans_keep_means(hb_handle* h, int on) {
  if (!h) return 1;
  h->kmeans_keep_means = on != 0;
  return 0;
}
int64_t hb_debug_kmeans_means(const hb_handle* h, float* out) {
  if (!h || h->kmeans_means.empty()) return 0;
  std::copy(h->kmeans_means.begin(), h->kmeans_means.end(), out);
  return (int64_t)h->kmeans_means.size();
}

int hb_enable_timing(hb_handle* h, int on) {
  if (!h) return 1;
  h->timing = on != 0;
  return 0;
}

}  // extern "C"
