// harmony_oracle.cpp — CPU restatement of the reference's harmonize() hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under harmony_b200/ may include, link or call this file;
// it is the checker for tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs.
//
// PARITY STATUS: pinned against numbers the reference itself printed for the assignment step and
// for cluster_cpp (update_R, compute_objective, convergence window); *parity unpinned* for the
// ridge correction.  The reference (immunogenomics/harmony @ df19af23, v2.0.4) ships no
// known-answer tests for this path (tests/testthat/*.R pin invariants only) and cannot be built
// here (needs R, Rcpp and an un-vendored, un-pinned RcppArmadillo).  Its rendered vignette,
// doc/detailedWalkthrough.html, does print tables of a run on data(cell_lines) with nclust = 5:
//   :656-708  round(O), round(E), cluster x cell-type counts after init_cluster_cpp
//   :733-786  round(O), cell-type counts and error rates after max_iter_kmeans <- 10; cluster_cpp()
//   :844-850  round((E / O)^theta, 2) of that state
// tests/golden/make_vignette_fixture.py recovers the k-means centroids that reproduce the first
// set (R's random stream cannot be replayed), and tests/test_oracle.py checks that this
// restatement (fp32 and fp64) and the numpy restatement reproduce all 55 printed integers exactly
// and the 15 ratios to 3 % — for cluster_cpp with `legacy_centroid_step` on: the vignette was
// rendered while STEP 1 of harmony.cpp:235-238 (commented out in the mounted 2.0.4) still ran,
// and the tables come out right only with it, for any update order, and only if the convergence
// window stops the loop after 5 rounds.  moe_correct_ridge_cpp has no printed output anywhere in
// the reference; for it this file follows the reference operation by operation (citations below)
// and is checked against the reference's own test invariants on the reference's own fixtures and
// against an independent numpy restatement of the plain-R formulas of
// vignettes/detailedWalkthrough.Rmd (tests/numpy_restatement.py).
//
// What is restated (all citations into /root/reference/):
//   setup / allocate_buffers      src/harmony.cpp:29-128
//   init_cluster_cpp (assign)     src/harmony.cpp:131-156   (centroids Y0 are injected)
//   compute_objective             src/harmony.cpp:158-170   + my_accu/safe_entropy utils.cpp:67-81
//   check_convergence             src/harmony.cpp:173-205
//   cluster_cpp                   src/harmony.cpp:208-262
//   update_R                      src/harmony.cpp:269-342   (permutation is injected; my_ceil utils.cpp:102-108)
//   moe_correct_ridge_cpp         src/harmony.cpp:345-638   (level filter, subset path, arrowhead / LU inverse)
//   find_lambda_cpp, harmony_pow  src/utils.cpp:159-163, 84-90
//   getLambda                     src/harmony.cpp:657-669
//
// It keeps the reference's *cost structure* too (physical column shuffles in update_R, one full
// Z copy + scale + gather-sums + dense*sparse update per cluster in the correction), so that it can
// serve as the "CPU restatement of reference" baseline.  The only BLAS call of the reference on
// this path, Y.t()*Z_corr (sgemm, harmony.cpp:141,221), goes through an sgemm loaded at run time
// (ho_load_blas) when one is available, else through a built-in loop.
//
// Scalar type: float (src/types.h:5-9 default) or double (the reference's HARMONY_SCALAR_DOUBLE
// build) — selected per object, the double instance serves as the "truth" run in the tests.
//
// Storage mirrors the reference: column-major with cells as columns (Z is d x N, R is K x N),
// i.e. each cell's d (K) values are contiguous.

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <limits>
#include <numeric>
#include <set>
#include <string>
#include <vector>

namespace {

// ---- optional BLAS (sgemm/dgemm) loaded at run time -----------------------------------------
typedef void (*cblas_gemm32_f)(int, int, int, int, int, int, float, const float*, int, const float*, int, float,
                               float*, int);
typedef void (*cblas_gemm32_d)(int, int, int, int, int, int, double, const double*, int, const double*, int, double,
                               double*, int);
typedef void (*cblas_gemm64_f)(int, int, int, int64_t, int64_t, int64_t, float, const float*, int64_t, const float*,
                               int64_t, float, float*, int64_t);
typedef void (*cblas_gemm64_d)(int, int, int, int64_t, int64_t, int64_t, double, const double*, int64_t,
                               const double*, int64_t, double, double*, int64_t);
struct Blas {
  void* handle = nullptr;
  cblas_gemm32_f s32 = nullptr;
  cblas_gemm32_d d32 = nullptr;
  cblas_gemm64_f s64 = nullptr;
  cblas_gemm64_d d64 = nullptr;
  void (*set_threads)(int) = nullptr;
  std::string name;
} g_blas;

enum { CblasColMajor = 102, CblasNoTrans = 111, CblasTrans = 112 };

// C(K x n) = A(d x K)^T * B(d x n), all column-major.
template <typename T>
void gemm_tn(int64_t K, int64_t n, int64_t d, const T* A, const T* B, T* C);

template <>
void gemm_tn<float>(int64_t K, int64_t n, int64_t d, const float* A, const float* B, float* C) {
  if (g_blas.s32) {
    g_blas.s32(CblasColMajor, CblasTrans, CblasNoTrans, (int)K, (int)n, (int)d, 1.f, A, (int)d, B, (int)d, 0.f, C,
               (int)K);
    return;
  }
  if (g_blas.s64) {
    g_blas.s64(CblasColMajor, CblasTrans, CblasNoTrans, K, n, d, 1.f, A, d, B, d, 0.f, C, K);
    return;
  }
  for (int64_t i = 0; i < n; ++i)
    for (int64_t k = 0; k < K; ++k) {
      float acc = 0.f;
      for (int64_t j = 0; j < d; ++j) acc += A[k * d + j] * B[i * d + j];
      C[i * K + k] = acc;
    }
}
template <>
void gemm_tn<double>(int64_t K, int64_t n, int64_t d, const double* A, const double* B, double* C) {
  if (g_blas.d32) {
    g_blas.d32(CblasColMajor, CblasTrans, CblasNoTrans, (int)K, (int)n, (int)d, 1.0, A, (int)d, B, (int)d, 0.0, C,
               (int)K);
    return;
  }
  if (g_blas.d64) {
    g_blas.d64(CblasColMajor, CblasTrans, CblasNoTrans, K, n, d, 1.0, A, d, B, d, 0.0, C, K);
    return;
  }
  for (int64_t i = 0; i < n; ++i)
    for (int64_t k = 0; k < K; ++k) {
      double acc = 0.0;
      for (int64_t j = 0; j < d; ++j) acc += A[k * d + j] * B[i * d + j];
      C[i * K + k] = acc;
    }
}

// utils.cpp:102-108
int my_ceil(float num) {
  int inum = (int)num;
  if (num == (float)inum) return inum;
  return inum + 1;
}

// Armadillo's trunc_log (used by safe_entropy, utils.cpp:77-81): clamps the argument to
// [smallest positive normal, max] before taking the log, so 0*log(0) evaluates to 0.
template <typename T>
T trunc_log(T x) {
  if (x >= std::numeric_limits<T>::max()) return std::log(std::numeric_limits<T>::max());
  if (x <= T(0)) return std::log(std::numeric_limits<T>::min());
  return std::log(x);
}

struct Base {
  virtual ~Base() {}
  std::string err;
};

template <typename T>
struct Harmony : Base {
  // harmony.h:50-68
  int64_t N = 0;
  int K = 0, B = 0, d = 0, C = 0;
  std::vector<T> R, Z_orig, Z_corr, Y, dist_mat, O, E, W;  // column-major, cells as columns
  std::vector<T> Pr_b, theta, sigma, lambda;
  std::vector<int32_t> lev;                 // N x C: the row indices of Phi's column i (its non-zeros)
  std::vector<std::vector<int64_t>> index;  // per level: cells (ascending), harmony.cpp:49-65
  std::vector<int64_t> batch_sizes;
  std::vector<int> B_vec, covariate_bounds, kmeans_rounds;
  std::vector<float> objective_kmeans, objective_kmeans_dist, objective_kmeans_entropy, objective_kmeans_cross,
      objective_harmony;
  float block_size = 0, epsilon_kmeans = 0, epsilon_harmony = 0, alpha = 0, batch_proportion_cutoff = 0;
  unsigned max_iter_kmeans = 0, window_size = 3;
  bool legacy_centroid_step = false;  // harmony.cpp:235-238 (see cluster())
  bool lambda_estimation = false, ran_setup = false, ran_init = false;
  int W_rows = 0;
  int warn_small = 0;

  // harmony.cpp:29-128
  int setup(const double* Zin, int d_, int64_t N_, const int32_t* phi_i, const int32_t* Bv, int C_,
            const double* sigma_, const double* theta_, const double* lambda_, double alpha_, int max_iter_kmeans_,
            double eps_k, double eps_h, int K_, double block_size_, double cutoff) {
    N = N_;
    d = d_;
    C = C_;
    K = K_;
    B_vec.assign(Bv, Bv + C);
    B = std::accumulate(B_vec.begin(), B_vec.end(), 0);
    Z_orig.resize((size_t)d * N);
    for (size_t i = 0; i < Z_orig.size(); ++i) Z_orig[i] = (T)Zin[i];  // :41 conv_to<MATTYPE>
    Z_corr = Z_orig;
    normalise_cols_l2(Z_corr.data(), d, N);  // :42
    lev.assign(phi_i, phi_i + (size_t)N * C);
    index.assign(B, {});
    batch_sizes.assign(B, 0);
    for (int64_t i = 0; i < N; ++i)
      for (int c = 0; c < C; ++c) {
        int b = lev[i * C + c];
        if (b < 0 || b >= B) {
          err = "level id out of range";
          return 2;
        }
        index[b].push_back(i);
        batch_sizes[b]++;
      }
    Pr_b.resize(B);
    for (int b = 0; b < B; ++b) Pr_b[b] = (T)batch_sizes[b] / (T)N;  // :67
    epsilon_kmeans = (float)eps_k;
    epsilon_harmony = (float)eps_h;
    if (lambda_ == nullptr || lambda_[0] == -1) {  // :75
      lambda_estimation = true;
    } else {
      lambda.resize(B + 1);
      for (int b = 0; b <= B; ++b) lambda[b] = (T)lambda_[b];
    }
    sigma.resize(K);
    for (int k = 0; k < K; ++k) sigma[k] = (T)sigma_[k];
    if (N < 6) {  // :83-91
      err = "Refusing to run with less than 6 cells";
      return 1;
    } else if (N < 40) {
      warn_small = 1;
      block_size = 0.2f;
    } else {
      block_size = (float)block_size_;
    }
    covariate_bounds.resize(C);
    std::partial_sum(B_vec.begin(), B_vec.end(), covariate_bounds.begin());
    theta.resize(B);
    for (int b = 0; b < B; ++b) theta[b] = (T)theta_[b];
    max_iter_kmeans = (unsigned)max_iter_kmeans_;
    // allocate_buffers :114-128
    dist_mat.assign((size_t)K * N, T(0));
    O.assign((size_t)K * B, T(0));
    E.assign((size_t)K * B, T(0));
    W.assign((size_t)(B + 1) * d, T(0));
    W_rows = B + 1;
    R.assign((size_t)K * N, T(0));
    Y.assign((size_t)d * K, T(0));
    alpha = (float)alpha_;
    batch_proportion_cutoff = (float)cutoff;
    ran_setup = true;
    return 0;
  }

  // arma::normalise(X, 2, 0): each column divided by its 2-norm (by 1 when the norm is 0).
  static void normalise_cols_l2(T* X, int64_t rows, int64_t cols) {
    for (int64_t c = 0; c < cols; ++c) {
      T* x = X + c * rows;
      T s = 0;
      for (int64_t r = 0; r < rows; ++r) s += x[r] * x[r];
      T nrm = std::sqrt(s);
      if (nrm == T(0)) nrm = T(1);
      for (int64_t r = 0; r < rows; ++r) x[r] /= nrm;
    }
  }
  // arma::normalise(X, 1, 0)
  static void normalise_cols_l1(T* X, int64_t rows, int64_t cols) {
    for (int64_t c = 0; c < cols; ++c) {
      T* x = X + c * rows;
      T s = 0;
      for (int64_t r = 0; r < rows; ++r) s += std::abs(x[r]);
      if (s == T(0)) s = T(1);
      for (int64_t r = 0; r < rows; ++r) x[r] /= s;
    }
  }

  // the assignment block shared by init_cluster_cpp (:141-150) and the cold start (:221-227)
  void assign_from_centroids() {
    gemm_tn<T>(K, N, d, Y.data(), Z_corr.data(), dist_mat.data());
    for (size_t i = 0; i < dist_mat.size(); ++i) dist_mat[i] = T(2) * (T(1) - dist_mat[i]);
    for (int64_t i = 0; i < N; ++i) {
      T* r = &R[i * K];
      const T* dm = &dist_mat[i * K];
      T s = 0;
      for (int k = 0; k < K; ++k) {
        r[k] = std::exp(-dm[k] / sigma[k]);
        s += r[k];
      }
      for (int k = 0; k < K; ++k) r[k] /= s;  // R.each_row() /= sum(R, 0): no zero guard
    }
    // E = sum(R, 1) * Pr_b.t()
    std::vector<T> rs(K, T(0));
    for (int64_t i = 0; i < N; ++i)
      for (int k = 0; k < K; ++k) rs[k] += R[i * K + k];
    for (int b = 0; b < B; ++b)
      for (int k = 0; k < K; ++k) E[(size_t)b * K + k] = rs[k] * Pr_b[b];
    // O = R * Phi_t  (dense x sparse: column b accumulates the cells of level b in ascending order)
    std::fill(O.begin(), O.end(), T(0));
    for (int b = 0; b < B; ++b)
      for (int64_t i : index[b])
        for (int k = 0; k < K; ++k) O[(size_t)b * K + k] += R[i * K + k];
  }

  // harmony.cpp:131-156 with the k-means centroids injected (Y0 is d x K column-major)
  int init_cluster(const double* Y0) {
    for (size_t i = 0; i < Y.size(); ++i) Y[i] = (T)Y0[i];
    normalise_cols_l2(Y.data(), d, K);  // :136
    assign_from_centroids();
    compute_objective();
    objective_harmony.push_back(objective_kmeans.back());
    ran_init = true;
    return 0;
  }

  // harmony.cpp:158-170
  void compute_objective() {
    const float norm_const = 2000 / ((float)N);
    T kmeans_error = 0, entropy = 0, cross = 0;
    // my_accu(R % dist_mat): one sequential sum over the K x N memory (utils.cpp:67-75)
    for (size_t i = 0; i < R.size(); ++i) kmeans_error += R[i] * dist_mat[i];
    for (int64_t i = 0; i < N; ++i)
      for (int k = 0; k < K; ++k) {
        T r = R[i * K + k];
        entropy += (r * trunc_log<T>(r)) * sigma[k];
      }
    std::vector<T> L((size_t)K * B);
    for (int b = 0; b < B; ++b)
      for (int k = 0; k < K; ++k) {
        size_t q = (size_t)b * K + k;
        L[q] = theta[b] * std::log((O[q] + E[q] + 1) / ((2 * E[q]) + 1));
      }
    for (int64_t i = 0; i < N; ++i)
      for (int k = 0; k < K; ++k) {
        T s = 0;
        for (int c = 0; c < C; ++c) s += L[(size_t)lev[i * C + c] * K + k];
        cross += (R[i * K + k] * sigma[k]) * s;
      }
    objective_kmeans.push_back((float)((kmeans_error + entropy + cross) * norm_const));
    objective_kmeans_dist.push_back((float)(kmeans_error * norm_const));
    objective_kmeans_entropy.push_back((float)(entropy * norm_const));
    objective_kmeans_cross.push_back((float)(cross * norm_const));
  }

  // harmony.cpp:173-205
  int check_convergence(int type) {
    float obj_new, obj_old;
    switch (type) {
      case 0:
        obj_old = 0;
        obj_new = 0;
        for (unsigned i = 0; i < window_size; i++) {
          obj_old += objective_kmeans[objective_kmeans.size() - 2 - i];
          obj_new += objective_kmeans[objective_kmeans.size() - 1 - i];
        }
        return (std::abs(obj_old - obj_new) / std::abs(obj_old) < epsilon_kmeans) ? 1 : 0;
      case 1:
        obj_old = objective_harmony[objective_harmony.size() - 2];
        obj_new = objective_harmony[objective_harmony.size() - 1];
        return ((obj_old - obj_new) / std::abs(obj_old) < epsilon_harmony) ? 1 : 0;
    }
    return 1;
  }

  // harmony.cpp:208-262.  perms: max_iter_kmeans x N update orders (one arma::shuffle per update_R).
  int cluster(const int64_t* perms) {
    unsigned iter;
    if (objective_harmony.size() != 1) {  // :214 cold start
      normalise_cols_l2(Z_corr.data(), d, N);
      assign_from_centroids();
    }
    for (iter = 0; iter < max_iter_kmeans; iter++) {
      if (legacy_centroid_step) {
        // STEP 1 of harmony.cpp:235-238 — commented out in the mounted 2.0.4, still run by the package
        // version that rendered doc/detailedWalkthrough.html (whose printed tables are golden values):
        //   Y = arma::normalise(Z_corr * R.t(), 2, 0);  dist_mat = 2 * (1 - Y.t() * Z_corr);
        std::fill(Y.begin(), Y.end(), T(0));
        for (int64_t i = 0; i < N; ++i)
          for (int k = 0; k < K; ++k) {
            const T r = R[i * K + k];
            for (int c = 0; c < d; ++c) Y[(size_t)k * d + c] += Z_corr[i * d + c] * r;
          }
        normalise_cols_l2(Y.data(), d, K);
        gemm_tn<T>(K, N, d, Y.data(), Z_corr.data(), dist_mat.data());
        for (size_t i = 0; i < dist_mat.size(); ++i) dist_mat[i] = T(2) * (T(1) - dist_mat[i]);
      }
      int st = update_R(perms + (size_t)iter * N);
      if (st != 0) return st;
      compute_objective();
      if (iter > window_size) {
        if (check_convergence(0)) {
          iter++;
          break;
        }
      }
    }
    kmeans_rounds.push_back((int)iter);
    objective_harmony.push_back(objective_kmeans.back());
    return 0;
  }

  // harmony.cpp:269-342
  int update_R(const int64_t* update_order) {
    std::vector<int64_t> reverse_index(N, 0);
    for (int64_t p = 0; p < N; ++p) reverse_index[update_order[p]] = p;  // :276-277
    unsigned n_blocks = (unsigned)my_ceil(1.0f / block_size);         // :280 (float arithmetic)
    unsigned cells_per_block = (unsigned)((float)N * block_size);      // :281 (float arithmetic)
    if (cells_per_block == 0) {
      err = "block_size * N < 1";
      return 3;
    }
    // :284-291 physical shuffles of R, dist_mat and Phi
    std::vector<T> Rr((size_t)K * N), Dr((size_t)K * N);
    std::vector<int32_t> levr((size_t)N * C);
    for (int64_t p = 0; p < N; ++p) {
      int64_t i = update_order[p];
      std::memcpy(&Rr[p * K], &R[i * K], sizeof(T) * K);
      std::memcpy(&Dr[p * K], &dist_mat[i * K], sizeof(T) * K);
      for (int c = 0; c < C; ++c) levr[p * C + c] = lev[i * C + c];
    }
    std::vector<T> rs(K), tmpO((size_t)K * B), P((size_t)K * B);
    for (unsigned blk = 0; blk < n_blocks; blk++) {
      int64_t idx_min = (int64_t)blk * cells_per_block;
      int64_t idx_max = ((int64_t)(blk + 1) * cells_per_block) - 1;
      if (blk == n_blocks - 1) idx_max = N - 1;
      if (idx_min > idx_max || idx_max >= N) continue;  // (reference would throw on an empty submat)
      // Step 1 :312-313  E -= sum(Rcells,1)*Pr_b.t();  O -= Rcells*Phi_tcells
      eo_update(Rr.data(), levr.data(), idx_min, idx_max, rs, tmpO, T(-1));
      // Step 2 :318-323
      for (int b = 0; b < B; ++b)
        for (int k = 0; k < K; ++k) {
          size_t q = (size_t)b * K + k;
          P[q] = std::pow(((2 * E[q]) + 1) / (O[q] + E[q] + 1), theta[b]);  // harmony_pow utils.cpp:84-90
        }
      for (int64_t p = idx_min; p <= idx_max; ++p) {
        T* r = &Rr[p * K];
        const T* dm = &Dr[p * K];
        for (int k = 0; k < K; ++k) r[k] = std::exp(-dm[k] / sigma[k]);
        normalise_cols_l1(r, K, 1);
        for (int k = 0; k < K; ++k) {
          T s = 0;
          for (int c = 0; c < C; ++c) s += P[(size_t)levr[p * C + c] * K + k];
          r[k] *= s;
        }
        normalise_cols_l1(r, K, 1);
      }
      // Step 3 :329-330
      eo_update(Rr.data(), levr.data(), idx_min, idx_max, rs, tmpO, T(1));
    }
    // :338-339 un-shuffle
    for (int64_t i = 0; i < N; ++i) {
      int64_t p = reverse_index[i];
      std::memcpy(&R[i * K], &Rr[p * K], sizeof(T) * K);
      std::memcpy(&dist_mat[i * K], &Dr[p * K], sizeof(T) * K);
    }
    return 0;
  }

  void eo_update(const T* Rr, const int32_t* levr, int64_t lo, int64_t hi, std::vector<T>& rs, std::vector<T>& tmpO,
                 T sign) {
    std::fill(rs.begin(), rs.end(), T(0));
    std::fill(tmpO.begin(), tmpO.end(), T(0));
    for (int64_t p = lo; p <= hi; ++p)
      for (int k = 0; k < K; ++k) rs[k] += Rr[p * K + k];
    // dense x sparse product: within a level the block's cells are accumulated in block order
    for (int64_t p = lo; p <= hi; ++p)
      for (int c = 0; c < C; ++c) {
        T* o = &tmpO[(size_t)levr[p * C + c] * K];
        for (int k = 0; k < K; ++k) o[k] += Rr[p * K + k];
      }
    for (int b = 0; b < B; ++b)
      for (int k = 0; k < K; ++k) {
        size_t q = (size_t)b * K + k;
        E[q] += sign * (rs[k] * Pr_b[b]);
        O[q] += sign * tmpO[q];
      }
  }

  // dense inverse by LU with partial pivoting (what arma::inv -> LAPACK getrf/getri computes)
  static bool invert(std::vector<T>& A, int n) {
    std::vector<T> inv((size_t)n * n, T(0));
    for (int i = 0; i < n; ++i) inv[(size_t)i * n + i] = 1;
    // column-major A[r + c*n]; Gauss-Jordan with partial pivoting
    for (int c = 0; c < n; ++c) {
      int piv = c;
      T best = std::abs(A[c + (size_t)c * n]);
      for (int r = c + 1; r < n; ++r)
        if (std::abs(A[r + (size_t)c * n]) > best) {
          best = std::abs(A[r + (size_t)c * n]);
          piv = r;
        }
      if (best == T(0) || !std::isfinite((double)best)) return false;
      if (piv != c)
        for (int j = 0; j < n; ++j) {
          std::swap(A[c + (size_t)j * n], A[piv + (size_t)j * n]);
          std::swap(inv[c + (size_t)j * n], inv[piv + (size_t)j * n]);
        }
      T p = A[c + (size_t)c * n];
      for (int j = 0; j < n; ++j) {
        A[c + (size_t)j * n] /= p;
        inv[c + (size_t)j * n] /= p;
      }
      for (int r = 0; r < n; ++r) {
        if (r == c) continue;
        T f = A[r + (size_t)c * n];
        if (f == T(0)) continue;
        for (int j = 0; j < n; ++j) {
          A[r + (size_t)j * n] -= f * A[c + (size_t)j * n];
          inv[r + (size_t)j * n] -= f * inv[c + (size_t)j * n];
        }
      }
    }
    A.swap(inv);
    return true;
  }

  // harmony.cpp:345-638
  int moe_correct_ridge() {
    Z_corr = Z_orig;  // :347
    std::vector<T> sizes(B);
    for (int b = 0; b < B; ++b) sizes[b] = (T)batch_sizes[b];
    for (int k = 0; k < K; ++k) {
      std::vector<T> avg_R(B);
      for (int b = 0; b < B; ++b) avg_R[b] = O[(size_t)b * K + k] / sizes[b];  // :358
      std::vector<unsigned> keep;
      std::vector<unsigned> cov_levels(C, 0);
      for (int b = 0, cc = 0; b < B; b++) {  // :368-380
        if (!(b < covariate_bounds[cc])) cc++;
        if ((float)avg_R[b] > batch_proportion_cutoff) cov_levels[cc]++;
      }
      for (int b = 0, cc = 0; b < B; b++) {  // :389-402
        if ((cc < C) && !(b < covariate_bounds[cc])) cc++;
        if ((float)avg_R[b] > batch_proportion_cutoff && cov_levels[cc] > 1) keep.push_back((unsigned)b);
      }
      unsigned active_covariates = 0;
      for (auto l : cov_levels)
        if (l > 1) active_covariates++;

      const int nb = (int)keep.size();  // kept levels B'
      std::vector<int64_t> keep_cols;   // cells taking part (ascending); all cells on the full path
      std::vector<std::vector<int64_t>> idx_local(nb);  // per kept level: positions within keep_cols
      std::vector<T> lam(nb + 1, T(0));
      bool subset = !(nb == B);
      if (!subset) {  // :421-439
        keep_cols.resize(N);
        std::iota(keep_cols.begin(), keep_cols.end(), 0);
        for (int j = 0; j < nb; ++j) idx_local[j] = index[j];
        if (!lambda_estimation) {
          for (int j = 0; j <= B; ++j) lam[j] = lambda[j];
        } else {
          for (int j = 0; j < B; ++j) lam[j + 1] = E[(size_t)j * K + k] * alpha;  // find_lambda_cpp
        }
      } else {  // :440-547
        if (active_covariates == 0) continue;  // :449-452
        std::set<int64_t> s;
        for (unsigned b : keep) s.insert(index[b].begin(), index[b].end());
        keep_cols.assign(s.begin(), s.end());
        std::vector<int64_t> cell_map(N, -1);
        for (size_t q = 0; q < keep_cols.size(); ++q) cell_map[keep_cols[q]] = (int64_t)q;
        for (int j = 0; j < nb; ++j) {
          idx_local[j].reserve(index[keep[j]].size());
          for (int64_t cidx : index[keep[j]]) idx_local[j].push_back(cell_map[cidx]);
        }
        if (!lambda_estimation) {
          for (int j = 0; j < nb; ++j) lam[j + 1] = lambda[keep[j] + 1];
        } else {
          for (int j = 0; j < nb; ++j) lam[j + 1] = E[(size_t)keep[j] * K + k] * alpha;
        }
      }
      const int64_t n = (int64_t)keep_cols.size();
      // _Z_tmp = Z_orig(.cols(keep_cols)), R_k (diag of _Rk)
      std::vector<T> Z_tmp((size_t)d * n), Rk(n);
      for (int64_t q = 0; q < n; ++q) {
        std::memcpy(&Z_tmp[q * d], &Z_orig[keep_cols[q] * d], sizeof(T) * d);
        Rk[q] = R[keep_cols[q] * K + k];
      }
      // Phi_cov = Phi_Rk * Phi_moe_t + lambda_mat  (:561-567), (nb+1) x (nb+1), column-major
      const int m = nb + 1;
      std::vector<T> cov((size_t)m * m, T(0));
      {
        T s0 = 0;
        for (int64_t q = 0; q < n; ++q) s0 += Rk[q];
        cov[0] = s0;
        // level -> kept position
        std::vector<int> pos(B, -1);
        for (int j = 0; j < nb; ++j) pos[keep[j]] = j;
        for (int j = 0; j < nb; ++j) {
          T sj = 0;
          for (int64_t q : idx_local[j]) sj += Rk[q];
          cov[(size_t)(j + 1) * m] = sj;  // row 0
          cov[(size_t)(j + 1)] = sj;      // col 0
        }
        for (int64_t q = 0; q < n; ++q) {
          int64_t cell = keep_cols[q];
          for (int c1 = 0; c1 < C; ++c1) {
            int p1 = pos[lev[cell * C + c1]];
            if (p1 < 0) continue;
            for (int c2 = 0; c2 < C; ++c2) {
              int p2 = pos[lev[cell * C + c2]];
              if (p2 < 0) continue;
              cov[(size_t)(p2 + 1) * m + (p1 + 1)] += Rk[q];
            }
          }
        }
        for (int j = 0; j < m; ++j) cov[(size_t)j * m + j] += lam[j];
      }
      std::vector<T> inv_cov;
      if (C > 1) {  // :572-573
        inv_cov = cov;
        if (!invert(inv_cov, m)) {
          err = "inv(): matrix is singular";
          return 4;
        }
      } else {  // :575-586 arrowhead
        std::vector<T> ac(m), bb(m), ac_b(m);
        for (int j = 0; j < m; ++j) ac[j] = -cov[(size_t)j * m];
        ac[0] = 1;
        T b0 = cov[0];
        for (int j = 0; j < m; ++j) bb[j] = T(1) / cov[(size_t)j * m + j];
        bb[0] = 0;
        T acc = 0;
        for (int j = 0; j < m; ++j) acc += (ac[j] * ac[j]) * bb[j];
        T u = b0 - acc;
        for (int j = 0; j < m; ++j) ac_b[j] = ac[j] * bb[j];
        ac_b[0] = 1;
        inv_cov.assign((size_t)m * m, T(0));
        for (int c2 = 0; c2 < m; ++c2)
          for (int r2 = 0; r2 < m; ++r2) inv_cov[(size_t)c2 * m + r2] = (T(1) / u) * (ac_b[r2] * ac_b[c2]);
        for (int j = 0; j < m; ++j) inv_cov[(size_t)j * m + j] += bb[j];
      }
      // :592 Z_tmp = Z_tmp.each_row() % R_k
      for (int64_t q = 0; q < n; ++q)
        for (int j = 0; j < d; ++j) Z_tmp[q * d + j] *= Rk[q];
      // :599 W = inv_cov.col(0) * sum(Z_tmp, 1).t()
      std::vector<T> Wk((size_t)m * d, T(0)), zs(d);
      std::fill(zs.begin(), zs.end(), T(0));
      for (int64_t q = 0; q < n; ++q)
        for (int j = 0; j < d; ++j) zs[j] += Z_tmp[q * d + j];
      for (int j = 0; j < d; ++j)
        for (int r2 = 0; r2 < m; ++r2) Wk[(size_t)j * m + r2] = inv_cov[r2] * zs[j];
      // :605-608
      for (int b2 = 0; b2 < nb; ++b2) {
        std::fill(zs.begin(), zs.end(), T(0));
        for (int64_t q : idx_local[b2])
          for (int j = 0; j < d; ++j) zs[j] += Z_tmp[q * d + j];
        for (int j = 0; j < d; ++j)
          for (int r2 = 0; r2 < m; ++r2) Wk[(size_t)j * m + r2] += inv_cov[(size_t)(b2 + 1) * m + r2] * zs[j];
      }
      for (int j = 0; j < d; ++j) {
        Y[(size_t)k * d + j] = Wk[(size_t)j * m];  // :610
        Wk[(size_t)j * m] = 0;                     // :611
      }
      // :615 Z_corr -= W.t() * Phi_Rk
      {
        std::vector<int> pos(B, -1);
        for (int j = 0; j < nb; ++j) pos[keep[j]] = j;
        for (int64_t q = 0; q < n; ++q) {
          int64_t cell = keep_cols[q];
          T* zc = &Z_corr[cell * d];
          for (int c1 = 0; c1 < C; ++c1) {
            int p1 = pos[lev[cell * C + c1]];
            if (p1 < 0) continue;
            for (int j = 0; j < d; ++j) zc[j] -= Wk[(size_t)j * m + (p1 + 1)] * Rk[q];
          }
        }
      }
      // the W field keeps the last cluster's betas (harmony.cpp:599-611); expanded to B+1 rows here
      std::fill(W.begin(), W.end(), T(0));
      for (int j = 0; j < d; ++j)
        for (int b2 = 0; b2 < nb; ++b2) W[(size_t)j * (B + 1) + keep[b2] + 1] = Wk[(size_t)j * m + b2 + 1];
    }
    normalise_cols_l2(Y.data(), d, K);  // :633
    return 0;
  }
};

struct Handle {
  int use_double;
  Harmony<float>* f = nullptr;
  Harmony<double>* dd = nullptr;
};

template <typename T>
void copy_out(const std::vector<T>& v, double* out) {
  for (size_t i = 0; i < v.size(); ++i) out[i] = (double)v[i];
}
template <typename T>
void copy_in(std::vector<T>& v, const double* in) {
  for (size_t i = 0; i < v.size(); ++i) v[i] = (T)in[i];
}

}  // namespace

#define DISPATCH(h, expr) ((h)->use_double ? (h)->dd->expr : (h)->f->expr)

extern "C" {

// Load cblas_sgemm/cblas_dgemm from a shared library (e.g. the OpenBLAS bundled with scipy/numpy/opencv).
// Returns 0 on success.  threads <= 0 keeps the library's default.
int ho_load_blas(const char* path, int threads) {
  void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!h) return 1;
  Blas b;
  b.handle = h;
  b.name = path;
  if (void* s = dlsym(h, "cblas_sgemm")) {
    b.s32 = (cblas_gemm32_f)s;
    b.d32 = (cblas_gemm32_d)dlsym(h, "cblas_dgemm");
    b.set_threads = (void (*)(int))dlsym(h, "openblas_set_num_threads");
  } else if (void* s2 = dlsym(h, "scipy_cblas_sgemm")) {
    b.s32 = (cblas_gemm32_f)s2;
    b.d32 = (cblas_gemm32_d)dlsym(h, "scipy_cblas_dgemm");
    b.set_threads = (void (*)(int))dlsym(h, "scipy_openblas_set_num_threads");
  } else if (void* s3 = dlsym(h, "scipy_cblas_sgemm64_")) {
    b.s64 = (cblas_gemm64_f)s3;
    b.d64 = (cblas_gemm64_d)dlsym(h, "scipy_cblas_dgemm64_");
    b.set_threads = (void (*)(int))dlsym(h, "scipy_openblas_set_num_threads64_");
  } else {
    dlclose(h);
    return 2;
  }
  if (threads > 0 && b.set_threads) b.set_threads(threads);
  g_blas = b;
  return 0;
}
int ho_blas_set_threads(int threads) {
  if (!g_blas.set_threads) return 1;
  g_blas.set_threads(threads);
  return 0;
}
const char* ho_blas_name() { return g_blas.handle ? g_blas.name.c_str() : "builtin-loops"; }

void* ho_create(int use_double) {
  Handle* h = new Handle();
  h->use_double = use_double;
  if (use_double)
    h->dd = new Harmony<double>();
  else
    h->f = new Harmony<float>();
  return h;
}
void ho_destroy(void* hv) {
  Handle* h = (Handle*)hv;
  delete h->f;
  delete h->dd;
  delete h;
}
const char* ho_last_error(void* hv) {
  Handle* h = (Handle*)hv;
  return h->use_double ? h->dd->err.c_str() : h->f->err.c_str();
}
// Z: d x N column-major (cells are columns); phi_i: N x C row indices of Phi's columns (global level ids);
// lambda: B+1 values, or NULL / first element -1 for automatic estimation.
int ho_setup(void* hv, const double* Z, int d, int64_t N, const int32_t* phi_i, const int32_t* B_vec, int C,
             const double* sigma, const double* theta, const double* lambda, double alpha, int max_iter_kmeans,
             double epsilon_kmeans, double epsilon_harmony, int K, double block_size, double cutoff) {
  Handle* h = (Handle*)hv;
  return DISPATCH(h, setup(Z, d, N, phi_i, B_vec, C, sigma, theta, lambda, alpha, max_iter_kmeans, epsilon_kmeans,
                           epsilon_harmony, K, block_size, cutoff));
}
int ho_init_cluster(void* hv, const double* Y0) { return DISPATCH((Handle*)hv, init_cluster(Y0)); }
int ho_cluster(void* hv, const int64_t* perms) { return DISPATCH((Handle*)hv, cluster(perms)); }
int ho_update_R(void* hv, const int64_t* perm) { return DISPATCH((Handle*)hv, update_R(perm)); }
int ho_moe_correct_ridge(void* hv) { return DISPATCH((Handle*)hv, moe_correct_ridge()); }
int ho_check_convergence(void* hv, int type) { return DISPATCH((Handle*)hv, check_convergence(type)); }
void ho_compute_objective(void* hv) { DISPATCH((Handle*)hv, compute_objective()); }
int ho_warned_small(void* hv) { return DISPATCH((Handle*)hv, warn_small); }
int ho_set_legacy_centroid_step(void* hv, int on) {
  Handle* h = (Handle*)hv;
  if (h->use_double)
    h->dd->legacy_centroid_step = on != 0;
  else
    h->f->legacy_centroid_step = on != 0;
  return 0;
}
int ho_set_max_iter_kmeans(void* hv, int v) {
  Handle* h = (Handle*)hv;
  if (h->use_double)
    h->dd->max_iter_kmeans = (unsigned)v;
  else
    h->f->max_iter_kmeans = (unsigned)v;
  return 0;
}

// field ids: 0 Z_corr (d x N), 1 Z_orig, 2 R (K x N), 3 Y (d x K), 4 O (K x B), 5 E (K x B), 6 W ((B+1) x d),
// 7 Pr_b, 8 theta, 9 sigma, 10 lambda (K x (B+1), getLambda), 11 dist_mat (K x N).  All column-major doubles.
int ho_get(void* hv, int field, double* out) {
  Handle* h = (Handle*)hv;
#define GET(obj)                                                                      \
  switch (field) {                                                                    \
    case 0: copy_out(obj->Z_corr, out); break;                                        \
    case 1: copy_out(obj->Z_orig, out); break;                                        \
    case 2: copy_out(obj->R, out); break;                                             \
    case 3: copy_out(obj->Y, out); break;                                             \
    case 4: copy_out(obj->O, out); break;                                             \
    case 5: copy_out(obj->E, out); break;                                             \
    case 6: copy_out(obj->W, out); break;                                             \
    case 7: copy_out(obj->Pr_b, out); break;                                          \
    case 8: copy_out(obj->theta, out); break;                                         \
    case 9: copy_out(obj->sigma, out); break;                                         \
    case 10:                                                                          \
      for (int k = 0; k < obj->K; ++k) {                                              \
        out[k] = 0;                                                                   \
        for (int b = 0; b < obj->B; ++b)                                              \
          out[(size_t)(b + 1) * obj->K + k] =                                         \
              obj->lambda_estimation ? (double)(obj->E[(size_t)b * obj->K + k] * obj->alpha) \
                                     : (double)obj->lambda[b + 1];                    \
        if (!obj->lambda_estimation) out[k] = (double)obj->lambda[0];                 \
      }                                                                               \
      break;                                                                          \
    case 11: copy_out(obj->dist_mat, out); break;                                     \
    default: return 1;                                                                \
  }
  if (h->use_double) {
    GET(h->dd)
  } else {
    GET(h->f)
  }
#undef GET
  return 0;
}

// writable fields (same ids and layouts as ho_get): 2 R, 3 Y, 4 O, 5 E, 8 theta, 9 sigma.  Lets a test plant the
// state a step starts from, like the `.field<-` writes of the reference's Rcpp module (a written sigma divides the
// kept dist_mat in the next update_R and compute_objective).
int ho_set(void* hv, int field, const double* in) {
  Handle* h = (Handle*)hv;
#define SET(obj)                                \
  switch (field) {                              \
    case 2: copy_in(obj->R, in); break;         \
    case 3: copy_in(obj->Y, in); break;         \
    case 4: copy_in(obj->O, in); break;         \
    case 5: copy_in(obj->E, in); break;         \
    case 8: copy_in(obj->theta, in); break;     \
    case 9: copy_in(obj->sigma, in); break;     \
    default: return 1;                          \
  }
  if (h->use_double) {
    SET(h->dd)
  } else {
    SET(h->f)
  }
#undef SET
  return 0;
}

// trace ids: 0 objective_kmeans, 1 _dist, 2 _entropy, 3 _cross, 4 objective_harmony, 5 kmeans_rounds
int64_t ho_trace(void* hv, int id, double* out, int64_t cap) {
  Handle* h = (Handle*)hv;
  std::vector<double> v;
#define TR(obj)                                                                                    \
  switch (id) {                                                                                    \
    case 0: v.assign(obj->objective_kmeans.begin(), obj->objective_kmeans.end()); break;           \
    case 1: v.assign(obj->objective_kmeans_dist.begin(), obj->objective_kmeans_dist.end()); break; \
    case 2: v.assign(obj->objective_kmeans_entropy.begin(), obj->objective_kmeans_entropy.end()); break; \
    case 3: v.assign(obj->objective_kmeans_cross.begin(), obj->objective_kmeans_cross.end()); break; \
    case 4: v.assign(obj->objective_harmony.begin(), obj->objective_harmony.end()); break;         \
    case 5: v.assign(obj->kmeans_rounds.begin(), obj->kmeans_rounds.end()); break;                 \
    default: return -1;                                                                            \
  }
  if (h->use_double) {
    TR(h->dd)
  } else {
    TR(h->f)
  }
#undef TR
  if (out)
    for (int64_t i = 0; i < (int64_t)v.size() && i < cap; ++i) out[i] = v[i];
  return (int64_t)v.size();
}

}  // extern "C"
