// harmony_shim.cpp — Rcpp module `harmony_module` exposing class `harmony` with the SAME method and field
// names as the reference (/root/reference/src/harmony.cpp:672-709), every body a marshalling call into the
// C ABI of include/harmony_b200.h (libharmony_b200.so).  No RcppArmadillo on the hot path.
//
// SOURCE ONLY as an R module: this image has no R / Rcpp (SURVEY.md §8f rank 3).  The CPU suite type-checks it against
// include/harmony_b200.h with an API-shaped stand-in for the few Rcpp types it uses (tests/stubs/Rcpp.h), links it to
// the in-tree library and drives it to its first library call (tests/test_host_cpu.py).
// Build (on a machine with R): R CMD SHLIB harmony_shim.cpp -I../../include -L<libdir> -lharmony_b200
// and keep R/harmony-package.R's `loadModule("harmony_module", TRUE)` unchanged.
#include <Rcpp.h>
#include <string>
#include <vector>
#include "harmony_b200.h"

using namespace Rcpp;

static void hb_check(hb_handle* h, int st) {
  char buf[512];
  while (hb_pop_warning(h, buf, sizeof(buf))) Rcpp::warning("%s", buf);  // harmony.cpp:86-88
  if (st > 0) Rcpp::stop("%s", hb_last_error(h));                         // harmony.cpp:83-85, arma::inv failures
}

class harmony {
 public:
  harmony() { if (hb_create(&h_, -1) != 0) Rcpp::stop("harmony_b200: no usable CUDA device"); }
  ~harmony() { hb_destroy(h_); }

  // harmony::setup (src/harmony.h:25-30; called from R/ui.R:271-275).  __Z: d x N numeric matrix;
  // __Phi: dgCMatrix B x N with exactly one non-zero per covariate in every column.
  void setup(const NumericMatrix& Z, const S4& Phi, const NumericVector sigma, const NumericVector theta,
             const NumericVector lambda, const float alpha, const int max_iter_kmeans, const float epsilon_kmeans,
             const float epsilon_harmony, const int K, const float block_size, const std::vector<int>& B_vec,
             float batch_proportion_cutoff, const bool verbose) {
    IntegerVector i = Phi.slot("i"), p = Phi.slot("p");
    const int C = (int)B_vec.size();
    const R_xlen_t N = Z.ncol();
    for (R_xlen_t n = 0; n <= N; ++n)
      if (p[n] != n * C) Rcpp::stop("Phi must hold exactly one level per covariate for every cell");
    // the `i` slot IS the N x C level table the C ABI takes (rows sorted within a column)
    const double* lam = (lambda.size() == 1 && lambda[0] == -1) ? nullptr : lambda.begin();
    hb_check(h_, hb_setup(h_, Z.begin(), Z.nrow(), (int64_t)N, i.begin(), B_vec.data(), C, sigma.begin(), theta.begin(),
                          lam, alpha, max_iter_kmeans, epsilon_kmeans, epsilon_harmony, K, block_size,
                          batch_proportion_cutoff, verbose));
    // R's RNG seeds the native generators so that set.seed() keeps runs reproducible (R/ui.R:263-266)
    Rcpp::RNGScope rng;   // GetRNGstate / PutRNGstate around the draw (module methods get no implicit scope)
    hb_set_seed(h_, (uint64_t)(R::unif_rand() * 9007199254740992.0));
    hb_set_abort_callback(h_, &harmony::check_abort, nullptr);
  }
  void init_cluster_cpp() { hb_check(h_, hb_init_cluster(h_, nullptr)); }
  int cluster_cpp() {
    int st = hb_cluster(h_, nullptr);
    if (st > 0) hb_check(h_, st);
    return st;                                   // 0, or -1 = user interrupt (R/utils.R:26-32)
  }
  void moe_correct_ridge_cpp() { hb_check(h_, hb_moe_correct_ridge(h_)); }
  bool check_convergence(int type) {
    int r = hb_check_convergence(h_, type);
    if (r < 0) Rcpp::stop("%s", hb_last_error(h_));
    return r != 0;
  }
  void compute_objective() { hb_check(h_, hb_compute_objective(h_)); }

  NumericMatrix getZcorr() { return mat(HB_Z_CORR, dim(HB_D), dim(HB_N_LOCAL)); }
  NumericMatrix getZorig() { return mat(HB_Z_ORIG, dim(HB_D), dim(HB_N_LOCAL)); }
  NumericMatrix getR() { return mat(HB_R, dim(HB_K), dim(HB_N_LOCAL)); }
  NumericMatrix getCentroids() { return mat(HB_Y, dim(HB_D), dim(HB_K)); }
  NumericMatrix getLambda() { return mat(HB_LAMBDA, dim(HB_K), dim(HB_B) + 1); }

  // ---- fields (.property get/set replaces .field of harmony.cpp:675-696) ----
  int get_N() { return dim(HB_N); }
  int get_B() { return dim(HB_B); }
  int get_K() { return dim(HB_K); }
  int get_d() { return dim(HB_D); }
  NumericMatrix get_O() { return mat(HB_O, dim(HB_K), dim(HB_B)); }
  NumericMatrix get_E() { return mat(HB_E, dim(HB_K), dim(HB_B)); }
  NumericMatrix get_Y() { return getCentroids(); }
  NumericMatrix get_W() { return mat(HB_W, dim(HB_B) + 1, dim(HB_D)); }
  NumericMatrix get_R() { return getR(); }
  NumericVector get_Pr_b() { return vec(HB_PR_B, dim(HB_B)); }
  NumericVector get_theta() { return vec(HB_THETA, dim(HB_B)); }
  NumericVector get_sigma() { return vec(HB_SIGMA, dim(HB_K)); }
  NumericVector get_lambda() { return vec(HB_LAMBDA_VEC, dim(HB_B) + 1); }
  std::vector<int> get_B_vec() { std::vector<int> v(dim(HB_C)); hb_get_B_vec(h_, v.data()); return v; }
  double get_alpha() { double v; hb_get_scalar(h_, HB_ALPHA, &v); return v; }
  int get_max_iter_kmeans() { return dim(HB_MAX_ITER_KMEANS); }
  void set_max_iter_kmeans(int v) { hb_check(h_, hb_set_scalar(h_, HB_MAX_ITER_KMEANS, v)); }  // walkthrough.Rmd:364
  void set_alpha(double v) { hb_check(h_, hb_set_scalar(h_, HB_ALPHA, v)); }
  // setters take their value the way Rcpp's .property(name, get, set) requires: `void (Class::*)(PROP)` with the
  // getter's PROP (an Rcpp matrix / vector is a cheap proxy of the SEXP)
  void set_Y(NumericMatrix m) { hb_check(h_, hb_set_field(h_, HB_Y, m.begin())); }
  void set_R(NumericMatrix m) { hb_check(h_, hb_set_field(h_, HB_R, m.begin())); }
  void set_O(NumericMatrix m) { hb_check(h_, hb_set_field(h_, HB_O, m.begin())); }
  void set_E(NumericMatrix m) { hb_check(h_, hb_set_field(h_, HB_E, m.begin())); }
  void set_theta(NumericVector v) { set_vec(HB_THETA, v, dim(HB_B), "theta"); }
  void set_sigma(NumericVector v) { set_vec(HB_SIGMA, v, dim(HB_K), "sigma"); }
  void set_lambda(NumericVector v) { set_vec(HB_LAMBDA_VEC, v, dim(HB_B) + 1, "lambda"); }
  std::vector<double> trace(int id) {
    int64_t n = hb_trace(h_, id, nullptr, 0);
    std::vector<double> v(n > 0 ? n : 0);
    if (n > 0) hb_trace(h_, id, v.data(), n);
    return v;
  }
  std::vector<double> get_objective_kmeans() { return trace(HB_OBJECTIVE_KMEANS); }
  std::vector<double> get_objective_kmeans_dist() { return trace(HB_OBJECTIVE_KMEANS_DIST); }
  std::vector<double> get_objective_kmeans_entropy() { return trace(HB_OBJECTIVE_KMEANS_ENTROPY); }
  std::vector<double> get_objective_kmeans_cross() { return trace(HB_OBJECTIVE_KMEANS_CROSS); }
  std::vector<double> get_objective_harmony() { return trace(HB_OBJECTIVE_HARMONY); }
  std::vector<int> get_kmeans_rounds() { auto v = trace(HB_KMEANS_ROUNDS); return std::vector<int>(v.begin(), v.end()); }

 private:
  static int check_abort(void*) {
    try { Rcpp::checkUserInterrupt(); } catch (...) { return 1; }       // Progress::check_abort(), harmony.cpp:233
    return 0;
  }
  int dim(int which) { double v = 0; hb_get_scalar(h_, which, &v); return (int)v; }
  // the library reads exactly n values
  void set_vec(int field, NumericVector& v, int n, const char* name) {
    if (v.size() != n) {
      const std::string msg = std::string(name) + " must have " + std::to_string(n) + " values, got " + std::to_string(v.size());
      Rcpp::stop("%s", msg.c_str());
    }
    hb_check(h_, hb_set_field(h_, field, v.begin()));
  }
  NumericMatrix mat(int field, int nr, int nc) {
    NumericMatrix m(nr, nc);                                            // column-major doubles: the ABI's layout
    hb_check(h_, hb_get_field(h_, field, m.begin()));
    return m;
  }
  NumericVector vec(int field, int n) {
    NumericVector v(n);
    hb_check(h_, hb_get_field(h_, field, v.begin()));
    return v;
  }
  hb_handle* h_ = nullptr;
};

RCPP_EXPOSED_CLASS(harmony)
RCPP_MODULE(harmony_module) {
  class_<harmony>("harmony")
      .constructor()
      .property("N", &harmony::get_N)
      .property("B", &harmony::get_B)
      .property("K", &harmony::get_K)
      .property("d", &harmony::get_d)
      .property("O", &harmony::get_O, &harmony::set_O)
      .property("E", &harmony::get_E, &harmony::set_E)
      .property("Y", &harmony::get_Y, &harmony::set_Y)
      .property("Pr_b", &harmony::get_Pr_b)
      .property("B_vec", &harmony::get_B_vec)
      .property("alpha", &harmony::get_alpha, &harmony::set_alpha)
      .property("W", &harmony::get_W)
      .property("R", &harmony::get_R, &harmony::set_R)
      .property("theta", &harmony::get_theta, &harmony::set_theta)
      .property("sigma", &harmony::get_sigma, &harmony::set_sigma)
      .property("lambda", &harmony::get_lambda, &harmony::set_lambda)
      .property("kmeans_rounds", &harmony::get_kmeans_rounds)
      .property("objective_kmeans", &harmony::get_objective_kmeans)
      .property("objective_kmeans_dist", &harmony::get_objective_kmeans_dist)
      .property("objective_kmeans_entropy", &harmony::get_objective_kmeans_entropy)
      .property("objective_kmeans_cross", &harmony::get_objective_kmeans_cross)
      .property("objective_harmony", &harmony::get_objective_harmony)
      .property("max_iter_kmeans", &harmony::get_max_iter_kmeans, &harmony::set_max_iter_kmeans)
      .method("getZcorr", &harmony::getZcorr)
      .method("getZorig", &harmony::getZorig)
      .method("getLambda", &harmony::getLambda)
      .method("getR", &harmony::getR)
      .method("getCentroids", &harmony::getCentroids)
      .method("check_convergence", &harmony::check_convergence)
      .method("setup", &harmony::setup)
      .method("compute_objective", &harmony::compute_objective)
      .method("init_cluster_cpp", &harmony::init_cluster_cpp)
      .method("cluster_cpp", &harmony::cluster_cpp)
      .method("moe_correct_ridge_cpp", &harmony::moe_correct_ridge_cpp);
}
