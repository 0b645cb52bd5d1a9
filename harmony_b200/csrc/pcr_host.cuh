// pcr_host.cuh — hb_pcr (DESIGN §14): the checks and launches of pcr.cuh (the batch index, the batch sums, the mean,
// the between-batch rows and the two Grams), the library's symmetric eigensolver and the fold of the R^2 on the host.
// The call needs no setup and touches no state of a Harmony run or a mapping.  Included by harmony_b200.cu.
#pragma once

namespace {

// The eigenvalues of the symmetric n x n matrix A (row-major; the upper triangle is read) in descending order into w,
// and V [n][n] row-major with column j the unit eigenvector of w[j], its entry of largest magnitude positive (the first
// such entry on a tie).  Householder reduction to tridiagonal form, then the implicit QL method with Wilkinson's shift
// on the tridiagonal matrix, accumulating the transformations (the EISPACK tred2 / tql2 pair).  A matrix with a
// non-finite entry, or one whose QL iteration does not converge in 64 steps per eigenvalue, gives NaN throughout.
void sym_eig(int n, const double* A, double* w, double* V) {
  std::vector<double> d(n), e(n);
  bool finite = true;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) {
      V[i * n + j] = A[std::min(i, j) * n + std::max(i, j)];
      finite &= std::isfinite(V[i * n + j]);
    }
  auto v = [&](int i, int j) -> double& { return V[i * n + j]; };
  auto fail_nan = [&] {
    for (int i = 0; i < n; ++i) w[i] = NAN;
    for (int i = 0; i < n * n; ++i) V[i] = NAN;
  };
  if (!finite) return fail_nan();
  // ---- tridiagonalisation: d the diagonal, e[1..n-1] the subdiagonal, V the accumulated transformation
  for (int j = 0; j < n; ++j) d[j] = v(n - 1, j);
  for (int i = n - 1; i > 0; --i) {
    double scale = 0.0, h = 0.0;
    for (int k = 0; k < i; ++k) scale += std::fabs(d[k]);
    if (scale == 0.0) {
      e[i] = d[i - 1];
      for (int j = 0; j < i; ++j) {
        d[j] = v(i - 1, j);
        v(i, j) = 0.0;
        v(j, i) = 0.0;
      }
    } else {
      for (int k = 0; k < i; ++k) {
        d[k] /= scale;
        h += d[k] * d[k];
      }
      double f = d[i - 1], g = std::sqrt(h);
      if (f > 0) g = -g;
      e[i] = scale * g;
      h -= f * g;
      d[i - 1] = f - g;
      for (int j = 0; j < i; ++j) e[j] = 0.0;
      for (int j = 0; j < i; ++j) {
        f = d[j];
        v(j, i) = f;
        g = e[j] + v(j, j) * f;
        for (int k = j + 1; k <= i - 1; ++k) {
          g += v(k, j) * d[k];
          e[k] += v(k, j) * f;
        }
        e[j] = g;
      }
      f = 0.0;
      for (int j = 0; j < i; ++j) {
        e[j] /= h;
        f += e[j] * d[j];
      }
      const double hh = f / (h + h);
      for (int j = 0; j < i; ++j) e[j] -= hh * d[j];
      for (int j = 0; j < i; ++j) {
        f = d[j];
        g = e[j];
        for (int k = j; k <= i - 1; ++k) v(k, j) -= f * e[k] + g * d[k];
        d[j] = v(i - 1, j);
        v(i, j) = 0.0;
      }
    }
    d[i] = h;
  }
  for (int i = 0; i < n - 1; ++i) {
    v(n - 1, i) = v(i, i);
    v(i, i) = 1.0;
    const double h = d[i + 1];
    if (h != 0.0) {
      for (int k = 0; k <= i; ++k) d[k] = v(k, i + 1) / h;
      for (int j = 0; j <= i; ++j) {
        double g = 0.0;
        for (int k = 0; k <= i; ++k) g += v(k, i + 1) * v(k, j);
        for (int k = 0; k <= i; ++k) v(k, j) -= g * d[k];
      }
    }
    for (int k = 0; k <= i; ++k) v(k, i + 1) = 0.0;
  }
  for (int j = 0; j < n; ++j) {
    d[j] = v(n - 1, j);
    v(n - 1, j) = 0.0;
  }
  v(n - 1, n - 1) = 1.0;
  e[0] = 0.0;
  // ---- implicit QL on the tridiagonal matrix
  for (int i = 1; i < n; ++i) e[i - 1] = e[i];
  e[n - 1] = 0.0;
  const double eps = std::ldexp(1.0, -52);
  double f = 0.0, tst1 = 0.0;
  for (int l = 0; l < n; ++l) {
    tst1 = std::max(tst1, std::fabs(d[l]) + std::fabs(e[l]));
    int m = l;
    while (m < n - 1 && std::fabs(e[m]) > eps * tst1) ++m;
    if (m > l) {
      int iter = 0;
      do {
        if (++iter > 64) return fail_nan();
        double g = d[l], p = (d[l + 1] - g) / (2.0 * e[l]), r = std::hypot(p, 1.0);
        if (p < 0) r = -r;
        d[l] = e[l] / (p + r);
        d[l + 1] = e[l] * (p + r);
        const double dl1 = d[l + 1];
        double h = g - d[l];
        for (int i = l + 2; i < n; ++i) d[i] -= h;
        f += h;
        p = d[m];
        double c = 1.0, c2 = c, c3 = c, s = 0.0, s2 = 0.0;
        const double el1 = e[l + 1];
        for (int i = m - 1; i >= l; --i) {
          c3 = c2;
          c2 = c;
          s2 = s;
          g = c * e[i];
          h = c * p;
          r = std::hypot(p, e[i]);
          e[i + 1] = s * r;
          s = e[i] / r;
          c = p / r;
          p = c * d[i] - s * g;
          d[i + 1] = h + s * (c * g + s * d[i]);
          for (int k = 0; k < n; ++k) {
            h = v(k, i + 1);
            v(k, i + 1) = s * v(k, i) + c * h;
            v(k, i) = c * v(k, i) - s * h;
          }
        }
        p = -s * s2 * c3 * el1 * e[l] / dl1;
        e[l] = s * p;
        d[l] = c * p;
      } while (std::fabs(e[l]) > eps * tst1);
    }
    d[l] += f;
    e[l] = 0.0;
  }
  // ---- descending order, and the sign rule
  std::vector<int> order(n);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return d[a] > d[b]; });
  std::vector<double> U(V, V + (size_t)n * n);
  for (int j = 0; j < n; ++j) {
    const int o = order[j];
    w[j] = d[o];
    int big = 0;
    for (int i = 1; i < n; ++i)
      if (std::fabs(U[i * n + o]) > std::fabs(U[big * n + o])) big = i;
    const double sign = U[big * n + o] < 0 ? -1.0 : 1.0;
    for (int i = 0; i < n; ++i) V[i * n + j] = sign * U[i * n + o];
  }
}

// Launch geometry of k_pcr_gram over n rows: at most two CTAs per SM, each a whole number of stages
struct PcrGram {
  int ctas = 0;
  int64_t rows_per_cta = 0;
};
PcrGram pcr_gram_geometry(int64_t n, int num_sms) {
  const int64_t stages = std::max<int64_t>(1, (n + PCR_GR - 1) / PCR_GR);
  const int64_t ctas = std::min<int64_t>(2 * (int64_t)num_sms, stages);
  PcrGram g;
  g.rows_per_cta = (stages + ctas - 1) / ctas * PCR_GR;
  g.ctas = (int)((std::max<int64_t>(n, 1) + g.rows_per_cta - 1) / g.rows_per_cta);
  return g;
}

// The Gram of n rows (centred on `centre` when it is given) into out [KD][KD] (upper-triangle tiles), through part
template <typename T>
int pcr_gram(hb_handle* h, const T* X, int64_t ld, int64_t n, int d, int KD, const double* centre, DevBuf<double>& part,
             double* out) {
  const PcrGram g = pcr_gram_geometry(n, h->num_sms);
  CK(part.reserve((size_t)g.ctas * KD * KD));
  const PcrGramArgs a{ld, n, g.rows_per_cta, d, centre, part.p};
  auto run = [&](auto kd) {
    constexpr int K = decltype(kd)::value;
    return launch(h, k_pcr_gram<T, K>, dim3((unsigned)g.ctas), dim3(32 * PCR_GW), pcr_gram_smem(K), a, X);
  };
  switch (KD) {
    case 16: TRY(run(std::integral_constant<int, 16>())); break;
    case 32: TRY(run(std::integral_constant<int, 32>())); break;
    case 48: TRY(run(std::integral_constant<int, 48>())); break;
    case 64: TRY(run(std::integral_constant<int, 64>())); break;
    case 80: TRY(run(std::integral_constant<int, 80>())); break;
    case 96: TRY(run(std::integral_constant<int, 96>())); break;
    case 112: TRY(run(std::integral_constant<int, 112>())); break;
    default: TRY(run(std::integral_constant<int, 128>())); break;  // KD = d rounded up to 16, d <= 128
  }
  return launch(h, k_pcr_reduce, dim3((unsigned)grid_for((int64_t)KD * KD, 256, h->num_sms)), dim3(256), 0,
                (const double*)part.p, g.ctas, KD, out);
}

// The whole call on h->stream, for arguments the caller has checked
int pcr_run(hb_handle* h, const DevRows& X, int d, const int32_t* batches, int n_batches, int n_comps, double* var,
            double* r2, double* components, double* score) {
  ScoreScratch& s = score_scratch(h);
  const int64_t N = X.n;
  const cudaStream_t st = h->stream;
  const int KD = (d + 15) & ~15;
  // ---- the index: the rows sorted by batch, each batch's sorted rows, and the batch sums
  TupleIndex ti;
  PcrSumArgs a;
  TRY(segment_sums(h, X, d, batches, n_batches, "hb_pcr: batches", ti, a));
  const int J = a.J;
  CK(s.centre.reserve((size_t)KNN_MAX_D));
  CK(s.stats.reserve((size_t)2 * KD * KD + 1));
  // ---- the mean, the between-batch rows
  double* C = s.stats.p;
  double* M = C + (size_t)KD * KD;
  double* n_d = M + (size_t)KD * KD;
  TRY(launch(h, k_pcr_mean, dim3((unsigned)d), dim3(256), 0, (const double*)s.chunk_edge.p + 2 * a.chunks * d,
             (const int*)s.chunk_n.p + 2 * a.chunks, a.chunks, d, s.centre.p, n_d));
  TRY(launch(h, k_pcr_combine, dim3((unsigned)((J + PCR_WARPS - 1) / PCR_WARPS)), dim3(32 * PCR_WARPS), 0, a,
             (const double*)s.centre.p));
  // ---- the covariance and the between-batch scatter
  TRY(with_rows(X, [&](auto x) { return pcr_gram(h, x, X.ld, N, d, KD, s.centre.p, s.cta_part, C); }));
  TRY(pcr_gram(h, (const double*)s.seg_sums.p, (int64_t)d, (int64_t)J, d, KD, (const double*)nullptr, s.cta_part, M));
  std::vector<double> out((size_t)2 * KD * KD + 1);
  std::vector<int> count(J);
  CK(cudaMemcpyAsync(out.data(), s.stats.p, sizeof(double) * out.size(), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(count.data(), s.count.p, sizeof(int) * J, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));

  // ---- the eigenvectors of C, and each component's share of the between-batch scatter
  const double n = out[(size_t)2 * KD * KD];
  int present = 0;
  for (int q = 0; q < J; ++q) present += count[q] > 0;
  std::vector<double> Cd((size_t)d * d), Md((size_t)d * d), w(d), V((size_t)d * d);
  for (int i = 0; i < d; ++i)
    for (int j = i; j < d; ++j) {
      Cd[i * d + j] = Cd[j * d + i] = out[(size_t)i * KD + j];
      Md[i * d + j] = Md[j * d + i] = out[(size_t)KD * KD + (size_t)i * KD + j];
    }
  sym_eig(d, Cd.data(), w.data(), V.data());
  const int m = (int)std::min<int64_t>({(int64_t)n_comps, N, (int64_t)d});
  const double nan = std::numeric_limits<double>::quiet_NaN();
  const double zero = d * std::numeric_limits<double>::epsilon() * w[0];  // below it, an eigenvalue is numerically 0
  std::vector<double> var_h(m), r2_h(m), comp_h((size_t)m * d);
  double num = 0.0, den = 0.0;
  for (int j = 0; j < m; ++j) {
    for (int i = 0; i < d; ++i) comp_h[(size_t)j * d + i] = V[i * d + j];
    double r = 0.0;
    if (present >= 2 && w[0] > 0 && w[j] > zero) {
      double q = 0.0;
      for (int i = 0; i < d; ++i) {
        double mv = 0.0;
        for (int k = 0; k < d; ++k) mv += Md[i * d + k] * V[k * d + j];
        q += V[i * d + j] * mv;
      }
      r = std::min(1.0, std::max(0.0, q / w[j]));
    }
    var_h[j] = n >= 2 ? w[j] / (n - 1) : nan;
    r2_h[j] = n >= 2 ? r : nan;
    num += r * w[j];
    den += w[j];
  }
  const double sc = n >= 2 && den != 0.0 ? num / den : nan;
  CK(cudaMemcpyAsync(var, var_h.data(), sizeof(double) * m, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(r2, r2_h.data(), sizeof(double) * m, cudaMemcpyHostToDevice, st));
  if (components) CK(cudaMemcpyAsync(components, comp_h.data(), sizeof(double) * m * d, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(score, &sc, sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));  // the host vectors go on return
  return 0;
}

int run_pcr(hb_handle* h, const DevRows& X, int d, const int32_t* batches, int n_batches, int n_comps, double* var,
            double* r2, double* components, double* score, cudaStream_t caller) {
  TRY(check_score_shape(h, "hb_pcr", X.n, d));
  if (n_batches < 1) return fail(h, 2, "hb_pcr: n_batches = %d, at least one batch is needed", n_batches);
  if (n_batches > X.n) return fail(h, 2, "hb_pcr: %d batches, more codes than the N = %lld rows", n_batches, (long long)X.n);
  if (n_comps < 1) return fail(h, 2, "hb_pcr: n_comps = %d, at least one component is needed", n_comps);
  TRY(check_rows(h, X, d, "X"));
  TRY(check_device_ptr(h, batches, "batches"));
  TRY(check_device_ptr(h, var, "var"));
  TRY(check_device_ptr(h, r2, "r2"));
  if (components) TRY(check_device_ptr(h, components, "components"));
  TRY(check_device_ptr(h, score, "score"));
  return run_score(h, caller, "pcr",
                   [&] { return pcr_run(h, X, d, batches, n_batches, n_comps, var, r2, components, score); });
}

}  // namespace
