// Per-point arithmetic of Pareto-smoothed importance-sampling leave-one-out (PSIS-LOO; Vehtari, Gelman & Gabry 2017;
// Vehtari et al., JMLR 2024) for sample_summary(..., loo=...), DESIGN.md §4.7: the generalised Pareto fit of Zhang & Stephens
// (2009) with the weakly informative prior on k, and the smoothed tail weights, in ArviZ's operations. The fit kernel of
// amwg_summary_loo.cuh forms its sums in parallel with these element functions; loo_fit_seq is the same fit with sequential sums,
// which tests/host_shim/loo_host.cpp compiles for the host. Plain __host__ __device__ code: no CUDA intrinsics.
#pragma once

#include <cmath>

namespace loo {

constexpr double kEps = 2.220446049250313e-16;       // numpy.finfo(float).eps
constexpr double kTiny = 2.2250738585072014e-308;    // numpy.finfo(float).tiny (DBL_MIN)
constexpr int kMaxTail = 1 << 20;                    // tail draws per point the fit kernel holds (its padded tail length)
constexpr int kMaxM = 30 + 1024;                     // fit_m(kMaxTail): candidates of b

// m = 30 + floor(sqrt(n)) candidate values of b
__host__ __device__ inline int fit_m(int n) { return 30 + (int)sqrt((double)n); }

// the 0-based index of the first-quartile order statistic that scales the candidates: int(n / 4 + 0.5) - 1
__host__ __device__ inline int fit_quartile(int n) { return (int)((double)n / 4.0 + 0.5) - 1; }

// candidate b_j, j = 1..m: 1 / x_max + (1 - sqrt(m / (j - 0.5))) / (3 x_q)
__host__ __device__ inline double fit_b(int j, int m, double xq, double xmax) {
  double b = 1.0 - sqrt((double)m / ((double)j - 0.5));
  b = b / (3.0 * xq);
  return b + 1.0 / xmax;
}

// one term of k(b) = mean log1p(-b x)
__host__ __device__ inline double fit_term(double b, double x) { return log1p(-b * x); }

// profile log-likelihood of candidate (b, k(b)) over n values
__host__ __device__ inline double fit_profile(int n, double b, double k) { return (double)n * (log(-(b / k)) - k - 1.0); }

// the prior on k: (n k + 10 * 0.5) / (n + 10)
__host__ __device__ inline double fit_prior_k(double k, int n) { return ((double)n * k + 5.0) / (double)(n + 10); }

// inverse CDF of the generalised Pareto distribution at p in (0, 1); NaN when sigma <= 0
__host__ __device__ inline double gpinv(double p, double k, double sigma) {
  if (sigma <= 0.0) return NAN;
  double x = fabs(k) < kEps ? -log1p(-p) : expm1(-k * log1p(-p)) / k;
  return x * sigma;
}

// smoothed log weight of the j-th smallest (0-based) of n tail draws: log(gpinv((j + 0.5) / n) + exp(cut)), clipped at 0
__host__ __device__ inline double smoothed(int j, int n, double k, double sigma, double expcut) {
  const double v = log(gpinv(((double)j + 0.5) / (double)n, k, sigma) + expcut);
  return v > 0.0 ? 0.0 : v;
}

// weight of candidate j from the m profile values L: 1 / sum_l exp(L_l - L_j) over the candidates whose L is finite, or 0 when
// L_j is not finite or the weight is below 10 eps (dropped). A candidate b of exactly 0 (a tied tail, where 1 - sqrt(m / (j - 0.5))
// = -3 meets x_q = x_max) has k(b) = 0 and L = NaN; x_q = 0 makes every b infinite and every L NaN. ArviZ lets such an L poison
// every weight; leaving it out keeps the fit of the other candidates (DESIGN.md §4.7).
__host__ __device__ inline double fit_weight(const double* L, int m, int j) {
  if (!(L[j] - L[j] == 0.0)) return 0.0;                       // NaN or infinite
  double s = 0.0;
  for (int l = 0; l < m; ++l)
    if (L[l] - L[l] == 0.0) s += exp(L[l] - L[j]);
  const double w = 1.0 / s;
  return w >= 10.0 * kEps ? w : 0.0;
}

// the weighted mean of the candidates b with the kept weights w normalised to sum 1; NaN when no candidate is kept (every L
// non-finite), which the fit reports as k = +inf: the tail keeps its raw weights, as a tail of at most 4 draws does
__host__ __device__ inline double fit_b_post(const double* b, const double* w, int m) {
  double tot = 0.0;
  for (int j = 0; j < m; ++j) tot += w[j];
  if (!(tot > 0.0)) return NAN;
  double bp = 0.0;
  for (int j = 0; j < m; ++j) bp += b[j] * (w[j] / tot);
  return bp;
}

// The whole fit over the n ascending values x (n >= 5), sequential sums; b, L, w: scratch of fit_m(n) doubles each.
// -> k (with the prior; +inf when no candidate has a finite profile value) and sigma (NaN then).
__host__ __device__ inline void loo_fit_seq(const double* x, int n, double* b, double* L, double* w, double* k_out, double* sigma_out) {
  const int m = fit_m(n);
  const double xq = x[fit_quartile(n)], xmax = x[n - 1];
  for (int j = 0; j < m; ++j) {
    b[j] = fit_b(j + 1, m, xq, xmax);
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += fit_term(b[j], x[i]);
    L[j] = fit_profile(n, b[j], s / (double)n);
  }
  for (int j = 0; j < m; ++j) w[j] = fit_weight(L, m, j);
  const double bp = fit_b_post(b, w, m);
  if (bp != bp) { *k_out = INFINITY; *sigma_out = NAN; return; }
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += fit_term(bp, x[i]);
  const double k = s / (double)n;
  *sigma_out = -k / bp;
  *k_out = fit_prior_k(k, n);
}

}  // namespace loo
