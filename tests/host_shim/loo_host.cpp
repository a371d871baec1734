// Test infrastructure: the generalised Pareto fit and the smoothed tail weights of csrc/amwg_loo.cuh (the element functions
// amwg_loo_fit_kernel uses, here with sequential sums) compiled for the HOST, for tests/test_summary_loo_host.py. Build with
// -ffp-contract=off, as the library is built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_loo.cuh"

#include <vector>

extern "C" {

// x ascending, n >= 5 -> out[0] = k (with the prior), out[1] = sigma
void hs_loo_fit(const double* x, int n, double* out) {
  const int m = loo::fit_m(n);
  std::vector<double> b((size_t)m), L((size_t)m), w((size_t)m);
  loo::loo_fit_seq(x, n, b.data(), L.data(), w.data(), &out[0], &out[1]);
}

// out[j] = the smoothed log weight of the j-th smallest of n tail draws, j < n
void hs_loo_smoothed(int n, double k, double sigma, double expcut, double* out) {
  for (int j = 0; j < n; ++j) out[j] = loo::smoothed(j, n, k, sigma, expcut);
}

}
