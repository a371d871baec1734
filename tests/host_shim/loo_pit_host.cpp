// Test infrastructure: the pieces of LOO-PIT's fit kernel in csrc/amwg_loo.cuh (the generalised Pareto fit, the smoothed tail
// weights and the run-mean step) compiled for the HOST, for tests/test_summary_loo_pit_host.py. Build with -ffp-contract=off, as the
// library is built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_loo.cuh"

#include <vector>

extern "C" {

// x ascending, n >= 5 -> out[0] = k (with the prior), out[1] = sigma
void hs_pit_fit(const double* x, int n, double* out) {
  const int m = loo::fit_m(n);
  std::vector<double> b((size_t)m), L((size_t)m), w((size_t)m);
  loo::loo_fit_seq(x, n, b.data(), L.data(), w.data(), &out[0], &out[1]);
}

// out[j] = the smoothed log weight of the j-th smallest of n tail draws, j < n
void hs_pit_smoothed(int n, double k, double sigma, double expcut, double* out) {
  for (int j = 0; j < n; ++j) out[j] = loo::smoothed(j, n, k, sigma, expcut);
}

// a[0 .. n) a tail's ll in descending order, w its weights by rank, f its flags by rank -> out[0] = sum w [y_rep <= y],
// out[1] = sum w [y_rep == y], each run of equal ll summed by loo::run_mean_sums (the fit kernel's step, one run per thread),
// the runs in rank order
void hs_pit_runs(const double* a, const double* w, const unsigned char* f, int n, double* out) {
  out[0] = out[1] = 0.0;
  for (int i = 0; i < n;) {
    int e = i + 1;
    while (e < n && a[e] == a[i]) ++e;
    double le, eq;
    loo::run_mean_sums(w + i, f + i, e - i, &le, &eq);
    out[0] += le;
    out[1] += eq;
    i = e;
  }
}

}
