// Test infrastructure: the two bin rules of the posterior histograms (csrc/amwg_hist.cuh, the text the histogram kernels run)
// compiled for the HOST behind a C ABI, for tests/test_summary_hist_host.py. Build with -ffp-contract=off, as the library is
// built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_hist.cuh"

extern "C" {
// out[i] = numpy.histogram's bin of x[i] over edges[k + 1]; -1 below edges[0], -2 above edges[k], -3 NaN (as the kernel sorts them)
void hs_hist_bin(const double* x, int64_t n, const double* edges, int k, int32_t* out) {
  for (int64_t i = 0; i < n; ++i) {
    const double v = x[i];
    out[i] = v < edges[0] ? -1 : v > edges[k] ? -2 : v != v ? -3 : summary::hist_bin(v, edges, k);
  }
}

// out[i] = the numpy.histogramdd bin of v[i] on one axis over edges[k + 1], -1 when it falls outside
void hs_hist2d_axis(const double* v, int64_t n, const double* edges, int k, int32_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = summary::hist2d_axis(v[i], edges, k);
}
}
