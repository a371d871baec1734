// The two bin rules of the posterior histograms (sample_summary(..., histogram=...)), one __host__ __device__ function each, so that
// the histogram kernels (amwg_summary.cuh) and the host-compiled copy the CPU tests hold against numpy are the same text.
// fp64, one rounding per operation (the library is built with --fmad=false; the host test with -ffp-contract=off).
#pragma once

namespace summary {

// numpy.histogram's equal-width fast path (numpy/lib/_histograms_impl.py, `_histogram`) for one value lo <= x <= hi, where
// lo = edges[0], hi = edges[k] and edges = numpy.linspace(lo, hi, k + 1): the same operations in the same order, so the index
// equals numpy's, including its one-step corrections at the edges. The final clamp only matters where numpy itself would index
// out of its edges (hi - lo overflowing to inf).
__host__ __device__ __forceinline__ int hist_bin(double x, const double* edges, int k) {
  const double lo = edges[0], hi = edges[k];
  const double f = ((x - lo) / (hi - lo)) * (double)k;
  int i = f >= 0.0 && f < (double)k ? (int)f : (f >= (double)k ? k : 0);     // truncation, as numpy's astype(intp)
  if (i == k) i = k - 1;
  if (x < edges[i]) --i;
  if (i < 0) i = 0;
  if (x >= edges[i + 1] && i != k - 1) ++i;
  return i;
}

// One axis of numpy.histogramdd: searchsorted(edges, v, side="right") - 1, with a value equal to the last edge moved into the last
// bin; -1 when v lies outside [edges[0], edges[k]] or is NaN (numpy's outlier bins, which histogramdd drops).
__host__ __device__ __forceinline__ int hist2d_axis(double v, const double* edges, int k) {
  if (!(v >= edges[0] && v <= edges[k])) return -1;
  if (v == edges[k]) return k - 1;
  int lo = 1, hi = k;                                  // the number of edges <= v lies in [1, k]: edges[0] <= v < edges[k]
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (edges[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

}  // namespace summary
