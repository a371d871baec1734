// Test infrastructure: amwg_summary_autocov run on the HOST with the kernel's per-half-chain text (csrc/amwg_autocov.cuh,
// autocov_half) and the launch it is given (csrc/amwg_summary.cuh): a grid of chain_ctas(C) CTAs of 256 threads walking the chains
// grid-stride, one kernel pass per 16 lags, the records through cta_merge's 256-thread tree and K_m2's 1024-thread merge, the lag
// sums through cta_sum's tree and K_a2's strided-then-tree sum, for tests/test_summary_diag_reduce_host.py. Build with
// -ffp-contract=off, as the library is built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_autocov.cuh"

#include <algorithm>
#include <vector>

using namespace summary;

namespace {

long long chain_ctas(long long n) { return std::min((n + 255) / 256, 1184LL); }     // amwg_summary.cuh

Moments tree_merge(std::vector<Moments> sh) {                   // cta_merge<THREADS>, THREADS = sh.size()
  for (size_t w = sh.size() >> 1; w > 0; w >>= 1)
    for (size_t t = 0; t < w; ++t) sh[t] = merge(sh[t], sh[t + w]);
  return sh[0];
}

double tree_sum(std::vector<double> sh) {                       // cta_sum<THREADS>
  for (size_t w = sh.size() >> 1; w > 0; w >>= 1)
    for (size_t t = 0; t < w; ++t) sh[t] += sh[t + w];
  return sh[0];
}

// one kernel pass (K_a1<NS>) over the whole grid: pmom[(e NS + s) bx + b] when pmom, psum[((e NS + s) n_total + k_base + k) bx + b]
template <int NS>
void pass(const double* x, long long rows, int entries, long long C, const double* thr, long long lag0, int n_lags, int k_base,
          int n_total, Moments* pmom, double* psum) {
  const long long bx = chain_ctas(C), h = rows / 2;
  const size_t stride = (size_t)entries * C;
  for (int e = 0; e < entries; ++e) {
    double q0 = 0.0, q1 = 0.0, sc = 1.0;
    if (NS == 3) { q0 = thr[2 * e]; q1 = thr[2 * e + 1]; sc = autocov_scale(q0, q1); }
    for (long long b = 0; b < bx; ++b) {
      std::vector<std::vector<Moments>> mt(NS, std::vector<Moments>(256));
      std::vector<std::vector<double>> st(NS * kLagSlots, std::vector<double>(256));
      for (int t = 0; t < 256; ++t) {
        double acc[NS][kLagSlots];
        Moments mom[NS];
        for (int s = 0; s < NS; ++s) {
          for (int k = 0; k < kLagSlots; ++k) acc[s][k] = 0.0;
          mom[s] = Moments{0.0, 0.0, 0.0, 0.0};
        }
        for (long long c = b * 256 + t; c < C; c += bx * 256)
          for (int half = 0; half < 2; ++half)
            autocov_half<NS>(x + (size_t)e * C + c + (size_t)(half ? rows - h : 0) * stride, h, stride, q0, q1, sc, lag0, acc, mom);
        for (int s = 0; s < NS; ++s) {
          mt[s][t] = mom[s];
          for (int k = 0; k < kLagSlots; ++k) st[s * kLagSlots + k][t] = acc[s][k];
        }
      }
      for (int s = 0; s < NS; ++s) {
        if (pmom) pmom[((size_t)e * NS + s) * bx + b] = tree_merge(mt[s]);
        for (int k = 0; k < n_lags; ++k) psum[(((size_t)e * NS + s) * n_total + k_base + k) * bx + b] = tree_sum(st[s * kLagSlots + k]);
      }
    }
  }
}

}  // namespace

extern "C" {
// out[entry][series][4 + n_lags] as amwg_summary_autocov forms it (series 3 with thr [entries][2], else 1)
int hs_autocov(const double* x, long long rows, int entries, long long C, const double* thr, long long lag0, int n_lags, double* out) {
  if (rows < 2 || entries <= 0 || C <= 0 || n_lags < 1 || n_lags > 2 * kLagSlots || lag0 < 0 || lag0 + n_lags > rows / 2) return -1;
  const int ns = thr ? 3 : 1;
  const long long bx = chain_ctas(C);
  const size_t rec = (size_t)entries * ns, sums = rec * n_lags;
  std::vector<Moments> pmom(rec * bx);
  std::vector<double> psum(sums * bx);
  for (int k0 = 0; k0 < n_lags; k0 += kLagSlots) {
    const int nk = std::min(kLagSlots, n_lags - k0);
    Moments* pm = k0 == 0 ? pmom.data() : nullptr;
    if (ns == 3) pass<3>(x, rows, entries, C, thr, lag0 + k0, nk, k0, n_lags, pm, psum.data());
    else pass<1>(x, rows, entries, C, nullptr, lag0 + k0, nk, k0, n_lags, pm, psum.data());
  }
  const size_t w = 4 + (size_t)n_lags;
  for (size_t r = 0; r < rec; ++r) {
    std::vector<Moments> sh(1024, Moments{0.0, 0.0, 0.0, 0.0});       // K_m2: strided merge per thread, then the 1024-thread tree
    for (long long i = 0; i < bx; ++i) sh[i % 1024] = merge(sh[i % 1024], pmom[r * bx + i]);
    const Moments m = tree_merge(sh);
    out[r * w + 0] = m.n; out[r * w + 1] = m.mean; out[r * w + 2] = m.m2; out[r * w + 3] = m.sum_w;
    for (int k = 0; k < n_lags; ++k) {
      std::vector<double> sd(256, 0.0);                                 // K_a2: strided sum per thread, then the 256-thread tree
      for (long long i = 0; i < bx; ++i) sd[i % 256] += psum[(r * n_lags + k) * bx + i];
      out[r * w + 4 + k] = tree_sum(sd);
    }
  }
  return 0;
}

double hs_autocov_scale(double q05, double q95) { return autocov_scale(q05, q95); }
}
