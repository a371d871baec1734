// Test infrastructure: amwg_summary_indicator_autocov run on the HOST with the kernel's per-half-chain text (csrc/amwg_indicator.cuh,
// indicator_half) for tests/test_summary_mcse_host.py. The device sink sums across a warp and the CTA before it adds; every value is
// an integer, so a sink that adds each half-chain's integers directly gives the same counters.
#include "cuda_runtime.h"
#include "amwg_indicator.cuh"

#include <cstddef>

using namespace summary;

namespace {

struct HostSink {
  long long* rec;        // [kIndGroup][2 + 2 n_lags] of the current entry and threshold group
  int w, n_lags, nk;     // record width, lags, thresholds of the group that exist
  void pair(int k, int i, unsigned v) { if (k < nk) rec[k * w + 2 + i] += v; }
  void edge(int k, int i, unsigned long long v) { if (k < nk) rec[k * w + 2 + n_lags + i] += (long long)v; }
  void count(int k, long long c) { if (k < nk) { rec[k * w] += c; rec[k * w + 1] += c * c; } }
};

}  // namespace

extern "C" {
// out[entry][K][2 + 2 n_lags] as amwg_summary_indicator_autocov forms it, thr [entries][K]
int hs_indicator(const double* x, long long rows, int entries, long long C, const double* thr, int K, long long lag0, int n_lags, long long* out) {
  if (rows < 2 || rows >= (1LL << 32) || entries <= 0 || C <= 0 || K < 1 || K > kIndMaxThresholds || n_lags < 1 || n_lags > kIndLags || lag0 < 0 ||
      lag0 + n_lags > rows / 2)
    return -1;
  const long long h = rows / 2;
  const size_t stride = (size_t)entries * C;
  const int w = 2 + 2 * n_lags;
  for (size_t i = 0; i < (size_t)entries * K * w; ++i) out[i] = 0;
  for (int e = 0; e < entries; ++e)
    for (int k0 = 0; k0 < K; k0 += kIndGroup) {
      double q[kIndGroup];
      for (int k = 0; k < kIndGroup; ++k) q[k] = k0 + k < K ? thr[(size_t)e * K + k0 + k] : __longlong_as_double(0x7ff8000000000000ll);
      HostSink sink{out + ((size_t)e * K + k0) * w, w, n_lags, K - k0};
      unsigned long long keep[4 * kIndGroup];
      for (long long c = 0; c < C; ++c)
        for (int half = 0; half < 2; ++half)
          indicator_half<kIndGroup>(x + (size_t)e * C + c + (size_t)(half ? rows - h : 0) * stride, h, stride, true, q, lag0, n_lags, keep, 1,
                                    sink);
    }
  return 0;
}
}
