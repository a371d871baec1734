// Test infrastructure: amwg_summary_nested run on the HOST with the kernels' arithmetic and addressing (csrc/amwg_nested.cuh, the
// text K_n1 and K_n2 use) and their grids: the segment kernel's CTAs and grid-stride threads, the fixed 256-thread CTA tree and the
// 1024-thread merge of K_m2, for tests/test_summary_nested_host.py. hs_nested returns the number of chain indices that fell outside
// the shard or segments that did not tile it. Build with -ffp-contract=off, as the library is built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_nested.cuh"

#include <cstddef>
#include <vector>

using namespace summary;

namespace {

// cta_merge<T> of amwg_summary.cuh: for w = T/2 .. 1, sh[t] = merge(sh[t], sh[t + w]) for t < w
Moments tree(std::vector<Moments> sh) {
  for (size_t w = sh.size() / 2; w > 0; w /= 2)
    for (size_t t = 0; t < w; ++t) sh[t] = merge(sh[t], sh[t + w]);
  return sh[0];
}

}  // namespace

extern "C" {

long long hs_nested(const double* x, long long rows, int entries, long long C, long long first_chain, long long M, double* out) {
  long long bad = 0;
  const long long n_seg = nested_segments(first_chain, C, M), sx = nested_seg_ctas(n_seg);
  std::vector<double> cm((size_t)C), cw((size_t)C);
  std::vector<int> seen((size_t)C);
  for (int e = 0; e < entries; ++e) {
    for (long long c = 0; c < C; ++c) {                                 // K_n1
      const Moments r = chain_record(x + (size_t)e * C + c, rows, (size_t)entries * C);
      cm[c] = r.mean;
      cw[c] = r.sum_w;
    }
    std::vector<Moments> partial((size_t)sx);
    Moments cut[2] = {{0.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0}};
    long long cut_id[2] = {-1, -1};
    std::fill(seen.begin(), seen.end(), 0);
    for (long long b = 0; b < sx; ++b) {                                // K_n2
      std::vector<Moments> sh(256);
      for (int t = 0; t < 256; ++t) {
        Moments acc{0.0, 0.0, 0.0, 0.0};
        for (long long s = b * 256 + t; s < n_seg; s += sx * 256) {
          long long c0, c1;
          nested_range(s, first_chain, C, M, c0, c1);
          if (c0 < 0 || c1 > C || c0 >= c1 || c1 - c0 > M) { ++bad; continue; }
          for (long long c = c0; c < c1; ++c) seen[c]++;
          const long long k = nested_superchain(s, first_chain, M);
          if (c0 + first_chain < k * M || c1 + first_chain > (k + 1) * M) ++bad;
          const Moments r = nested_chain_merge(cm.data(), cw.data(), c0, c1);
          const int slot = nested_cut_slot(s, first_chain, C, M);
          if (slot < 0) acc = merge(acc, nested_unit(r, M, rows));
          else { cut[slot] = r; cut_id[slot] = k; }
        }
        sh[t] = acc;
      }
      partial[b] = tree(sh);
    }
    for (long long c = 0; c < C; ++c) bad += seen[c] != 1;
    std::vector<Moments> sh(1024, Moments{0.0, 0.0, 0.0, 0.0});         // K_m2
    for (int t = 0; t < 1024; ++t)
      for (long long i = t; i < sx; i += 1024) sh[t] = merge(sh[t], partial[i]);
    const Moments tot = tree(sh);
    double* o = out + (size_t)e * kNestedRecord;
    o[0] = tot.n; o[1] = tot.mean; o[2] = tot.m2; o[3] = tot.sum_w;
    for (int slot = 0; slot < 2; ++slot) {
      double* q = o + 4 + 5 * slot;
      q[0] = (double)cut_id[slot];
      q[1] = cut[slot].n; q[2] = cut[slot].mean; q[3] = cut[slot].m2; q[4] = cut[slot].sum_w;
    }
  }
  return bad;
}

}
