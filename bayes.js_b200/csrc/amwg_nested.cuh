// Moment records and their Chan merge, and the superchain addressing of amwg_summary_nested (sample_summary(..., nested=...),
// DESIGN.md §4.6). One __host__ __device__ text, so that the kernels (amwg_summary.cuh) and the host build the CPU tests run
// (tests/host_shim/nested_host.cpp) merge and address alike.
//
// Superchain k is the global chains [k M, (k + 1) M). A shard holds the global chains [first_chain, first_chain + C): its
// segments are its pieces of the superchains it touches, in chain order. A segment is complete when it holds all M chains of its
// superchain; only the first and the last segment can be cut (by the ends of the shard's range).
#pragma once

namespace summary {

struct Moments { double n, mean, m2, sum_w; };     // n records merged so far, mean of their means, M2 of their means, sum of their sum_w

// Chan's merge of two records (b after a): the same arithmetic as merge_moment_records in summary.py
__host__ __device__ __forceinline__ Moments merge(const Moments& a, const Moments& b) {
  if (b.n == 0.0) return a;
  if (a.n == 0.0) return b;
  Moments r;
  r.n = a.n + b.n;
  const double d = b.mean - a.mean;
  r.mean = a.mean + d * (b.n / r.n);
  r.m2 = a.m2 + b.m2 + d * d * (a.n * b.n / r.n);
  r.sum_w = a.sum_w + b.sum_w;
  return r;
}

// The bits of x, for the constant-run test of run_mean: equal bits, not equal values, so that a mix of -0 and +0 is not a run.
__host__ __device__ __forceinline__ unsigned long long run_bits(double x) {
#ifdef __CUDA_ARCH__
  return (unsigned long long)__double_as_longlong(x);
#else
  unsigned long long u;
  memcpy(&u, &x, sizeof u);
  return u;
#endif
}

// The mean of a run of n values summed to s, whose first value is x0; `diff` is the OR over the run of run_bits(v) ^ run_bits(x0),
// 0 exactly when every value has x0's bits. A constant run of finite values has x0 as its mean, so that the values centred on it
// are exactly 0: fl(fl(n x0) / n) is x0 only for some x0 (7.25, but not 0.1 or 184.3), and a mean one ulp off would give a constant
// entry a within-chain variance of ~1e-33 where it has none. Every other run (a mix of -0 and +0, a NaN, an infinity, any two
// values that differ) keeps fl(s / n).
__host__ __device__ __forceinline__ double run_mean(double s, long long n, double x0, unsigned long long diff) {
  const bool finite = (run_bits(x0) & 0x7ff0000000000000ull) != 0x7ff0000000000000ull;     // exponent not all ones
  return diff == 0 && finite ? x0 : s / (double)n;
}

// the record (1, mean, 0, M2) of one chain's column p[r * stride], r < rows >= 1: two sequential passes, eight loads in flight per
// thread; the mean is run_mean's
__host__ __device__ __forceinline__ Moments chain_record(const double* __restrict__ p, long long rows, size_t stride) {
  const unsigned long long b0 = run_bits(p[0]);
  unsigned long long diff = 0;
  double s = 0.0;
  long long r = 0;
  for (; r + 8 <= rows; r += 8) {                            // the sum stays sequential
    double v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = p[(r + u) * stride];
#pragma unroll
    for (int u = 0; u < 8; ++u) { s += v[u]; diff |= run_bits(v[u]) ^ b0; }
  }
  for (; r < rows; ++r) { const double v = p[r * stride]; s += v; diff |= run_bits(v) ^ b0; }
  const double m = run_mean(s, rows, p[0], diff);
  double m2 = 0.0;
  r = 0;
  for (; r + 8 <= rows; r += 8) {
    double v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = p[(r + u) * stride];
#pragma unroll
    for (int u = 0; u < 8; ++u) { double d = v[u] - m; m2 = fma(d, d, m2); }
  }
  for (; r < rows; ++r) { double d = p[r * stride] - m; m2 = fma(d, d, m2); }
  return Moments{1.0, m, 0.0, m2};
}

constexpr int kNestedRecord = 14;     // doubles per entry of amwg_summary_nested's output: complete record, then two cut records

constexpr long long kNestedCtas = 1184;     // the CTA cap of the chain-wise kernels (amwg_summary.cuh kChainCtas)

// CTAs of the segment kernel: one thread per segment, capped; a function of the number of segments only
__host__ __device__ __forceinline__ long long nested_seg_ctas(long long n_seg) {
  return (n_seg + 255) / 256 < kNestedCtas ? (n_seg + 255) / 256 : kNestedCtas;
}

// segments of the shard [first_chain, first_chain + C): the superchains from floor(first / M) to floor((first + C - 1) / M)
__host__ __device__ __forceinline__ long long nested_segments(long long first_chain, long long C, long long M) {
  return (first_chain + C - 1) / M - first_chain / M + 1;
}

// the superchain of segment s and its local chains [c0, c1)
__host__ __device__ __forceinline__ long long nested_superchain(long long s, long long first_chain, long long M) {
  return first_chain / M + s;
}
__host__ __device__ __forceinline__ void nested_range(long long s, long long first_chain, long long C, long long M, long long& c0, long long& c1) {
  const long long k = nested_superchain(s, first_chain, M);
  c0 = k * M - first_chain;
  c1 = c0 + M;
  if (c0 < 0) c0 = 0;
  if (c1 > C) c1 = C;
}

// the output slot of a cut segment: 0 for the first segment, 1 for the last when it is another one; -1 for a complete segment
__host__ __device__ __forceinline__ int nested_cut_slot(long long s, long long first_chain, long long C, long long M) {
  long long c0, c1;
  nested_range(s, first_chain, C, M, c0, c1);
  if (c1 - c0 == M) return -1;
  return s == 0 ? 0 : 1;
}

// The chain-level record of local chains [c0, c1): each chain is (1, its mean, 0, its within-chain M2), merged in chain order.
// mean / m2 hold one entry's chains.
__host__ __device__ __forceinline__ Moments nested_chain_merge(const double* mean, const double* m2, long long c0, long long c1) {
  Moments r{0.0, 0.0, 0.0, 0.0};
  for (long long c = c0; c < c1; ++c) r = merge(r, Moments{1.0, mean[c], 0.0, m2[c]});
  return r;
}

// A whole superchain as one unit of the superchain-to-total level: (1, its mean, 0, B~_k + W-_k), with B~_k = M2 of its chain
// means / (M - 1) (0 when M = 1) and W-_k = its summed within-chain M2 / (M (rows - 1)) (0 when rows = 1)
__host__ __device__ __forceinline__ Moments nested_unit(const Moments& sc, long long M, long long rows) {
  const double b = M > 1 ? sc.m2 / (double)(M - 1) : 0.0;
  const double w = rows > 1 ? sc.sum_w / ((double)M * (double)(rows - 1)) : 0.0;
  return Moments{1.0, sc.mean, 0.0, b + w};
}

}  // namespace summary
