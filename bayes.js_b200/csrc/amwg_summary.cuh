// Post-path reductions on device (SURVEY 8(f).3). The reference hands back raw draws only (mcmc.js:1029) and leaves the
// summary (mean / sd / quantiles, README.md:44-52 plots them) to the caller; with 2^20..2^22 chains the raw block is GBs, so the
// summary is formed where the draws are and only a few hundred bytes cross PCIe / NVLink.
//
// Input everywhere: a device-resident sample block in amwg_sample_device's layout, x[row][entry][chain] (chain fastest).
//   K_m1  amwg_chain_moments_kernel : one thread per (chain, entry): mean and M2 of the chain over its rows, two sequential passes
//                                     (coalesced over chains; HBM-bound: 2 reads of the block), Chan-merged per CTA in a fixed tree
//   K_m2  amwg_merge_moments_kernel : one CTA per entry merges the per-CTA records, again in a FIXED order, so the result does
//                                     not depend on scheduling
//   K_q   amwg_digit_hist_kernel    : one pass of an exact MSD radix select over the order-preserving 64-bit key of the draws:
//                                     counts of the next 8-bit digit among the values whose higher digits equal a given prefix
//                                     (integer counts: exact, order independent, summed across GPUs by the caller)
//   K_a1  amwg_autocov_kernel       : one thread per chain: split-chain (two halves) moment records and lag sums of the draws and
//                                     of two tail indicators, for 16 lags per pass (effective sample size, split R-hat)
//   K_a2  amwg_merge_sums_kernel    : one CTA per (entry, series, lag) sums the per-CTA lag sums in a FIXED order
//   K_a3  amwg_autocov_sq_kernel    : K_a1's draws series of the squared deviations ((x - centre) * scale)^2 (mcse_sd)
//   K_i1  amwg_indicator_kernel     : one thread per chain: exact integer pair counts, edge terms and counts of the indicators
//                                     1[x <= q_k] of both halves, 4 thresholds and 64 lags per read (ess_quantile, mcse_quantile)
//   K_r0..K_r3  amwg_rank_hist / sort_count / sort_scan / sort_scatter : LSD radix sort of one entry's half-chain keys (8-bit
//                                     digits, stable; digit positions equal in all keys skipped) for the rank-normalised diagnostics
//   K_r4  amwg_rank_count_kernel    : merge-path rank counts of a sorted key array against another (integer, exact)
//   K_r5  amwg_rank_z_kernel        : normal scores of the average ranks, scattered into a [2h][1][chains] z-block
//   K_h0  amwg_finite_range_kernel  : smallest / largest finite draw (as order-preserving keys: u64 atomicMin / Max, exact and
//                                     order independent) and the counts of -inf, +inf and NaN, per entry
//   K_h1  amwg_hist_kernel          : equal-width 1-D histogram per entry (numpy.histogram's bin rule, amwg_hist.cuh) plus the
//                                     counts below / above the range and of NaN; 32-bit shared bins per CTA, 64-bit global flush
//   K_h2  amwg_hist2d_kernel        : 2-D histogram of a pair of entries (numpy.histogramdd's rule), up to 128 x 128 shared bins
//   K_c1  amwg_chain_means_kernel   : one thread per (chain, selected entry): the chain's mean over its rows (sequential sum)
//   K_c2  amwg_shard_mean_kernel    : one CTA per selected entry: the mean of the chain means, summed in a fixed tree
//   K_c3  amwg_gram_kernel          : upper-triangle 8 x 8 tiles of the Gram matrix of centred draws on the fp64 tensor core
//                                     (mma.sync m8n8k4 f64), 32-chain stages in shared memory; addressing in amwg_comoments.cuh
//   K_c4  amwg_sum_tiles_kernel     : sums the per-CTA partial tiles in CTA order
//   K_n1  amwg_nested_chain_kernel  : one thread per (chain, entry): mean and M2 of the chain over its rows (as K_m1), stored
//   K_n2  amwg_nested_seg_kernel    : one thread per superchain segment: its chains merged in chain order; complete superchains
//                                     as unit records into a fixed CTA tree (then K_m2), cut ones stored for the host
// Included at the end of amwg_kernels.cu (same translation unit: shares CUDA_TRY / fail()).
#pragma once

#include "amwg_autocov.cuh"      // the half-chain walk of K_a1
#include "amwg_comoments.cuh"
#include "amwg_hist.cuh"
#include "amwg_indicator.cuh"    // the half-chain walk of K_i1
#include "amwg_nested.cuh"      // Moments and merge

namespace summary {

constexpr int kMaxPrefixes = 32;      // distinct prefixes per entry and pass (order statistics being selected at once)
// CTAs per entry of the chain-wise kernels at most (chain_ctas): a fixed number, not the device's SM count; ~9 CTAs per SM of an
// H100.
constexpr long long kChainCtas = 1184;
static_assert(kNestedCtas == kChainCtas, "amwg_nested.cuh caps the segment kernel's grid like the chain-wise kernels");

// CTAs of a grid-stride kernel over n chains (or draws): min(ceil(n / 256), kChainCtas). It depends on n only, so the order in
// which the per-CTA records are merged, and with it the last bits of the result, is fixed.
inline long long chain_ctas(long long n) { return std::min((n + 255) / 256, kChainCtas); }

__device__ __forceinline__ unsigned long long ordered_key(double x) {
  unsigned long long u = (unsigned long long)__double_as_longlong(x);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);      // ascending keys == ascending doubles (-0 < +0, NaN on top)
}

template <int THREADS>
__device__ __forceinline__ Moments cta_merge(Moments* sh, Moments mine) {      // fixed tree: the result does not depend on scheduling
  const int t = threadIdx.x;
  sh[t] = mine;
  __syncthreads();
  for (int w = THREADS >> 1; w > 0; w >>= 1) {
    if (t < w) sh[t] = merge(sh[t], sh[t + w]);
    __syncthreads();
  }
  return sh[0];
}

// K_m1: per chain, mean and M2 over its rows (two sequential passes over a coalesced column); the CTA's chains are merged in a
// fixed order into one record per (entry, CTA).
__global__ void __launch_bounds__(256) amwg_chain_moments_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                                 Moments* __restrict__ partial) {
  __shared__ Moments sh[256];
  const int e = blockIdx.y;
  const size_t stride = (size_t)entries * C;
  Moments acc{0.0, 0.0, 0.0, 0.0};
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    acc = merge(acc, chain_record(x + (size_t)e * C + c, rows, stride));
  }
  const Moments tot = cta_merge<256>(sh, acc);
  if (threadIdx.x == 0) partial[(size_t)e * gridDim.x + blockIdx.x] = tot;
}

// K_m2: one CTA per entry merges the per-CTA records. out[entry][4] = {chains, mean of the chain means, M2 of the chain means,
// sum over chains of the within-chain M2}
__global__ void __launch_bounds__(1024) amwg_merge_moments_kernel(const Moments* __restrict__ partial, int n_partial, double* __restrict__ out) {
  __shared__ Moments sh[1024];
  const int e = blockIdx.x;
  Moments acc{0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < n_partial; i += 1024) acc = merge(acc, partial[(size_t)e * n_partial + i]);
  const Moments tot = cta_merge<1024>(sh, acc);
  if (threadIdx.x == 0) { out[e * 4 + 0] = tot.n; out[e * 4 + 1] = tot.mean; out[e * 4 + 2] = tot.m2; out[e * 4 + 3] = tot.sum_w; }
}

// counts[entry][prefix][256] += number of values of `entry` whose key's top 8*pass bits equal prefix[entry][p] and whose next
// byte is the bin. Grid: (chain blocks, entries). Shared-memory histogram per CTA, flushed with 64-bit global atomics.
__global__ void __launch_bounds__(256) amwg_digit_hist_kernel(const double* __restrict__ x, long long rows, int entries, long long C, int pass,
                                                              const unsigned long long* __restrict__ prefix, int n_prefix,
                                                              unsigned long long* __restrict__ counts) {
  __shared__ unsigned int hist[kMaxPrefixes * 256];
  __shared__ unsigned long long pre[kMaxPrefixes];
  const int e = blockIdx.y;
  for (int i = threadIdx.x; i < n_prefix * 256; i += blockDim.x) hist[i] = 0u;
  if (threadIdx.x < n_prefix) pre[threadIdx.x] = prefix[(size_t)e * n_prefix + threadIdx.x];
  __syncthreads();
  unsigned long long pre_lo = pre[0], pre_hi = pre[0];        // most values lie outside [lowest, highest] prefix in the late passes
  for (int q = 1; q < n_prefix; ++q) { pre_lo = pre[q] < pre_lo ? pre[q] : pre_lo; pre_hi = pre[q] > pre_hi ? pre[q] : pre_hi; }
  const int shift = 56 - 8 * pass;
  const size_t stride = (size_t)entries * C;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* p = x + (size_t)e * C + c;
    // consecutive rows of one chain mostly fall in the same bin (always, in the leading passes of a narrow posterior): count the
    // run in a register and touch the shared histogram once per run instead of once per value
    int last = -1;
    unsigned int run = 0;
    auto count = [&](double x) {
      const unsigned long long k = ordered_key(x);
      int idx = (int)((k >> shift) & 255ull);
      if (pass) {
        const unsigned long long hi = k >> (shift + 8);
        int q = n_prefix;
        if (hi >= pre_lo && hi <= pre_hi) { q = 0; while (q < n_prefix && pre[q] != hi) ++q; }   // the first match counts (padding repeats a prefix)
        idx = (q < n_prefix) ? q * 256 + idx : -1;
      }
      if (idx == last) { ++run; return; }
      if (last >= 0) atomicAdd(&hist[last], run);
      last = idx; run = 1;
    };
    long long r = 0;
    for (; r + 8 <= rows; r += 8) {                          // eight loads in flight per thread
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = p[(r + u) * stride];
#pragma unroll
      for (int u = 0; u < 8; ++u) count(v[u]);
    }
    for (; r < rows; ++r) count(p[r * stride]);
    if (last >= 0) atomicAdd(&hist[last], run);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_prefix * 256; i += blockDim.x)
    if (hist[i]) atomicAdd(&counts[(size_t)e * n_prefix * 256 + i], (unsigned long long)hist[i]);
}

// CTAs per entry of the counting kernels (digit_hist, the histograms): at most kChainCtas, doubled while one CTA would see 2^32
// values or more, because its shared bins are 32-bit (rows < 2^32 is checked by the callers).
inline int64_t count_ctas(int64_t chains, int64_t rows) {
  int64_t bx = chain_ctas(chains);
  while (256 * bx < chains && ((chains + bx - 1) / bx) * rows >= ((int64_t)1 << 32)) bx *= 2;     // bx < ceil(chains / 256)
  return bx;
}

// ---- posterior histograms (sample_summary(..., histogram=...)) -------------------------------------------------------------
constexpr int kMaxHistBins = 4096;     // 1-D bins per entry: (4097 edges x 8 B) + (4099 bins x 4 B) = 48 KB of shared memory
constexpr int kMaxPairBins = 128;      // bins per axis of a 2-D histogram: 128 x 128 x 4 B = 64 KB of shared memory
constexpr int kMaxPairs = 64;
constexpr unsigned long long kNoKey = ~0ull;     // above every finite value's key: "no finite draw" for the minimum

__device__ __forceinline__ double key_to_double(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// K_h0: one thread per chain walking its rows. Keys, not doubles, so that -0 < +0 and the extremes do not depend on the order in
// which the threads meet them. keys[entry][2] = {min, max} key of the finite draws; nonfinite[entry][3] = #-inf, #+inf, #NaN.
__global__ void __launch_bounds__(256) amwg_finite_range_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                                unsigned long long* __restrict__ keys, unsigned long long* __restrict__ nonfinite) {
  __shared__ unsigned long long sh[5][8];
  const int e = blockIdx.y;
  const size_t stride = (size_t)entries * C;
  unsigned long long kmin = kNoKey, kmax = 0ull, n_lo = 0, n_hi = 0, n_nan = 0;
  auto see = [&](double v) {
    if (isfinite(v)) {
      const unsigned long long k = ordered_key(v);
      kmin = k < kmin ? k : kmin;
      kmax = k > kmax ? k : kmax;
    } else if (v != v) {
      ++n_nan;
    } else if (v < 0.0) {
      ++n_lo;
    } else {
      ++n_hi;
    }
  };
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* p = x + (size_t)e * C + c;
    long long r = 0;
    for (; r + 8 <= rows; r += 8) {                          // eight loads in flight per thread
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = p[(r + u) * stride];
#pragma unroll
      for (int u = 0; u < 8; ++u) see(v[u]);
    }
    for (; r < rows; ++r) see(p[r * stride]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmin, o), b = __shfl_xor_sync(0xffffffffu, kmax, o);
    kmin = a < kmin ? a : kmin;
    kmax = b > kmax ? b : kmax;
    n_lo += __shfl_xor_sync(0xffffffffu, n_lo, o);
    n_hi += __shfl_xor_sync(0xffffffffu, n_hi, o);
    n_nan += __shfl_xor_sync(0xffffffffu, n_nan, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sh[0][w] = kmin; sh[1][w] = kmax; sh[2][w] = n_lo; sh[3][w] = n_hi; sh[4][w] = n_nan; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int v = 1; v < (int)(blockDim.x >> 5); ++v) {
      kmin = sh[0][v] < kmin ? sh[0][v] : kmin;
      kmax = sh[1][v] > kmax ? sh[1][v] : kmax;
      n_lo += sh[2][v]; n_hi += sh[3][v]; n_nan += sh[4][v];
    }
    if (kmin != kNoKey) atomicMin(&keys[2 * e], kmin);
    if (kmax != 0ull) atomicMax(&keys[2 * e + 1], kmax);
    if (n_lo) atomicAdd(&nonfinite[3 * e], n_lo);
    if (n_hi) atomicAdd(&nonfinite[3 * e + 1], n_hi);
    if (n_nan) atomicAdd(&nonfinite[3 * e + 2], n_nan);
  }
}

__global__ void amwg_range_init_kernel(unsigned long long* __restrict__ keys, unsigned long long* __restrict__ nonfinite, int entries) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < entries; i += gridDim.x * blockDim.x) {
    keys[2 * i] = kNoKey; keys[2 * i + 1] = 0ull;
    nonfinite[3 * i] = nonfinite[3 * i + 1] = nonfinite[3 * i + 2] = 0ull;
  }
}

// in place: the keys become the doubles they stand for, +inf / -inf when the entry has no finite draw
__global__ void amwg_range_final_kernel(unsigned long long* __restrict__ keys, int entries) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < entries; i += gridDim.x * blockDim.x) {
    const unsigned long long lo = keys[2 * i], hi = keys[2 * i + 1];
    reinterpret_cast<double*>(keys)[2 * i] = lo == kNoKey ? CUDART_INF : key_to_double(lo);
    reinterpret_cast<double*>(keys)[2 * i + 1] = hi == 0ull ? -CUDART_INF : key_to_double(hi);
  }
}

// K_h1: counts[entry][bins + 3] += the entry's 1-D histogram over edges[entry][bins + 1], then the draws below edges[0] (-inf
// included), above edges[bins] (+inf included) and NaN. Grid and run counting as in amwg_digit_hist_kernel: a rejected step repeats
// its value, so a chain's consecutive rows mostly share a bin and the shared bins are touched once per run. Dynamic shared memory:
// edges (doubles), then the bins (u32). Bounded to 64 registers (four CTAs per SM, which 4096 bins' 48 KB also allow): without
// the bound ptxas picks 64 registers anyway and spills.
__global__ void __launch_bounds__(256, 4) amwg_hist_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                        const double* __restrict__ edges, int bins, unsigned long long* __restrict__ counts) {
  extern __shared__ double hist_smem[];
  double* ed = hist_smem;
  unsigned* hist = reinterpret_cast<unsigned*>(ed + bins + 1);
  const int e = blockIdx.y;
  for (int i = threadIdx.x; i <= bins; i += blockDim.x) ed[i] = edges[(size_t)e * (bins + 1) + i];
  for (int i = threadIdx.x; i < bins + 3; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  const double lo = ed[0], hi = ed[bins];
  const size_t stride = (size_t)entries * C;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* p = x + (size_t)e * C + c;
    int last = -1;
    unsigned int run = 0;
    auto count = [&](double v) {
      const int idx = v < lo ? bins : v > hi ? bins + 1 : v != v ? bins + 2 : hist_bin(v, ed, bins);
      if (idx == last) { ++run; return; }
      if (last >= 0) atomicAdd(&hist[last], run);
      last = idx; run = 1;
    };
    long long r = 0;
    for (; r + 8 <= rows; r += 8) {                          // eight loads in flight per thread
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = p[(r + u) * stride];
#pragma unroll
      for (int u = 0; u < 8; ++u) count(v[u]);
    }
    for (; r < rows; ++r) count(p[r * stride]);
    if (last >= 0) atomicAdd(&hist[last], run);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bins + 3; i += blockDim.x)
    if (hist[i]) atomicAdd(&counts[(size_t)e * (bins + 3) + i], (unsigned long long)hist[i]);
}

struct PairList { int a[kMaxPairs], b[kMaxPairs]; };   // entry indices, passed by value (512 B of kernel parameters)

// K_h2: counts[pair][bins][bins] += the 2-D histogram of entries (a, b) of the pair, a on axis 0; a draw counts only when both of
// its values fall inside their axis's edges. Grid (chain blocks, pairs); runs as in K_h1. Dynamic shared memory: both axes'
// edges (doubles), then bins * bins u32 cells (64 KB at 128 bins).
__global__ void __launch_bounds__(256) amwg_hist2d_kernel(const double* __restrict__ x, long long rows, int entries, long long C, PairList pl,
                                                          const double* __restrict__ edges, int bins, unsigned long long* __restrict__ counts) {
  extern __shared__ double hist_smem[];
  double* ea = hist_smem;
  double* eb = ea + bins + 1;
  unsigned* cell = reinterpret_cast<unsigned*>(eb + bins + 1);
  const int pr = blockIdx.y, a = pl.a[pr], b = pl.b[pr];
  const int cells = bins * bins;
  for (int i = threadIdx.x; i <= bins; i += blockDim.x) { ea[i] = edges[(size_t)a * (bins + 1) + i]; eb[i] = edges[(size_t)b * (bins + 1) + i]; }
  for (int i = threadIdx.x; i < cells; i += blockDim.x) cell[i] = 0u;
  __syncthreads();
  const size_t stride = (size_t)entries * C;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* pa = x + (size_t)a * C + c;
    const double* pb = x + (size_t)b * C + c;
    int last = -1;
    unsigned int run = 0;
    auto count = [&](double va, double vb) {
      const int ia = hist2d_axis(va, ea, bins), ib = hist2d_axis(vb, eb, bins);
      const int idx = (ia < 0 || ib < 0) ? -1 : ia * bins + ib;
      if (idx == last) { ++run; return; }
      if (last >= 0) atomicAdd(&cell[last], run);
      last = idx; run = 1;
    };
    long long r = 0;
    for (; r + 8 <= rows; r += 8) {                          // eight rows (sixteen loads) in flight per thread
      double va[8], vb[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) { va[u] = pa[(r + u) * stride]; vb[u] = pb[(r + u) * stride]; }
#pragma unroll
      for (int u = 0; u < 8; ++u) count(va[u], vb[u]);
    }
    for (; r < rows; ++r) count(pa[r * stride], pb[r * stride]);
    if (last >= 0) atomicAdd(&cell[last], run);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cells; i += blockDim.x)
    if (cell[i]) atomicAdd(&counts[(size_t)pr * cells + i], (unsigned long long)cell[i]);
}

// ---- split-chain autocovariances (effective sample size, split R-hat) ------------------------------------------------------
// Every chain of `rows` kept draws is split into a first half (rows [0, h)) and a second half (rows [rows-h, rows)), h = rows/2.
// The per-half-chain records and lag sums, and the scaling of the draws series, are autocov_half's (amwg_autocov.cuh).

template <int THREADS>
__device__ __forceinline__ double cta_sum(double* sh, double mine) {            // fixed tree, like cta_merge
  const int t = threadIdx.x;
  sh[t] = mine;
  __syncthreads();
  for (int w = THREADS >> 1; w > 0; w >>= 1) {
    if (t < w) sh[t] += sh[t + w];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();                                                               // sh is reused by the next call
  return r;
}

// K_a1: one thread per chain (grid-stride), both halves, each by autocov_half. NS = 1: the draws only; NS = 3: also the two
// indicators of thr[e][0] and thr[e][1], and the draws scaled by autocov_scale(thr[e][0], thr[e][1]).
// pmom[(e*NS + s)][block] (skipped when null), psum[((e*NS + s)*n_total + k_base + k)][block] for k < n_lags.
template <int NS>
__global__ void __launch_bounds__(256) amwg_autocov_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                           const double* __restrict__ thr, long long lag0, int n_lags, int k_base, int n_total,
                                                           Moments* __restrict__ pmom, double* __restrict__ psum) {
  __shared__ Moments sh[256];
  const int e = blockIdx.y;
  const long long h = rows / 2;
  const size_t stride = (size_t)entries * C;
  double q0 = 0.0, q1 = 0.0, sc = 1.0;
  if constexpr (NS == 3) { q0 = thr[2 * e]; q1 = thr[2 * e + 1]; sc = autocov_scale(q0, q1); }
  double acc[NS][kLagSlots];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int k = 0; k < kLagSlots; ++k) acc[s][k] = 0.0;
  Moments mom[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) mom[s] = Moments{0.0, 0.0, 0.0, 0.0};

  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    for (int half = 0; half < 2; ++half)
      autocov_half<NS>(x + (size_t)e * C + c + (size_t)(half ? rows - h : 0) * stride, h, stride, q0, q1, sc, lag0, acc, mom);
  }
  if (pmom) {
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const Moments tot = cta_merge<256>(sh, mom[s]);
      if (threadIdx.x == 0) pmom[((size_t)e * NS + s) * gridDim.x + blockIdx.x] = tot;
      __syncthreads();
    }
  }
  double* shd = reinterpret_cast<double*>(sh);
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int k = 0; k < kLagSlots; ++k)
      if (k < n_lags) {
        const double tot = cta_sum<256>(shd, acc[s][k]);
        if (threadIdx.x == 0) psum[(((size_t)e * NS + s) * n_total + k_base + k) * gridDim.x + blockIdx.x] = tot;
      }
}

// K_a3: K_a1<1>'s walk and reductions for the draws series y = ((x - cs[e][0]) * cs[e][1])^2, the squared deviations behind
// mcse_sd: autocov_half with the SquaredDeviation transform. K_a1's text is left as it is, so its instructions do not change.
__global__ void __launch_bounds__(256) amwg_autocov_sq_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                              const double* __restrict__ cs, long long lag0, int n_lags, int k_base, int n_total,
                                                              Moments* __restrict__ pmom, double* __restrict__ psum) {
  __shared__ Moments sh[256];
  const int e = blockIdx.y;
  const long long h = rows / 2;
  const size_t stride = (size_t)entries * C;
  const SquaredDeviation tf{cs[2 * e], cs[2 * e + 1]};
  double acc[1][kLagSlots];
#pragma unroll
  for (int k = 0; k < kLagSlots; ++k) acc[0][k] = 0.0;
  Moments mom[1] = {Moments{0.0, 0.0, 0.0, 0.0}};
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    for (int half = 0; half < 2; ++half)
      autocov_half<1>(x + (size_t)e * C + c + (size_t)(half ? rows - h : 0) * stride, h, stride, 0.0, 0.0, 1.0, lag0, acc, mom, tf);
  }
  if (pmom) {
    const Moments tot = cta_merge<256>(sh, mom[0]);
    if (threadIdx.x == 0) pmom[(size_t)e * gridDim.x + blockIdx.x] = tot;
    __syncthreads();
  }
  double* shd = reinterpret_cast<double*>(sh);
#pragma unroll
  for (int k = 0; k < kLagSlots; ++k)
    if (k < n_lags) {
      const double tot = cta_sum<256>(shd, acc[0][k]);
      if (threadIdx.x == 0) psum[((size_t)e * n_total + k_base + k) * gridDim.x + blockIdx.x] = tot;
    }
}

// K_a2: one CTA per (entry, series, lag) sums the per-CTA lag sums in a fixed order.
__global__ void __launch_bounds__(256) amwg_merge_sums_kernel(const double* __restrict__ psum, int n_partial, double* __restrict__ out) {
  __shared__ double sh[256];
  const size_t row = blockIdx.x;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_partial; i += 256) acc += psum[row * n_partial + i];
  const double tot = cta_sum<256>(sh, acc);
  if (threadIdx.x == 0) out[row] = tot;
}

// ---- exact indicator autocovariances (ess_quantile and mcse_quantile of sample_summary(..., mcse=True)) ---------------------
// K_i1: one thread per chain (grid-stride in warp-uniform steps), both halves, each by indicator_half (amwg_indicator.cuh) for the
// kIndGroup thresholds of blockIdx.z. The sink sums each word's pair counts across the warp (redux.sync), gathers the sums of 32
// consecutive lags into the 32 lanes (lane l holds lag 32m + l) and adds them to per-CTA shared counters with one 64-bit shared
// atomic per lane; the edge terms go the same way (one 32-bit warp sum while h < 2048, else three 21-bit limbs), and the counts c
// and c^2 stay in registers until the end.
// The CTA then adds each counter to out with one 64-bit global atomic. Integers throughout: the result does not depend on the
// order of the atomics, the chain order or the launch shape.
struct WarpIndicatorSink {
  unsigned long long (*cnt)[2 + 2 * kIndLags];          // shared [kIndGroup][2 + 2 kIndLags]: C1, C2, P_t (i < 64), G_t (i < 64)
  unsigned lane;
  int n_lags;
  bool small;                                           // h < 2048: an edge term and its warp sum fit in 32 bits
  unsigned long long mine;                              // this lane's lag of the current block of 32
  unsigned long long c1[kIndGroup], c2[kIndGroup];

  __device__ __forceinline__ void flush(int k, int i, int base) {                // after lag i: lanes 0 .. i & 31 hold their lags
    if ((i & 31) == 31 || i == n_lags - 1)
      if (lane <= (unsigned)(i & 31)) atomicAdd(&cnt[k][base + (i & ~31) + (int)lane], mine);
  }
  __device__ __forceinline__ void pair(int k, int i, unsigned v) {
    const unsigned s = __reduce_add_sync(0xffffffffu, v);                 // <= 32 * 64
    if (lane == (unsigned)(i & 31)) mine = s;
    flush(k, i, 2);
  }
  // v = c (F_t + L_t) <= 2 h^2. h < 2048 (warp-uniform): v < 2^23, one 32-bit warp sum (< 2^28); else v < 2^63 in three limbs of
  // 21 bits, each warp sum < 2^26
  __device__ __forceinline__ void edge(int k, int i, unsigned long long v) {
    unsigned long long s;
    if (small) {
      s = __reduce_add_sync(0xffffffffu, (unsigned)v);
    } else {
      const unsigned long long s0 = __reduce_add_sync(0xffffffffu, (unsigned)(v & 0x1FFFFFull));
      const unsigned long long s1 = __reduce_add_sync(0xffffffffu, (unsigned)((v >> 21) & 0x1FFFFFull));
      const unsigned long long s2 = __reduce_add_sync(0xffffffffu, (unsigned)(v >> 42));
      s = s0 + (s1 << 21) + (s2 << 42);
    }
    if (lane == (unsigned)(i & 31)) mine = s;
    flush(k, i, 2 + kIndLags);
  }
  __device__ __forceinline__ void count(int k, long long c) {
    c1[k] += (unsigned long long)c;
    c2[k] += (unsigned long long)(c * c);
  }
};

// out[(e*K + k)][2 + 2*n_lags] += {C1, C2, P_t..., G_t...} (zeroed by the caller), thr[e][K]
__global__ void __launch_bounds__(256, 2) amwg_indicator_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                             const double* __restrict__ thr, int K, long long lag0, int n_lags,
                                                             unsigned long long* __restrict__ out) {
  __shared__ unsigned long long sh[kIndGroup][2 + 2 * kIndLags];
  __shared__ unsigned long long keep[4 * kIndGroup][256];            // indicator_half's four kept words per threshold and thread
  const int e = blockIdx.y, k0 = blockIdx.z * kIndGroup;
  const long long h = rows / 2;
  const size_t stride = (size_t)entries * C;
  double q[kIndGroup];
#pragma unroll
  for (int k = 0; k < kIndGroup; ++k) q[k] = k0 + k < K ? thr[(size_t)e * K + k0 + k] : __longlong_as_double(0x7ff8000000000000ll);   // NaN: no bits
  for (int i = threadIdx.x; i < kIndGroup * (2 + 2 * kIndLags); i += blockDim.x) (&sh[0][0])[i] = 0ull;
  __syncthreads();
  WarpIndicatorSink sink;
  sink.cnt = sh;
  sink.lane = threadIdx.x & 31u;
  sink.n_lags = n_lags;
  sink.small = h < 2048;
  sink.mine = 0ull;
#pragma unroll
  for (int k = 0; k < kIndGroup; ++k) sink.c1[k] = sink.c2[k] = 0ull;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long c0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); c0 < C; c0 += step) {   // warp-uniform bound
    const long long c = c0 + sink.lane;
    const bool live = c < C;
    const double* col = x + (size_t)e * C + (live ? c : 0);
    for (int half = 0; half < 2; ++half)
      indicator_half<kIndGroup>(col + (size_t)(half ? rows - h : 0) * stride, h, stride, live, q, lag0, n_lags, &keep[0][threadIdx.x], 256, sink);
  }
#pragma unroll
  for (int k = 0; k < kIndGroup; ++k) {
    unsigned long long a = sink.c1[k], b = sink.c2[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
    if (sink.lane == 0) { atomicAdd(&sh[k][0], a); atomicAdd(&sh[k][1], b); }
  }
  __syncthreads();
  const int w = 2 + 2 * n_lags;
  for (int i = threadIdx.x; i < kIndGroup * w; i += blockDim.x) {
    const int k = i / w, f = i % w;
    const int src = f < 2 + n_lags ? f : f - n_lags + kIndLags;       // G_t sits at 2 + kIndLags + i in shared memory
    const unsigned long long v = sh[k][src];
    if (k0 + k < K && v != 0ull) atomicAdd(&out[((size_t)e * K + k0 + k) * w + f], v);
  }
}

// ---- ranks over the pooled half-chain draws (rank-normalised R-hat, bulk effective sample size) -------------------------------
// One entry at a time. Its n = 2h * chains half-chain draws are numbered i = r * chains + c, r < 2h: rows [0, h) are r = 0..h-1
// and rows [rows-h, rows) are r = h..2h-1 (the middle row of odd rows is not ranked). A (key, i) pair per draw is sorted by an LSD
// radix sort of 8-bit digits with a stable scatter; ties keep the order of i, so the result is fully determined.
constexpr int kSortThreads = 256;
constexpr int kSortItems = 8;
constexpr int kSortTile = kSortThreads * kSortItems;           // keys per CTA in the count and scatter kernels
constexpr int kMergeItems = 8;
constexpr int kMergeTile = 256 * kMergeItems;                  // merged elements per CTA of the rank-count kernel

// canonical rank key: ordered_key of x (bulk) or of |x - centre| (folded), with -0 made +0 so that the two zeros tie
__device__ __forceinline__ unsigned long long rank_key(double x, bool folded, double centre) {
  const double v = folded ? fabs(x - centre) : x;
  return ordered_key(v == 0.0 ? 0.0 : v);
}

// Where a pass reads its (key, index) pairs: the first executed pass forms them from the block (index = i), later passes read
// the previous pass's output.
struct RankSource {
  const double* x; long long rows, C; size_t stride; int e; bool folded; double centre;
  const unsigned long long* keys; const unsigned* index;
  template <bool FROM_BLOCK>
  __device__ __forceinline__ void load(long long i, unsigned long long& k, unsigned& idx) const {
    if constexpr (FROM_BLOCK) {
      const long long h = rows / 2, r = i / C, c = i - r * C;
      k = rank_key(x[(size_t)(r < h ? r : rows - 2 * h + r) * stride + (size_t)e * C + c], folded, centre);
      idx = (unsigned)i;
    } else {
      k = keys[i];
      idx = index[i];
    }
  }
};

// K_r0: the eight digit histograms of one entry's keys, from one read of the block (hist[digit position][256], position 0 the
// least significant byte). Per thread, a run of equal bins is counted in a register (the high bytes of one parameter's draws
// rarely change) and added to the shared histogram once per run.
__global__ void __launch_bounds__(256) amwg_rank_hist_kernel(RankSource src, long long n, unsigned long long* __restrict__ hist) {
  __shared__ unsigned sh[8 * 256];
  for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) sh[i] = 0u;
  __syncthreads();
  int last[8];
  unsigned run[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) { last[d] = -1; run[d] = 0u; }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long k;
    unsigned idx;
    src.load<true>(i, k, idx);
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      const int b = d * 256 + (int)((k >> (8 * d)) & 255ull);
      if (b == last[d]) { ++run[d]; continue; }
      if (last[d] >= 0) atomicAdd(&sh[last[d]], run[d]);
      last[d] = b; run[d] = 1u;
    }
  }
#pragma unroll
  for (int d = 0; d < 8; ++d)
    if (last[d] >= 0) atomicAdd(&sh[last[d]], run[d]);
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], (unsigned long long)sh[i]);
}

// every pass skipped (all keys equal): the keys in input order
__global__ void __launch_bounds__(256) amwg_rank_fill_kernel(RankSource src, long long n, unsigned long long* __restrict__ keys,
                                                             unsigned* __restrict__ index) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    src.load<true>(i, keys[i], index[i]);
}

__device__ __forceinline__ int sort_digit(unsigned long long k, int shift) { return (int)((k >> shift) & 255ull); }

// K_r1 (upsweep): counts[digit][tile] of one pass's digit among the keys of each tile of kSortTile keys
template <bool FROM_BLOCK>
__global__ void __launch_bounds__(kSortThreads) amwg_sort_count_kernel(RankSource src, long long n, int shift, unsigned* __restrict__ counts) {
  __shared__ unsigned sh[256];
  const long long tiles = gridDim.x, tile = blockIdx.x, base = tile * kSortTile;
  sh[threadIdx.x] = 0u;
  __syncthreads();
  const unsigned lane = threadIdx.x & 31u;
#pragma unroll
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = base + j * kSortThreads + threadIdx.x;
    int d = 256;                                               // 256: past the end, counted nowhere
    if (i < n) { unsigned long long k; unsigned idx; src.load<FROM_BLOCK>(i, k, idx); d = sort_digit(k, shift); }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d < 256 && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&sh[d], (unsigned)__popc(peers));
  }
  __syncthreads();
  counts[(size_t)threadIdx.x * tiles + tile] = sh[threadIdx.x];
}

// K_r2 (scan): one CTA per digit turns counts[digit][tile] into the global position of the tile's first key of that digit:
// (keys of smaller digits, from the pass's histogram) + (keys of this digit in earlier tiles)
__global__ void __launch_bounds__(1024) amwg_sort_scan_kernel(const unsigned* __restrict__ counts, long long tiles,
                                                              const unsigned long long* __restrict__ hist, unsigned* __restrict__ offsets) {
  __shared__ unsigned long long sh[1024];
  const int d = blockIdx.x, t = threadIdx.x;
  unsigned long long below = 0;
  for (int b = t; b < d; b += 1024) below += hist[b];
  const long long per = (tiles + 1023) / 1024, lo = t * per, hi = lo + per < tiles ? lo + per : tiles;
  unsigned long long mine = 0;
  for (long long i = lo; i < hi; ++i) mine += counts[(size_t)d * tiles + i];
  sh[t] = below;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) { if (t < w) sh[t] += sh[t + w]; __syncthreads(); }
  const unsigned long long start = sh[0];
  __syncthreads();
  sh[t] = mine;                                                // inclusive Hillis-Steele scan of the per-thread sums
  __syncthreads();
  for (int w = 1; w < 1024; w <<= 1) {
    const unsigned long long v = t >= w ? sh[t - w] : 0ull;
    __syncthreads();
    sh[t] += v;
    __syncthreads();
  }
  unsigned long long run = start + sh[t] - mine;
  for (long long i = lo; i < hi; ++i) {
    const unsigned c = counts[(size_t)d * tiles + i];
    offsets[(size_t)d * tiles + i] = (unsigned)run;
    run += c;
  }
}

// K_r3 (downsweep): every tile ranks its keys stably by digit (rounds of 256 keys in input order; within a round, warp-level
// matching gives each key its place among equal digits), reorders them in shared memory and writes each digit's keys as one
// contiguous run at the tile's offset for that digit.
template <bool FROM_BLOCK>
__global__ void __launch_bounds__(kSortThreads) amwg_sort_scatter_kernel(RankSource src, long long n, int shift,
                                                                         const unsigned* __restrict__ counts, const unsigned* __restrict__ offsets,
                                                                         unsigned long long* __restrict__ keys_out, unsigned* __restrict__ index_out) {
  __shared__ unsigned long long sk[kSortTile];
  __shared__ unsigned si[kSortTile];
  __shared__ unsigned warp_cnt[kSortThreads / 32][256];
  __shared__ unsigned warp_off[kSortThreads / 32][256];
  __shared__ unsigned start[256];                              // first local position of each digit in the tile
  __shared__ unsigned seen[256];                               // keys of each digit placed by earlier rounds
  __shared__ long long dest[256];                              // global position of local position start[d]
  const long long tiles = gridDim.x, tile = blockIdx.x, base = tile * kSortTile;
  const int t = threadIdx.x, w = t >> 5;
  const unsigned lane = t & 31u, lt = (1u << lane) - 1u;
  {
    const unsigned c = counts[(size_t)t * tiles + tile];
    start[t] = c;
    __syncthreads();
    for (int s = 1; s < 256; s <<= 1) {                        // inclusive scan of the tile's digit counts
      const unsigned v = t >= s ? start[t - s] : 0u;
      __syncthreads();
      start[t] += v;
      __syncthreads();
    }
    const unsigned st = start[t] - c;
    __syncthreads();
    start[t] = st;
    seen[t] = 0u;
    dest[t] = (long long)offsets[(size_t)t * tiles + tile] - (long long)st;
    for (int v = 0; v < kSortThreads / 32; ++v) warp_cnt[v][t] = 0u;
  }
  __syncthreads();
#pragma unroll 1
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = base + j * kSortThreads + t;
    unsigned long long k = 0;
    unsigned idx = 0;
    int d = 256;
    if (i < n) { src.load<FROM_BLOCK>(i, k, idx); d = sort_digit(k, shift); }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & lt);
    if (d < 256 && rank == 0) warp_cnt[w][d] = __popc(peers);
    __syncthreads();
    unsigned run = seen[t];                                    // thread t owns digit t: exclusive prefix over the warps
#pragma unroll
    for (int v = 0; v < kSortThreads / 32; ++v) { const unsigned c = warp_cnt[v][t]; warp_off[v][t] = run; run += c; warp_cnt[v][t] = 0u; }
    seen[t] = run;
    __syncthreads();
    if (d < 256) {
      const unsigned pos = start[d] + warp_off[w][d] + rank;
      sk[pos] = k;
      si[pos] = idx;
    }
  }
  __syncthreads();
  const long long m = n - base < kSortTile ? n - base : kSortTile;
  for (int p = t; p < m; p += kSortThreads) {
    const unsigned long long k = sk[p];
    const long long g = dest[sort_digit(k, shift)] + p;
    keys_out[g] = k;
    index_out[g] = si[p];
  }
}

// K_r4: rank counts by merge path. acc[i] += #(R < Q[i]) (UPPER = false: Q first on ties) or #(R <= Q[i]) (UPPER = true: R
// first). Every CTA takes kMergeTile consecutive elements of the merged sequence; its share of Q and R is found by a binary
// search on the two cross diagonals, staged in shared memory, and merged there kMergeItems elements per thread.
template <bool UPPER>
__device__ __forceinline__ bool q_first(unsigned long long q, unsigned long long r) { return UPPER ? q < r : q <= r; }

template <bool UPPER>
__device__ __forceinline__ long long merge_path(const unsigned long long* Q, long long nq, const unsigned long long* R, long long nr, long long diag) {
  long long lo = diag > nr ? diag - nr : 0, hi = diag < nq ? diag : nq;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (q_first<UPPER>(Q[mid], R[diag - 1 - mid])) lo = mid + 1; else hi = mid;
  }
  return lo;                                                   // elements of Q among the first `diag` of the merge
}

template <bool UPPER>
__global__ void __launch_bounds__(256) amwg_rank_count_kernel(const unsigned long long* __restrict__ Q, long long nq,
                                                              const unsigned long long* __restrict__ R, long long nr, long long* __restrict__ acc) {
  __shared__ unsigned long long s[kMergeTile];                 // Q's share at [0, na), R's at [na, na + nb)
  __shared__ long long cnt[kMergeTile];
  __shared__ long long bounds[2];
  const long long d0 = (long long)blockIdx.x * kMergeTile, total = nq + nr;
  const long long d1 = d0 + kMergeTile < total ? d0 + kMergeTile : total;
  if (threadIdx.x < 2) bounds[threadIdx.x] = merge_path<UPPER>(Q, nq, R, nr, threadIdx.x ? d1 : d0);
  __syncthreads();
  const long long a0 = bounds[0], a1 = bounds[1], b0 = d0 - a0, b1 = d1 - a1;
  const int na = (int)(a1 - a0), nb = (int)(b1 - b0);
  for (int i = threadIdx.x; i < na + nb; i += blockDim.x) s[i] = i < na ? Q[a0 + i] : R[b0 + i - na];
  __syncthreads();
  const int diag = threadIdx.x * kMergeItems;
  if (diag < na + nb) {
    const unsigned long long* sq = s;
    const unsigned long long* sr = s + na;
    int i = (int)merge_path<UPPER>(sq, na, sr, nb, diag), j = diag - i;
    for (int step = 0; step < kMergeItems && i + j < na + nb; ++step) {
      if (i < na && (j >= nb || q_first<UPPER>(sq[i], sr[j]))) { cnt[i] = b0 + j; ++i; }
      else ++j;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < na; i += blockDim.x) acc[a0 + i] += cnt[i];
}

// K_r5: z = Phi^-1((r - 3/8) / (S + 1/4)) with the average rank r = (acc + 1) / 2, written at the draw's place in the z-block
__global__ void __launch_bounds__(256) amwg_rank_z_kernel(const long long* __restrict__ acc, const unsigned* __restrict__ index, long long n,
                                                          double total, double* __restrict__ z) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double r = (double)(acc[i] + 1) * 0.5;
    z[index[i]] = normcdfinv((r - 0.375) / (total + 0.25));
  }
}

// ---- posterior covariance (sample_summary(..., covariance=...)) -------------------------------------------------------------
// Record of a shard: chains, m[s] (mean of the chain means), B = sum_c (xbar_c - m)(xbar_c - m)^T and W = sum_c sum_r (x_rc -
// xbar_c)(x_rc - xbar_c)^T over the selected entries. W is the Gram matrix of the block's draws centred by their chain means; B is
// the same kernel's Gram matrix of the [1][sel][C] block of chain means centred by m.
struct SelList { int e[kMaxSel]; };      // block entry of each selected slot, passed by value (512 B of kernel parameters)

// K_c1: xbar[s][c] = the mean over rows of chain c of entry sel[s] (co_chain_mean, amwg_comoments.cuh)
__global__ void __launch_bounds__(256) amwg_chain_means_kernel(const double* __restrict__ x, long long rows, int entries, long long C, SelList sel,
                                                               double* __restrict__ xbar) {
  const int s = blockIdx.y;
  const size_t stride = (size_t)entries * C;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x)
    xbar[(size_t)s * C + c] = co_chain_mean(x + (size_t)sel.e[s] * C + c, rows, stride);
}

// K_c2: m[s] = (sum over chains of xbar[s][c], in a fixed order) / C, or the chain means' common value (co_mean_part)
__global__ void __launch_bounds__(256) amwg_shard_mean_kernel(const double* __restrict__ xbar, long long C, double* __restrict__ m) {
  __shared__ double sh[256];
  const int s = blockIdx.x;
  const CoMeanPart part = co_mean_part(xbar + (size_t)s * C, C, threadIdx.x, 256);
  const double tot = cta_sum<256>(sh, part.sum);
  const bool differ = __syncthreads_or(part.diff != 0);
  if (threadIdx.x == 0) m[s] = run_mean(tot, C, xbar[(size_t)s * C], differ ? 1 : 0);
}

__device__ __forceinline__ void dmma_8x8x4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// *a when p, else 0 without touching memory: a predicated load, which the compiler schedules together with its neighbours (a load
// under an `if` becomes a branch around it)
__device__ __forceinline__ double load_if(bool p, const double* a) {
  double v = 0.0;
  asm("{\n .reg .pred q;\n setp.ne.b32 q, %2, 0;\n @q ld.global.nc.f64 %0, [%1];\n}" : "+d"(v) : "l"(a), "r"((int)p));
  return v;
}

// stages values U0 .. U0 + 3 of this thread (value u is stage element i = threadIdx.x + u * kCoThreads; its chain is the lane,
// kCoThreads and kCoChains being multiples of 32): eight loads in flight, then the stores to shared memory
template <int U0>
__device__ __forceinline__ void gram_stage_part(double* st, const double* __restrict__ x, long long rows, int entries, long long C,
                                                const SelList& sel, int n_sel, const double* __restrict__ cen, long long cen_se,
                                                long long cen_sc, int nb, int per_stage, long long c0, long long r0) {
  double v[4];
  int sm[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = threadIdx.x + (U0 + u) * kCoThreads;
    const CoStageElem el = co_stage_elem(i, nb);
    const long long r = r0 + el.rr, c = c0 + el.cc;
    const bool p = i < per_stage && co_loads(r, el.s, c, rows, n_sel, C);
    const int e = p ? sel.e[el.s] : 0;
    v[u] = load_if(p, x + co_x_index(r, e, c, entries, C)) - load_if(p, cen + co_cen_index(el.s, c, cen_se, cen_sc));
    sm[u] = i < per_stage ? co_smem_index(el.rr, el.s, el.cc, nb) : -1;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (sm[u] >= 0) st[sm[u]] = v[u];
}

// K_c3: partial[cta][rep][tile][8][8] = this CTA's share of the upper-triangle tiles of sum_k d[i][k] d[j][k], with d the draws
// of x[row][sel[s]][chain] centred by cen[s * cen_se + chain * cen_sc]. Each CTA walks 32-chain groups (grid-stride) and, in each,
// stages of co_stage_rows(nb) rows: the threads stage the centred values in shared memory (two parts of four values, each part's
// eight loads in flight together; slots past n_sel and chains past C stage 0 and load nothing), then the warps add one DMMA per
// (row, quad) to each of the <= 9 tiles they own (per rep, amwg_comoments.cuh). The accumulators stay in registers for the whole
// walk: 128 registers, no spills, one 16-warp CTA per SM.
__global__ void __launch_bounds__(kCoThreads, 1) amwg_gram_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                                  SelList sel, int n_sel, const double* __restrict__ cen, long long cen_se,
                                                                  long long cen_sc, double* __restrict__ partial) {
  __shared__ double st[kCoSmem];
  const int nb = co_blocks(n_sel), srows = co_stage_rows(nb), reps = co_reps(nb);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, rep = co_warp_rep(warp, nb);
  const int per_stage = srows * 8 * nb * kCoChains;
  double acc[kCoSlots][2];
  unsigned frag[kCoSlots];                                   // the slot's A and B fragment offsets (co_frag_lane < 2^16), packed
  unsigned active = 0u;                                      // bit s: slot s holds a tile (warp-uniform)
#pragma unroll
  for (int s = 0; s < kCoSlots; ++s) {
    acc[s][0] = acc[s][1] = 0.0;
    const int t = co_slot_tile(warp, s, nb);
    int bi = 0, bj = 0;
    if (t >= 0) { co_tile(t, nb, bi, bj); active |= 1u << s; }
    frag[s] = (unsigned)co_frag_lane(lane, bi) | ((unsigned)co_frag_lane(lane, bj) << 16);
  }
  static_assert(kCoStageValues == 8 * kCoThreads && kCoThreads % 32 == 0 && kCoChains == 32, "stage layout");
  for (long long g = blockIdx.x; g * kCoChains < C; g += gridDim.x) {
    const long long c0 = g * kCoChains;
    const int nq = (int)((C - c0 < kCoChains ? C - c0 + 3 : kCoChains) / 4);     // quads holding at least one chain
    for (long long r0 = 0; r0 < rows; r0 += srows) {
      __syncthreads();                                       // every warp is done with the previous stage
      gram_stage_part<0>(st, x, rows, entries, C, sel, n_sel, cen, cen_se, cen_sc, nb, per_stage, c0, r0);
      gram_stage_part<4>(st, x, rows, entries, C, sel, n_sel, cen, cen_se, cen_sc, nb, per_stage, c0, r0);
      __syncthreads();
      const int nr = (int)(rows - r0 < srows ? rows - r0 : srows);
      for (int k = rep; k < nr * nq; k += reps) {
        const double* base = st + co_frag_base(k % nq, k / nq, nb);
#pragma unroll
        for (int s = 0; s < kCoSlots; ++s)
          if (active & (1u << s)) dmma_8x8x4(acc[s], base[frag[s] & 0xffffu], base[frag[s] >> 16]);
      }
    }
  }
#pragma unroll
  for (int s = 0; s < kCoSlots; ++s) {
    const int t = co_slot_tile(warp, s, nb);
    if (t >= 0) {
      partial[co_partial_index(blockIdx.x, rep, t, nb, lane, 0)] = acc[s][0];
      partial[co_partial_index(blockIdx.x, rep, t, nb, lane, 1)] = acc[s][1];
    }
  }
}

// K_c4: out[v] = sum over the n_parts = CTAs * reps records, in that order, of partial[part][v] for v < n_vals (= tiles * 64)
__global__ void __launch_bounds__(256) amwg_sum_tiles_kernel(const double* __restrict__ partial, int n_parts, int n_vals, double* __restrict__ out) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vals; v += gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int k = 0; k < n_parts; ++k) acc += partial[(size_t)k * n_vals + v];
    out[v] = acc;
  }
}

// ---- nested R-hat (sample_summary(..., nested=M), DESIGN.md §4.6); addressing and merges in amwg_nested.cuh -------------------
// K_n1: cm[e][c], cw[e][c] = mean and M2 of chain c of entry e over its rows (two sequential passes, as in K_m1)
__global__ void __launch_bounds__(256) amwg_nested_chain_kernel(const double* __restrict__ x, long long rows, int entries, long long C,
                                                                double* __restrict__ cm, double* __restrict__ cw) {
  const int e = blockIdx.y;
  const size_t stride = (size_t)entries * C;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const Moments r = chain_record(x + (size_t)e * C + c, rows, stride);
    cm[(size_t)e * C + c] = r.mean;
    cw[(size_t)e * C + c] = r.sum_w;
  }
}

// K_n2: one thread per segment (grid-stride): its chains merged in chain order. A complete segment becomes its superchain's unit
// record, merged into the thread's accumulator and then in the fixed CTA tree into partial[e][cta]; a cut one goes to cut[e][slot]
// as its chain-level record. The grid depends on the number of segments only, so the merge order is fixed.
__global__ void __launch_bounds__(256) amwg_nested_seg_kernel(const double* __restrict__ cm, const double* __restrict__ cw, long long C,
                                                              long long first_chain, long long M, long long rows, long long n_seg,
                                                              Moments* __restrict__ partial, Moments* __restrict__ cut) {
  __shared__ Moments sh[256];
  const int e = blockIdx.y;
  Moments acc{0.0, 0.0, 0.0, 0.0};
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += (long long)gridDim.x * blockDim.x) {
    long long c0, c1;
    nested_range(s, first_chain, C, M, c0, c1);
    const Moments r = nested_chain_merge(cm + (size_t)e * C, cw + (size_t)e * C, c0, c1);
    const int slot = nested_cut_slot(s, first_chain, C, M);
    if (slot < 0) acc = merge(acc, nested_unit(r, M, rows));
    else cut[(size_t)e * 2 + slot] = r;
  }
  const Moments tot = cta_merge<256>(sh, acc);
  if (threadIdx.x == 0) partial[(size_t)e * gridDim.x + blockIdx.x] = tot;
}

}  // namespace summary

extern "C" int amwg_summary_moments(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, double* host_stats) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_moments: empty sample block");
  if (!dev_samples || !host_stats) return fail("amwg_summary_moments: null pointer");
  if (summary::select_device(device, "amwg_summary_moments")) return -1;
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  const size_t need_out = (size_t)entries * 4 * sizeof(double);
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_moments", {(size_t)entries * bx * sizeof(summary::Moments), need_out})) return -1;
  auto* partial = sc.part<summary::Moments>(0);
  auto* d_out = sc.part<double>(1);
  summary::amwg_chain_moments_kernel<<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, partial);
  summary::amwg_merge_moments_kernel<<<(unsigned)entries, 1024>>>(partial, (int)bx, d_out);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(host_stats, d_out, need_out, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(std::string("amwg_summary_moments: ") + cudaGetErrorString(e));
  return 0;
}

extern "C" int amwg_summary_digit_hist(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int32_t pass,
                                       const uint64_t* dev_prefix, int32_t n_prefix, uint64_t* dev_counts) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_digit_hist: empty sample block");
  if (pass < 0 || pass > 7) return fail("amwg_summary_digit_hist: pass must be 0..7");
  if (n_prefix < 1 || n_prefix > summary::kMaxPrefixes) return fail("amwg_summary_digit_hist: n_prefix must be 1.." + std::to_string(summary::kMaxPrefixes));
  if (rows >= (int64_t)1 << 32) return fail("amwg_summary_digit_hist: more than 2^32 rows");
  if (!dev_samples || !dev_prefix || !dev_counts) return fail("amwg_summary_digit_hist: null pointer");
  if (summary::select_device(device, "amwg_summary_digit_hist")) return -1;
  const int64_t bx = summary::count_ctas(chains, rows);
  summary::amwg_digit_hist_kernel<<<dim3((unsigned)bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, pass,
                                                                                  reinterpret_cast<const unsigned long long*>(dev_prefix), n_prefix,
                                                                                  reinterpret_cast<unsigned long long*>(dev_counts));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

namespace summary {
// amwg_summary_autocov and amwg_summary_autocov_sq: the checks, the K_a1 / K_a3 passes (one per kLagSlots lags), the merges and
// the host record. sq: params[entry][2] = {centre, scale} of the squared deviations (K_a3); else thresholds[entry][2] or null (K_a1).
static int autocov_entry(const char* name, bool sq, int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                         const double* host_params, int64_t lag0, int32_t n_lags, double* host_out) {
  const std::string who(name);
  if (rows < 2) return fail(who + ": rows must be at least 2 (two half-chains of one draw)");
  if (entries <= 0 || chains <= 0) return fail(who + ": empty sample block");
  if (n_lags < 1 || n_lags > 2 * kLagSlots) return fail(who + ": n_lags must be 1.." + std::to_string(2 * kLagSlots));
  if (lag0 < 0 || lag0 + n_lags > rows / 2)
    return fail(who + ": the lag window [lag0, lag0 + n_lags) must lie in [0, rows/2) (rows/2 = " + std::to_string(rows / 2) + ")");
  if (!dev_samples || !host_out || (sq && !host_params)) return fail(who + ": null pointer");
  if (select_device(device, name)) return -1;
  const int ns = (host_params && !sq) ? 3 : 1;
  const unsigned bx = (unsigned)chain_ctas(chains);
  const size_t rec = (size_t)entries * ns, sums = rec * n_lags;
  Scratch sc;
  if (sc.acquire(device, name, {rec * bx * sizeof(Moments), sums * bx * sizeof(double), rec * 4 * sizeof(double),
                                sums * sizeof(double), (size_t)entries * 2 * sizeof(double)}))
    return -1;
  auto* pmom = sc.part<Moments>(0);
  auto* psum = sc.part<double>(1);
  auto* d_mom = sc.part<double>(2);
  auto* d_sum = sc.part<double>(3);
  auto* d_thr = sc.part<double>(4);
  if (host_params) CUDA_TRY(cudaMemcpy(d_thr, host_params, (size_t)entries * 2 * sizeof(double), cudaMemcpyHostToDevice));
  for (int k0 = 0; k0 < n_lags; k0 += kLagSlots) {                          // one pass over the block per kLagSlots lags
    const int nk = std::min(kLagSlots, n_lags - k0);
    Moments* pm = k0 == 0 ? pmom : nullptr;                                  // the records do not depend on the lags
    if (sq)
      amwg_autocov_sq_kernel<<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, d_thr, lag0 + k0, nk, k0, n_lags, pm, psum);
    else if (ns == 3)
      amwg_autocov_kernel<3><<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, d_thr, lag0 + k0, nk, k0, n_lags, pm, psum);
    else
      amwg_autocov_kernel<1><<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, nullptr, lag0 + k0, nk, k0, n_lags, pm, psum);
  }
  amwg_merge_moments_kernel<<<(unsigned)rec, 1024>>>(pmom, (int)bx, d_mom);
  amwg_merge_sums_kernel<<<(unsigned)sums, 256>>>(psum, (int)bx, d_sum);
  std::vector<double> mom(rec * 4), sm(sums);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(mom.data(), d_mom, mom.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(sm.data(), d_sum, sm.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(who + ": " + cudaGetErrorString(e));
  const size_t w = 4 + (size_t)n_lags;                                        // host_out[entry][series][4 + n_lags]
  for (size_t r = 0; r < rec; ++r) {
    for (int i = 0; i < 4; ++i) host_out[r * w + i] = mom[r * 4 + i];
    for (int k = 0; k < n_lags; ++k) host_out[r * w + 4 + k] = sm[r * n_lags + k];
  }
  return 0;
}
}  // namespace summary

extern "C" int amwg_summary_autocov(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                    const double* host_thresholds, int64_t lag0, int32_t n_lags, double* host_out) {
  return summary::autocov_entry("amwg_summary_autocov", false, device, dev_samples, rows, entries, chains, host_thresholds, lag0, n_lags, host_out);
}

extern "C" int amwg_summary_autocov_sq(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                       const double* host_centre, const double* host_scale, int64_t lag0, int32_t n_lags, double* host_out) {
  std::vector<double> cs;
  if (host_centre && host_scale && entries > 0) {
    cs.resize((size_t)entries * 2);
    for (int32_t e = 0; e < entries; ++e) { cs[2 * (size_t)e] = host_centre[e]; cs[2 * (size_t)e + 1] = host_scale[e]; }
  }
  return summary::autocov_entry("amwg_summary_autocov_sq", true, device, dev_samples, rows, entries, chains, cs.empty() ? nullptr : cs.data(),
                                lag0, n_lags, host_out);
}

extern "C" int amwg_summary_indicator_autocov(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                              const double* host_thresholds, int32_t n_thresholds, int64_t lag0, int32_t n_lags, int64_t* host_out) {
  if (rows < 2) return fail("amwg_summary_indicator_autocov: rows must be at least 2 (two half-chains of one draw)");
  if (rows >= (int64_t)1 << 32) return fail("amwg_summary_indicator_autocov: more than 2^32 rows");
  if (entries <= 0 || chains <= 0) return fail("amwg_summary_indicator_autocov: empty sample block");
  if (n_thresholds < 1 || n_thresholds > summary::kIndMaxThresholds)
    return fail("amwg_summary_indicator_autocov: n_thresholds must be 1.." + std::to_string(summary::kIndMaxThresholds));
  if (n_lags < 1 || n_lags > summary::kIndLags) return fail("amwg_summary_indicator_autocov: n_lags must be 1.." + std::to_string(summary::kIndLags));
  if (lag0 < 0 || lag0 + n_lags > rows / 2)
    return fail("amwg_summary_indicator_autocov: the lag window [lag0, lag0 + n_lags) must lie in [0, rows/2) (rows/2 = " + std::to_string(rows / 2) + ")");
  if (!dev_samples || !host_thresholds || !host_out) return fail("amwg_summary_indicator_autocov: null pointer");
  if (summary::select_device(device, "amwg_summary_indicator_autocov")) return -1;
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  const unsigned groups = (unsigned)((n_thresholds + summary::kIndGroup - 1) / summary::kIndGroup);
  const size_t n_thr = (size_t)entries * n_thresholds, n_out = n_thr * (2 + 2 * (size_t)n_lags);
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_indicator_autocov", {n_thr * sizeof(double), n_out * sizeof(int64_t)})) return -1;
  auto* d_thr = sc.part<double>(0);
  auto* d_out = sc.part<unsigned long long>(1);
  CUDA_TRY(cudaMemcpy(d_thr, host_thresholds, n_thr * sizeof(double), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(d_out, 0, n_out * sizeof(int64_t)));
  summary::amwg_indicator_kernel<<<dim3(bx, (unsigned)entries, groups), 256>>>(dev_samples, rows, entries, chains, d_thr, n_thresholds, lag0,
                                                                              n_lags, d_out);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(host_out, d_out, n_out * sizeof(int64_t), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(std::string("amwg_summary_indicator_autocov: ") + cudaGetErrorString(e));
  return 0;
}

extern "C" int amwg_summary_rank_sort(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int32_t entry,
                                      double centre, uint64_t* dev_keys, uint32_t* dev_index, int32_t* host_passes) {
  if (rows < 2) return fail("amwg_summary_rank_sort: rows must be at least 2 (two half-chains of one draw)");
  if (entries <= 0 || chains <= 0) return fail("amwg_summary_rank_sort: empty sample block");
  if (entry < 0 || entry >= entries) return fail("amwg_summary_rank_sort: entry outside [0, entries)");
  const int64_t n = 2 * (rows / 2) * chains;
  if (n >= ((int64_t)1 << 32) || chains >= ((int64_t)1 << 32))
    return fail("amwg_summary_rank_sort: 2 * (rows / 2) * chains = " + std::to_string(n) + " draws, the indices hold fewer than 2^32");
  if (!dev_samples || !dev_keys || !dev_index) return fail("amwg_summary_rank_sort: null pointer");
  if (summary::select_device(device, "amwg_summary_rank_sort")) return -1;
  const long long tiles = (n + summary::kSortTile - 1) / summary::kSortTile;
  const size_t b_tab = (size_t)256 * tiles * sizeof(unsigned);
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_rank_sort", {8 * 256 * sizeof(unsigned long long), b_tab, b_tab})) return -1;
  auto* hist = sc.part<unsigned long long>(0);
  auto* counts = sc.part<unsigned>(1);
  auto* offsets = sc.part<unsigned>(2);
  auto* keys = reinterpret_cast<unsigned long long*>(dev_keys);
  summary::RankSource src{dev_samples, rows, chains, (size_t)entries * chains, entry, !std::isnan(centre), centre, nullptr, nullptr};
  CUDA_TRY(cudaMemset(hist, 0, 8 * 256 * sizeof(unsigned long long)));
  // one read of the block forms all eight digit histograms. A digit position where one bin holds every key has the same digit
  // in all keys: its pass would move nothing and is skipped. The first executed pass forms the keys from the block again, into
  // the half that makes the last pass end in the first half.
  const unsigned gx = (unsigned)summary::chain_ctas(n);
  summary::amwg_rank_hist_kernel<<<gx, 256>>>(src, n, hist);
  CUDA_TRY(cudaGetLastError());
  std::vector<unsigned long long> h(8 * 256);
  CUDA_TRY(cudaMemcpy(h.data(), hist, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  std::vector<int> run;
  for (int d = 0; d < 8; ++d)
    if (*std::max_element(h.begin() + d * 256, h.begin() + (d + 1) * 256) != (unsigned long long)n) run.push_back(d);
  if (run.empty()) summary::amwg_rank_fill_kernel<<<gx, 256>>>(src, n, keys, dev_index);
  int dst = run.size() % 2 ? 0 : 1;
  for (size_t p = 0; p < run.size(); ++p) {
    const int d = run[p];
    const unsigned tg = (unsigned)tiles;
    if (p == 0) {
      summary::amwg_sort_count_kernel<true><<<tg, summary::kSortThreads>>>(src, n, 8 * d, counts);
      summary::amwg_sort_scan_kernel<<<256, 1024>>>(counts, tiles, hist + d * 256, offsets);
      summary::amwg_sort_scatter_kernel<true><<<tg, summary::kSortThreads>>>(src, n, 8 * d, counts, offsets, keys + dst * n, dev_index + dst * n);
    } else {
      summary::RankSource prev = src;
      prev.keys = keys + (1 - dst) * n;
      prev.index = dev_index + (1 - dst) * n;
      summary::amwg_sort_count_kernel<false><<<tg, summary::kSortThreads>>>(prev, n, 8 * d, counts);
      summary::amwg_sort_scan_kernel<<<256, 1024>>>(counts, tiles, hist + d * 256, offsets);
      summary::amwg_sort_scatter_kernel<false><<<tg, summary::kSortThreads>>>(prev, n, 8 * d, counts, offsets, keys + dst * n, dev_index + dst * n);
    }
    dst = 1 - dst;
  }
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  if (host_passes) *host_passes = (int32_t)run.size();
  return 0;
}

extern "C" int amwg_summary_rank_count(int device, const uint64_t* dev_q, int64_t nq, const uint64_t* dev_r, int64_t nr, int64_t* dev_acc) {
  if (nq < 1 || nr < 1) return fail("amwg_summary_rank_count: empty key array");
  if (nq >= ((int64_t)1 << 32) || nr >= ((int64_t)1 << 32)) return fail("amwg_summary_rank_count: more than 2^32 - 1 keys");
  if (!dev_q || !dev_r || !dev_acc) return fail("amwg_summary_rank_count: null pointer");
  if (summary::select_device(device, "amwg_summary_rank_count")) return -1;
  const unsigned grid = (unsigned)((nq + nr + summary::kMergeTile - 1) / summary::kMergeTile);
  auto* q = reinterpret_cast<const unsigned long long*>(dev_q);
  auto* r = reinterpret_cast<const unsigned long long*>(dev_r);
  auto* acc = reinterpret_cast<long long*>(dev_acc);
  summary::amwg_rank_count_kernel<false><<<grid, 256>>>(q, nq, r, nr, acc);
  summary::amwg_rank_count_kernel<true><<<grid, 256>>>(q, nq, r, nr, acc);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

extern "C" int amwg_summary_rank_z(int device, const int64_t* dev_acc, const uint32_t* dev_index, int64_t n, int64_t total, double* dev_z) {
  if (n < 1 || n >= ((int64_t)1 << 32)) return fail("amwg_summary_rank_z: n must be 1..2^32-1");
  if (total < n || total >= ((int64_t)1 << 52)) return fail("amwg_summary_rank_z: total must be at least n and below 2^52");
  if (!dev_acc || !dev_index || !dev_z) return fail("amwg_summary_rank_z: null pointer");
  if (summary::select_device(device, "amwg_summary_rank_z")) return -1;
  const unsigned grid = (unsigned)summary::chain_ctas(n);
  summary::amwg_rank_z_kernel<<<grid, 256>>>(reinterpret_cast<const long long*>(dev_acc), dev_index, n, (double)total, dev_z);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

extern "C" int amwg_summary_finite_range(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                         double* dev_range, int64_t* dev_nonfinite) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_finite_range: empty sample block");
  if (!dev_samples || !dev_range || !dev_nonfinite) return fail("amwg_summary_finite_range: null pointer");
  if (summary::select_device(device, "amwg_summary_finite_range")) return -1;
  auto* keys = reinterpret_cast<unsigned long long*>(dev_range);
  auto* nonfinite = reinterpret_cast<unsigned long long*>(dev_nonfinite);
  const unsigned small = (unsigned)std::min<int64_t>((entries + 255) / 256, 1024);
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  summary::amwg_range_init_kernel<<<small, 256>>>(keys, nonfinite, entries);
  summary::amwg_finite_range_kernel<<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, keys, nonfinite);
  summary::amwg_range_final_kernel<<<small, 256>>>(keys, entries);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

extern "C" int amwg_summary_histogram(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                      const double* dev_edges, int32_t bins, int64_t* dev_counts) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_histogram: empty sample block");
  if (bins < 1 || bins > summary::kMaxHistBins) return fail("amwg_summary_histogram: bins must be 1.." + std::to_string(summary::kMaxHistBins));
  if (rows >= (int64_t)1 << 32) return fail("amwg_summary_histogram: more than 2^32 rows");
  if (!dev_samples || !dev_edges || !dev_counts) return fail("amwg_summary_histogram: null pointer");
  if (summary::select_device(device, "amwg_summary_histogram")) return -1;
  const size_t smem = (size_t)(bins + 1) * sizeof(double) + (size_t)(bins + 3) * sizeof(unsigned);
  CUDA_TRY(cudaFuncSetAttribute(summary::amwg_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t bx = summary::count_ctas(chains, rows);
  summary::amwg_hist_kernel<<<dim3((unsigned)bx, (unsigned)entries), 256, smem>>>(dev_samples, rows, entries, chains, dev_edges, bins,
                                                                                  reinterpret_cast<unsigned long long*>(dev_counts));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

extern "C" int amwg_summary_histogram2d(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                        const int32_t* host_pairs, int32_t n_pairs, const double* dev_edges, int32_t bins, int64_t* dev_counts) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_histogram2d: empty sample block");
  if (bins < 1 || bins > summary::kMaxPairBins) return fail("amwg_summary_histogram2d: bins must be 1.." + std::to_string(summary::kMaxPairBins));
  if (n_pairs < 1 || n_pairs > summary::kMaxPairs) return fail("amwg_summary_histogram2d: n_pairs must be 1.." + std::to_string(summary::kMaxPairs));
  if (rows >= (int64_t)1 << 32) return fail("amwg_summary_histogram2d: more than 2^32 rows");
  if (!dev_samples || !host_pairs || !dev_edges || !dev_counts) return fail("amwg_summary_histogram2d: null pointer");
  summary::PairList pl;
  for (int i = 0; i < n_pairs; ++i) {
    pl.a[i] = host_pairs[2 * i];
    pl.b[i] = host_pairs[2 * i + 1];
    if (pl.a[i] < 0 || pl.a[i] >= entries || pl.b[i] < 0 || pl.b[i] >= entries)
      return fail("amwg_summary_histogram2d: pair " + std::to_string(i) + " names an entry outside [0, entries)");
  }
  if (summary::select_device(device, "amwg_summary_histogram2d")) return -1;
  const size_t smem = (size_t)2 * (bins + 1) * sizeof(double) + (size_t)bins * bins * sizeof(unsigned);
  CUDA_TRY(cudaFuncSetAttribute(summary::amwg_hist2d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t bx = summary::count_ctas(chains, rows);
  summary::amwg_hist2d_kernel<<<dim3((unsigned)bx, (unsigned)n_pairs), 256, smem>>>(dev_samples, rows, entries, chains, pl, dev_edges, bins,
                                                                                    reinterpret_cast<unsigned long long*>(dev_counts));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

extern "C" int amwg_summary_comoments(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                      const int32_t* host_sel, int32_t n_sel, double* host_out) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_comoments: empty sample block");
  if (n_sel < 1 || n_sel > summary::kMaxSel) return fail("amwg_summary_comoments: n_sel must be 1.." + std::to_string(summary::kMaxSel));
  if (!dev_samples || !host_sel || !host_out) return fail("amwg_summary_comoments: null pointer");
  summary::SelList sel{};
  for (int i = 0; i < n_sel; ++i) {
    if (host_sel[i] < 0 || host_sel[i] >= entries)
      return fail("amwg_summary_comoments: selected entry " + std::to_string(i) + " is outside [0, entries)");
    sel.e[i] = host_sel[i];
  }
  if (rows > (((int64_t)1 << 53) - 1) / chains) return fail("amwg_summary_comoments: rows * chains must be below 2^53");
  if (summary::select_device(device, "amwg_summary_comoments")) return -1;
  const int nb = summary::co_blocks(n_sel), tiles = summary::co_tiles(nb), n_vals = tiles * 64;
  const long long gx = summary::co_ctas(chains), parts = gx * summary::co_reps(nb);
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_comoments", {(size_t)n_sel * chains * 8, (size_t)n_sel * 8, (size_t)parts * n_vals * 8, (size_t)2 * n_vals * 8}))
    return -1;
  auto* xbar = sc.part<double>(0);
  auto* m = sc.part<double>(1);
  auto* part = sc.part<double>(2);
  auto* tw = sc.part<double>(3);
  double* tb = tw + n_vals;
  summary::SelList ident{};
  for (int i = 0; i < n_sel; ++i) ident.e[i] = i;
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  const unsigned sx = (unsigned)((n_vals + 255) / 256);
  summary::amwg_chain_means_kernel<<<dim3(bx, (unsigned)n_sel), 256>>>(dev_samples, rows, entries, chains, sel, xbar);
  summary::amwg_shard_mean_kernel<<<(unsigned)n_sel, 256>>>(xbar, chains, m);
  summary::amwg_gram_kernel<<<(unsigned)gx, summary::kCoThreads>>>(dev_samples, rows, entries, chains, sel, n_sel, xbar, chains, 1, part);
  summary::amwg_sum_tiles_kernel<<<sx, 256>>>(part, (int)parts, n_vals, tw);
  summary::amwg_gram_kernel<<<(unsigned)gx, summary::kCoThreads>>>(xbar, 1, n_sel, chains, ident, n_sel, m, 1, 0, part);
  summary::amwg_sum_tiles_kernel<<<sx, 256>>>(part, (int)parts, n_vals, tb);
  std::vector<double> hm(n_sel), ht(2 * (size_t)n_vals);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(hm.data(), m, hm.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(ht.data(), tw, ht.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(std::string("amwg_summary_comoments: ") + cudaGetErrorString(e));
  // host_out = { C, m[n], B[n][n], W[n][n] }: the upper triangle of each tile, mirrored, so both matrices are exactly symmetric
  const size_t n = (size_t)n_sel;
  double* oB = host_out + 1 + n;
  double* oW = oB + n * n;
  host_out[0] = (double)chains;
  for (size_t i = 0; i < n; ++i) host_out[1 + i] = hm[i];
  for (int t = 0; t < tiles; ++t) {
    int bi = 0, bj = 0;
    summary::co_tile(t, nb, bi, bj);
    for (int r = 0; r < 8; ++r)
      for (int c = 0; c < 8; ++c) {
        const size_t i = 8 * (size_t)bi + r, j = 8 * (size_t)bj + c;
        if (i > j || j >= n) continue;
        oW[i * n + j] = oW[j * n + i] = ht[(size_t)t * 64 + r * 8 + c];
        oB[i * n + j] = oB[j * n + i] = ht[(size_t)n_vals + (size_t)t * 64 + r * 8 + c];
      }
  }
  return 0;
}

extern "C" int amwg_summary_nested(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int64_t first_chain,
                                   int64_t superchain_size, double* host_out) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_nested: empty sample block");
  if (!dev_samples || !host_out) return fail("amwg_summary_nested: null pointer");
  if (superchain_size < 1) return fail("amwg_summary_nested: superchain_size must be >= 1");
  if (first_chain < 0) return fail("amwg_summary_nested: first_chain must be >= 0");
  if (first_chain > ((int64_t)1 << 53) - chains) return fail("amwg_summary_nested: first_chain + chains must be at most 2^53");
  if (summary::select_device(device, "amwg_summary_nested")) return -1;
  const long long M = superchain_size, n_seg = summary::nested_segments(first_chain, chains, M);
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  const unsigned sx = (unsigned)summary::nested_seg_ctas(n_seg);     // depends on n_seg only: a fixed merge order
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_nested", {(size_t)entries * chains * 16, (size_t)entries * sx * sizeof(summary::Moments),
                                                 (size_t)entries * 4 * sizeof(double), (size_t)entries * 2 * sizeof(summary::Moments)}))
    return -1;
  auto* cm = sc.part<double>(0);
  auto* cw = cm + (size_t)entries * chains;
  auto* part = sc.part<summary::Moments>(1);
  auto* d_out = sc.part<double>(2);
  auto* cut = sc.part<summary::Moments>(3);
  summary::amwg_nested_chain_kernel<<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, cm, cw);
  summary::amwg_nested_seg_kernel<<<dim3(sx, (unsigned)entries), 256>>>(cm, cw, chains, first_chain, M, rows, n_seg, part, cut);
  summary::amwg_merge_moments_kernel<<<(unsigned)entries, 1024>>>(part, (int)sx, d_out);
  std::vector<double> tot((size_t)entries * 4), cr((size_t)entries * 8);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(tot.data(), d_out, tot.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(cr.data(), cut, cr.size() * sizeof(double), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(std::string("amwg_summary_nested: ") + cudaGetErrorString(e));
  // host_out[entry][14] = { complete record (4), then per cut slot { superchain id (-1: none), chains, mean, M2, sum_w } }
  long long slot_seg[2] = {-1, -1};
  for (long long s : {0LL, n_seg - 1}) {
    const int slot = summary::nested_cut_slot(s, first_chain, chains, M);
    if (slot >= 0) slot_seg[slot] = s;
  }
  for (int32_t en = 0; en < entries; ++en) {
    double* o = host_out + (size_t)en * summary::kNestedRecord;
    for (int i = 0; i < 4; ++i) o[i] = tot[(size_t)en * 4 + i];
    for (int slot = 0; slot < 2; ++slot) {
      double* q = o + 4 + 5 * slot;
      const double* r = cr.data() + ((size_t)en * 2 + slot) * 4;
      if (slot_seg[slot] < 0) { q[0] = -1.0; q[1] = q[2] = q[3] = q[4] = 0.0; continue; }
      q[0] = (double)summary::nested_superchain(slot_seg[slot], first_chain, M);
      for (int i = 0; i < 4; ++i) q[1 + i] = r[i];
    }
  }
  return 0;
}
