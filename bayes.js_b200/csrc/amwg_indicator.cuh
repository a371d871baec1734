// The per-half-chain walk of amwg_indicator_kernel (amwg_summary.cuh, K_i1): exact integer autocovariance sums of the indicators
// b_n = 1[x_n <= q_k] of one half-chain, for a group of kIndGroup thresholds and a window of up to kIndLags lags, from one read of
// the half. One __host__ __device__ text, so that the kernel and the host build the CPU tests run (tests/host_shim/indicator_host.cpp)
// count alike.
//
// Per half-chain of h positions and threshold q (c = sum_n b_n, F_t / L_t = the count among the first / last t positions):
//   pair  P_t = sum_{n<h-t} b_n b_{n+t}            for t = lag0 + i, i < kIndLags
//   edge  c * (F_t + L_t)                          for the same t
//   count c (and c^2)
// The half is read in 64-row words; each draw read is compared against every threshold of the group and sets one bit of that
// threshold's word. A word of the half at positions [64j, 64j + 64) is ANDed with the lead bits at positions 64j + t + [0, 64):
// lag0 is split into a = lag0 / 64 words and r = lag0 % 64 bits, a ring holds the lead words j + a .. j + a + 2, and two
// funnel shifts by r align them at lag0, so every lag of the window is one more shift, an AND and a popcount. Positions at or past
// h are 0 bits, so a pair counts exactly when both ends lie in the half. When a = 0 the half's own word is the ring's first word
// and the half is read once; otherwise the half's word is read separately (two reads).
//
// The sink receives the integers: pair(k, i, v) once per word and (k, i) with this half's popcount v <= 64, edge(k, i, v) and
// count(k, c) once per half; pair and edge come in ascending i for each k. All lanes of a warp call it in step (the walk's control flow depends on h and lag0 only), so the
// device sink can sum across the warp.
#pragma once

namespace summary {

constexpr int kIndGroup = 4;          // thresholds per read of the block (the kernel's register ring holds 3 lead words each)
constexpr int kIndLags = 64;          // lags per window: one 64-bit word of lead bits
constexpr int kIndMaxThresholds = 16; // thresholds per call (amwg_summary_indicator_autocov)

// bits of 64 rows [64j, 64j + 64) of a half (rows at or past h, and every row when !live, give 0 bits)
template <int G>
__host__ __device__ __forceinline__ void indicator_word(const double* __restrict__ p, long long h, size_t stride, bool live, const double (&q)[G],
                                                        long long j, unsigned long long (&w)[G]) {
#pragma unroll
  for (int k = 0; k < G; ++k) w[k] = 0ull;
  const long long n0 = j * 64;
  if (!live || n0 >= h) return;
  const int nb = (int)(h - n0 < 64 ? h - n0 : 64);
  int b = 0;
  for (; b + 8 <= nb; b += 8) {                          // eight loads in flight per thread
    double v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = p[(size_t)(n0 + b + u) * stride];
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
      for (int k = 0; k < G; ++k) w[k] |= (unsigned long long)(v[u] <= q[k]) << (b + u);
  }
  for (; b < nb; ++b) {
    const double v = p[(size_t)(n0 + b) * stride];
#pragma unroll
    for (int k = 0; k < G; ++k) w[k] |= (unsigned long long)(v <= q[k]) << b;
  }
}

__host__ __device__ __forceinline__ int popcount64(unsigned long long v) {
#ifdef __CUDA_ARCH__
  return __popcll(v);
#else
  return __builtin_popcountll(v);
#endif
}

// bits [s, s + 64) of the 128-bit value (hi:lo), 0 <= s < 64
__host__ __device__ __forceinline__ unsigned long long shift128(unsigned long long lo, unsigned long long hi, int s) {
  return s == 0 ? lo : (lo >> s) | (hi << (64 - s));
}

// the low s bits, 0 <= s <= 64
__host__ __device__ __forceinline__ unsigned long long low_bits(int s) { return s >= 64 ? ~0ull : ((1ull << s) - 1ull); }

// F(s) = the count of positions [0, s) from the words w0 (at word s0 = the word index of the first position asked for) and
// w1 (word s0 + 1) and the count p0 of the positions before word s0
__host__ __device__ __forceinline__ long long prefix_count(long long s, long long s0, unsigned long long w0, unsigned long long w1, long long p0) {
  const long long ws = s >> 6;
  const int bits = (int)(s & 63);
  return ws == s0 ? p0 + popcount64(w0 & low_bits(bits)) : p0 + popcount64(w0) + popcount64(w1 & low_bits(bits));
}

// One half-chain p[n * stride], n < h < 2^31 (live: this lane holds a chain; a lane without one walks zero bits, so the sink's warp
// sums see every lane). n_lags <= kIndLags lags t = lag0 + i, lag0 + n_lags <= h. keep holds the four words the edge terms read
// (the two at F_t's positions, the two at F_{h-t}'s), word (slot, k) at keep[(slot * G + k) * kstride]: the kernel keeps them in
// shared memory, out of the registers the walk needs.
template <int G, class Sink>
__host__ __device__ __forceinline__ void indicator_half(const double* __restrict__ p, long long h, size_t stride, bool live, const double (&q)[G],
                                                        long long lag0, int n_lags, unsigned long long* keep, int kstride, Sink& sink) {
  const long long nw = (h + 63) >> 6;
  const long long a = lag0 >> 6;
  const int r = (int)(lag0 & 63);
  // the words that hold the positions F_t and F_{h-t} need: s in [lag0, lag0 + n_lags) and in [h - lag0 - n_lags + 1, h - lag0]
  const long long jf = lag0 >> 6;
  const long long jl = (h - lag0 - n_lags + 1) >> 6;
  unsigned long long ring[3][G];
  int pc[G], pf[G], pl[G];                               // counts below 2^31
  auto kept = [&](int slot, int k) -> unsigned long long& { return keep[(size_t)(slot * G + k) * kstride]; };
#pragma unroll
  for (int k = 0; k < G; ++k) {
    pc[k] = pf[k] = pl[k] = 0;
#pragma unroll
    for (int slot = 0; slot < 4; ++slot) kept(slot, k) = 0ull;
  }
  indicator_word<G>(p, h, stride, live, q, a, ring[0]);
  indicator_word<G>(p, h, stride, live, q, a + 1, ring[1]);
  indicator_word<G>(p, h, stride, live, q, a + 2, ring[2]);
  for (long long j = 0; j < nw; ++j) {
    unsigned long long base[G];
    if (a == 0) {
#pragma unroll
      for (int k = 0; k < G; ++k) base[k] = ring[0][k];
    } else {
      indicator_word<G>(p, h, stride, live, q, j, base);
    }
#pragma unroll
    for (int k = 0; k < G; ++k) {
      if (j == jf) { kept(0, k) = base[k]; pf[k] = pc[k]; }
      if (j == jf + 1) kept(1, k) = base[k];
      if (j == jl) { kept(2, k) = base[k]; pl[k] = pc[k]; }
      if (j == jl + 1) kept(3, k) = base[k];
      const unsigned long long l0 = shift128(ring[0][k], ring[1][k], r), l1 = shift128(ring[1][k], ring[2][k], r);
#pragma unroll 8
      for (int i = 0; i < kIndLags; ++i)
        if (i < n_lags) sink.pair(k, i, (unsigned)popcount64(base[k] & shift128(l0, l1, i)));
      pc[k] += popcount64(base[k]);
      ring[0][k] = ring[1][k];
      ring[1][k] = ring[2][k];
    }
    unsigned long long next[G];
    indicator_word<G>(p, h, stride, live, q, j + a + 3, next);
#pragma unroll
    for (int k = 0; k < G; ++k) ring[2][k] = next[k];
  }
#pragma unroll
  for (int k = 0; k < G; ++k) {
    const long long c = pc[k];
    if (jl >= nw) pl[k] = pc[k];                          // s = h = 64 nw (t = 0): the word past the half, all positions before it
    const unsigned long long wf0 = kept(0, k), wf1 = kept(1, k), wl0 = kept(2, k), wl1 = kept(3, k);
    sink.count(k, c);
#pragma unroll 4
    for (int i = 0; i < kIndLags; ++i)
      if (i < n_lags) {
        const long long t = lag0 + i;
        const long long ft = prefix_count(t, jf, wf0, wf1, pf[k]);
        const long long lt = c - prefix_count(h - t, jl, wl0, wl1, pl[k]);
        sink.edge(k, i, (unsigned long long)(c * (ft + lt)));
      }
  }
}

}  // namespace summary
