// The per-half-chain walk of amwg_autocov_kernel (amwg_summary.cuh, K_a1): one __host__ __device__ text, so that the kernel and the
// host build the CPU tests run (tests/host_shim/autocov_host.cpp) centre, scale and accumulate alike.
//
// Per half-chain m of h draws and series y (the draws, or an indicator 1[x <= q] of them), centred by the half-chain's own mean:
//   record  {1, mean_m, 0, sum_n d_n^2}                 merged like Moments (Chan, fixed order)
//   lag sum sum_n d_n d_{n+t} = h * acov_m(t)           for t in the lag window [lag0, lag0 + kLagSlots)
// For the draws series of NS = 3 (the thresholds q05, q95 given) the centred values d and the mean are multiplied by
// autocov_scale(q05, q95), a power of two: exact while the scaled values stay normal, so the ESS and split R-hat formed from the
// records (ratios of these sums) do not depend on the scale of the draws, and draws far from 1 in magnitude neither underflow nor
// overflow their squares. The scale leaves about 2^511 between the q05..q95 spread and the largest |x - mean|: outliers further out
// overflow once scaled (the host then gives NaN).
#pragma once

#include "amwg_nested.cuh"      // Moments, merge, run_bits, run_mean

namespace summary {

constexpr int kLagSlots = 16;         // lags per kernel pass: the ring of centred lead values a thread keeps in registers

// 2^k with k = -ilogb(q95/2 - q05/2), clamped to [-1022, 1023] so that 2^k is a normal double: the spread between the thresholds
// is brought into [1, 2). 1 when that spread is 0 (q05 == q95: at least 90 % of the draws share one value), infinite or NaN.
// q95/2 - q05/2 cannot overflow, and halving is exact for every normal threshold.
__host__ __device__ __forceinline__ double autocov_scale(double q05, double q95) {
  const double s = q95 * 0.5 - q05 * 0.5;
  if (!(s > 0.0 && s <= 1.7976931348623157e308)) return 1.0;
  int k = -ilogb(s);
  k = k < -1022 ? -1022 : k > 1023 ? 1023 : k;
  return ldexp(1.0, k);
}

struct SeriesIdentity {
  __host__ __device__ __forceinline__ double operator()(double v) const { return v; }
};

// y = ((x - centre) * scale)^2: the squared deviations whose ESS gives mcse_sd. scale is a power of two (the host takes it from the
// pooled sd), so y is exactly scale^2 times the unscaled square while that stays normal.
struct SquaredDeviation {
  double centre, scale;
  __host__ __device__ __forceinline__ double operator()(double v) const {
    const double d = (v - centre) * scale;
    return d * d;
  }
};

// One half-chain p[n * stride], n < h, of a thread's chain: adds its lag sums for the lags lag0 + k, k < kLagSlots, to acc and
// merges its record into mom. Pass 1 reads the half for its means; pass 2 reads it again and keeps the kLagSlots centred values at
// positions n+lag0 .. n+lag0+15 in a register ring, so every loaded value serves all lags of the window. NS = 1: the draws only;
// NS = 3: also 1[x <= q0] and 1[x <= q1], formed from the same loads (the ring holds their bits), and the draws scaled by sc.
// Positions at or past h count as 0, so a product exists exactly when both ends lie in the half. tf maps every value read to the
// series walked (SeriesIdentity: the draws; SquaredDeviation: y = ((x - centre) * scale)^2 of amwg_summary_autocov_sq).
template <int NS, class Tf = SeriesIdentity>
__host__ __device__ __forceinline__ void autocov_half(const double* __restrict__ p, long long h, size_t stride, double q0, double q1, double sc,
                                                      long long lag0, double (&acc)[NS][kLagSlots], Moments (&mom)[NS], Tf tf = Tf()) {
  const double x0 = tf(p[0]);
  const unsigned long long x0_bits = run_bits(x0);
  unsigned long long diff = 0;
  double s0 = 0.0;
  long long n0 = 0, n1 = 0;
  long long r = 0;
  for (; r + 8 <= h; r += 8) {                           // eight loads in flight per thread, the sum stays sequential
    double v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = tf(p[(r + u) * stride]);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      s0 += v[u];
      diff |= run_bits(v[u]) ^ x0_bits;
      if constexpr (NS == 3) { n0 += v[u] <= q0; n1 += v[u] <= q1; }
    }
  }
  for (; r < h; ++r) {
    const double v = tf(p[r * stride]);
    s0 += v;
    diff |= run_bits(v) ^ x0_bits;
    if constexpr (NS == 3) { n0 += v <= q0; n1 += v <= q1; }
  }
  double m[NS];
  m[0] = run_mean(s0, h, x0, diff);                      // a constant half-chain is centred on its value (amwg_nested.cuh)
  if constexpr (NS == 3) { m[1] = (double)n0 / (double)h; m[2] = (double)n1 / (double)h; }
  // the draws' centred value, scaled (NS = 3)
  auto centred = [&](double v) { if constexpr (NS == 3) return (v - m[0]) * sc; else return v - m[0]; };

  double ring[kLagSlots];
  unsigned valid = 0u, b0 = 0u, b1 = 0u;                  // bit k: slot k lies in the half / its draw is <= q0 / <= q1
#pragma unroll
  for (int k = 0; k < kLagSlots; ++k) {
    const long long pp = lag0 + k;
    ring[k] = 0.0;
    if (pp < h) {
      const double v = tf(p[pp * stride]);
      ring[k] = centred(v);
      valid |= 1u << k;
      if constexpr (NS == 3) { b0 |= (unsigned)(v <= q0) << k; b1 |= (unsigned)(v <= q1) << k; }
    }
  }
  double sw[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) sw[s] = 0.0;
  for (long long j = 0; j < h; j += kLagSlots) {
#pragma unroll
    for (int u = 0; u < kLagSlots; ++u) {                 // unrolled: the ring's slot indices are compile-time constants
      const long long n = j + u;
      if (n < h) {
        const double v = tf(p[n * stride]);
        double cur[NS];
        cur[0] = centred(v);
        if constexpr (NS == 3) { cur[1] = v <= q0 ? 1.0 - m[1] : -m[1]; cur[2] = v <= q1 ? 1.0 - m[2] : -m[2]; }
#pragma unroll
        for (int s = 0; s < NS; ++s) sw[s] = fma(cur[s], cur[s], sw[s]);
#pragma unroll
        for (int k = 0; k < kLagSlots; ++k) {
          const int slot = (u + k) % kLagSlots;         // holds position n + lag0 + k
          acc[0][k] = fma(cur[0], ring[slot], acc[0][k]);
          if constexpr (NS == 3) {
            const bool in = (valid >> slot) & 1u;
            const double a0 = in ? (((b0 >> slot) & 1u) ? 1.0 - m[1] : -m[1]) : 0.0;
            const double a1 = in ? (((b1 >> slot) & 1u) ? 1.0 - m[2] : -m[2]) : 0.0;
            acc[1][k] = fma(cur[1], a0, acc[1][k]);
            acc[2][k] = fma(cur[2], a1, acc[2][k]);
          }
        }
        const long long pp = n + lag0 + kLagSlots;        // slot u moves on to position n + lag0 + kLagSlots
        const unsigned bit = 1u << u;
        ring[u] = 0.0;
        valid &= ~bit; b0 &= ~bit; b1 &= ~bit;
        if (pp < h) {
          const double w = tf(p[pp * stride]);
          ring[u] = centred(w);
          valid |= bit;
          if constexpr (NS == 3) { if (w <= q0) b0 |= bit; if (w <= q1) b1 |= bit; }
        }
      }
    }
  }
  if constexpr (NS == 3) m[0] *= sc;                    // the record's mean in the units of its centred values
#pragma unroll
  for (int s = 0; s < NS; ++s) mom[s] = merge(mom[s], Moments{1.0, m[s], 0.0, sw[s]});
}

}  // namespace summary
