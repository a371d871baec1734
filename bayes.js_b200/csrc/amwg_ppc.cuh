// amwg_ppc.cuh -- replicated data for the posterior predictive checks of sample_summary(..., ppc=...) (DESIGN.md §4.8): one sampler
// per ld.* family, drawn from the chain's own Math.random() stream at a position reserved for (kept row, point).
//
// Stream. y_rep of point i at kept row r (of this call) of global chain g takes the uniforms #(2^62 + (r N + i) 2^16 + k), k = 0, 1, ...,
// of chain g's Philox stream (DESIGN.md §2). The region lies below the dispersal region (>= 2^63) and far above any position
// sampling reaches; it is keyed by the global chain, so the draws do not depend on how the chains are sharded. A draw that would
// need k >= 2^16 gives NaN (no sampler below comes near that). Repeated calls reuse these uniforms for new posterior draws.
//
// Arithmetic. Only + - * /, sqrt, floor, comparisons, js_log, js_exp and js_rnorm (mcmc.js's Leva rnorm), each one IEEE-754
// operation (the library is built with --fmad=false, the host shim with -ffp-contract=off), so the host-compiled header and a
// Python restatement give the device's bits. pow and tan are not used: CUDA's and libm's differ in the last bits.
//
// Domains (anything else, or a non-finite parameter, gives NaN without consuming a uniform):
//   norm(mean, sd), lnorm(meanlog, sdlog)       sd > 0          Z sd + mean; lnorm: js_exp of it
//   cauchy(location, scale)                      scale > 0       location + scale Z1 / Z2
//   laplace = dexp(location, scale)              scale > 0       location + scale (E1 - E2), E = -js_log(1 - U)
//   logis(location, scale)                       scale > 0       location + scale (js_log(U) - js_log(1 - U)), U = 0 redrawn
//   exp(rate)                                    rate > 0        E / rate
//   weibull(shape, scale)                        both > 0        scale js_exp(js_log(E) / shape)
//   pareto(scale, shape)                         both > 0        scale js_exp(E / shape)
//   unif(min, max)                               min < max       min + (max - min) U
//   gamma(shape, rate)                           both > 0        G(shape) / rate: Marsaglia & Tsang (2000) without the squeeze (Z,
//                                                                then U); shape < 1: G(shape + 1) js_exp(js_log(U) / shape)
//   invgamma(shape, scale)                       both > 0        scale / G(shape)
//   beta(a, b)                                   both > 0        X / (X + Y), X = G(a) drawn first, Y = G(b)
//   t(location, scale, df)                       scale, df > 0   location + scale Z / sqrt(2 G(df / 2) / df), Z first
//   bern(prob)                                   0 <= prob <= 1  U < prob ? 1 : 0
//   pois(lambda)                                 lambda >= 0     lambda < 10: multiplication against js_exp(-lambda); else PTRS
//                                                                (Hoermann 1993)
//   binom(size, prob)                            integer size >= 0, 0 <= prob <= 1: on q = min(prob, 1 - prob), inversion by
//                                                                sequential search when size q < 10, else BTRS (Hoermann 1993);
//                                                                size - x when prob > 1/2
//   nbinom(size, prob)                           size > 0, 0 < prob <= 1: pois(G(size) / (prob / (1 - prob))), the failures before
//                                                                the size-th success as ld.nbinom counts them
// Z: js_rnorm_ratio (one standard normal); U: one uniform; G(a): a Gamma(a, 1) draw as above.
#pragma once

#include "amwg_math.cuh"

namespace ppc {

using amwg::js_exp;
using amwg::js_log;

// family codes of amwg_ppc_pointwise (include/amwg.h); summary.PPC_FAMILIES lists the ld names in this order
enum Family : int { kNorm = 0, kLnorm, kCauchy, kLaplace, kLogis, kExp, kWeibull, kPareto, kUnif, kGamma, kInvgamma, kBeta, kT, kBern,
                    kPois, kBinom, kNbinom, kFamilies };

__host__ __device__ inline int arity(int fam) {
  switch (fam) {
    case kExp: case kBern: case kPois: return 1;
    case kT: return 3;
    default: return 2;
  }
}

constexpr uint64_t kStreamBase = 1ull << 62;
constexpr int kPointShift = 16;                // 2^16 uniforms per (kept row, point)

__host__ __device__ inline uint64_t stream_position(uint64_t row, uint64_t points, uint64_t i) {
  return kStreamBase + ((row * points + i) << kPointShift);
}

// the uniforms of one (kept row, point, chain): chain g's Math.random() stream from stream_position on
struct PhiloxSource {
  amwg::RandomStream g;
  uint64_t seed, chain, end;
  __device__ void init(uint64_t s, uint64_t c, uint64_t pos) { g.init(pos); seed = s; chain = c; end = pos + (1ull << kPointShift); }
  __device__ double u() { return g.next(seed, chain); }
  __device__ double z() { return amwg::js_rnorm_ratio(g, seed, chain); }
  __device__ bool spent() const { return g.n > end; }     // a uniform #k >= 2^16 was taken
};

// log k! for an integer k >= 0: correctly rounded below 128, Stirling's series (three terms, error < 1e-18 relative) above.
// (ld_lgamma's 6-term Lanczos is about 1e-10 off, which would bias the acceptance tests of PTRS and BTRS.)
__device__ const double kLogFactorial[128] = {
    0.0, 0.0, 0.6931471805599453, 1.791759469228055,
    3.1780538303479458, 4.787491742782046, 6.579251212010101, 8.525161361065415,
    10.60460290274525, 12.801827480081469, 15.104412573075516, 17.502307845873887,
    19.987214495661885, 22.552163853123425, 25.19122118273868, 27.89927138384089,
    30.671860106080672, 33.50507345013689, 36.39544520803305, 39.339884187199495,
    42.335616460753485, 45.38013889847691, 48.47118135183523, 51.60667556776438,
    54.78472939811232, 58.00360522298052, 61.261701761002, 64.55753862700634,
    67.88974313718154, 71.25703896716801, 74.65823634883016, 78.0922235533153,
    81.55795945611504, 85.05446701758152, 88.58082754219768, 92.1361756036871,
    95.7196945421432, 99.33061245478743, 102.96819861451381, 106.63176026064346,
    110.32063971475739, 114.0342117814617, 117.77188139974507, 121.53308151543864,
    125.3172711493569, 129.12393363912722, 132.95257503561632, 136.80272263732635,
    140.67392364823425, 144.5657439463449, 148.47776695177302, 152.40959258449735,
    156.3608363030788, 160.3311282166309, 164.32011226319517, 168.32744544842765,
    172.3527971391628, 176.39584840699735, 180.45629141754378, 184.53382886144948,
    188.6281734236716, 192.7390472878449, 196.86618167289, 201.00931639928152,
    205.1681994826412, 209.34258675253685, 213.53224149456327, 217.73693411395422,
    221.95644181913033, 226.1905483237276, 230.43904356577696, 234.70172344281826,
    238.97838956183432, 243.2688490029827, 247.57291409618688, 251.8904022097232,
    256.22113555000954, 260.5649409718632, 264.9216497985528, 269.2910976510198,
    273.6731242856937, 278.0675734403661, 282.4742926876304, 286.893133295427,
    291.3239500942703, 295.76660135076065, 300.22094864701415, 304.6868567656687,
    309.1641935801469, 313.65282994987905, 318.1526396202093, 322.66349912672615,
    327.1852877037752, 331.7178871969285, 336.26118197919845, 340.815058870799,
    345.37940706226686, 349.95411804077025, 354.5390855194408, 359.1342053695754,
    363.73937555556347, 368.35449607240474, 372.979468885689, 377.61419787391867,
    382.25858877306, 386.91254912321756, 391.5759882173296, 396.24881705179155,
    400.93094827891576, 405.6222961611449, 410.32277652693733, 415.03230672824964,
    419.7508055995447, 424.4781934182571, 429.21439186665157, 433.9593239950148,
    438.71291418612117, 443.47508812091894, 448.2457727453846, 453.0248962384961,
    457.81238798127816, 462.6081785268749, 467.4121995716082, 472.2243839269806,
    477.04466549258564, 481.87297922988796, 486.7092611368394, 491.553448223298,
};

__device__ inline double log_factorial(double k) {
  if (k < 128.0) return kLogFactorial[(int)k];
  const double r = 1.0 / k, r2 = r * r;
  return (k + 0.5) * js_log(k) - k + 0.91893853320467274178 + r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0)));
}

template <class S> __device__ inline double expo(S& s) { return -js_log(1.0 - s.u()); }

// Marsaglia & Tsang (2000), a >= 1, without the squeeze
template <class S> __device__ double gamma_mt(S& s, double a) {
  const double d = a - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
  while (!s.spent()) {
    double x, v;
    do { x = s.z(); v = 1.0 + c * x; } while (v <= 0.0 && !s.spent());
    v = v * v * v;
    const double U = s.u();
    if (js_log(U) < 0.5 * x * x + d - d * v + d * js_log(v)) return d * v;
  }
  return CUDART_NAN;
}

// G(a): Gamma(a, 1), a > 0
template <class S> __device__ double gamma1(S& s, double a) {
  if (a >= 1.0) return gamma_mt(s, a);
  const double g = gamma_mt(s, a + 1.0);
  return g * js_exp(js_log(s.u()) / a);
}

template <class S> __device__ double pois(S& s, double lam) {
  if (lam < 10.0) {                                          // multiplication method
    const double L = js_exp(-lam);
    double p = 1.0, k = -1.0;
    do { k += 1.0; p = p * s.u(); } while (p > L && !s.spent());
    return k;
  }
  // PTRS, Hoermann (1993), "The transformed rejection method for generating Poisson random variables"
  const double slam = sqrt(lam), loglam = js_log(lam), b = 0.931 + 2.53 * slam, a = -0.059 + 0.02483 * b,
               lia = js_log(1.1239 + 1.1328 / (b - 3.4)), vr = 0.9277 - 3.6224 / (b - 2.0);
  while (!s.spent()) {
    const double U = s.u() - 0.5, V = s.u(), us = 0.5 - fabs(U);
    const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
    if (k < 0.0) continue;
    if (us >= 0.07 && V <= vr) return k;
    if (us < 0.013 && V > us) continue;
    if (js_log(V) + lia - js_log(a / (us * us) + b) <= -lam + k * loglam - log_factorial(k)) return k;
  }
  return CUDART_NAN;
}

// binomial on q <= 1/2
template <class S> __device__ double binom_low(S& s, double n, double q) {
  if (n * q < 10.0) {                                        // inversion by sequential search from 0
    const double qn = js_exp(n * js_log(1.0 - q)), r = q / (1.0 - q), g = r * (n + 1.0);
    while (!s.spent()) {
      double U = s.u(), f = qn, k = 0.0;
      for (;;) {
        if (U < f) return k;
        if (k >= n) break;                                   // rounding left U above the total mass: draw again
        U = U - f;
        k += 1.0;
        f = f * (g / k - r);
      }
    }
    return CUDART_NAN;
  }
  // BTRS, Hoermann (1993), "The generation of binomial random variates"
  const double spq = sqrt(n * q * (1.0 - q)), b = 1.15 + 2.53 * spq, a = -0.0873 + 0.0248 * b + 0.01 * q, c = n * q + 0.5,
               vr = 0.92 - 4.2 / b, alpha = (2.83 + 5.1 / b) * spq, lpq = js_log(q / (1.0 - q)), m = floor((n + 1.0) * q),
               h = log_factorial(m) + log_factorial(n - m);
  while (!s.spent()) {
    const double U = s.u() - 0.5, V = s.u(), us = 0.5 - fabs(U);
    const double k = floor((2.0 * a / us + b) * U + c);
    if (k < 0.0 || k > n) continue;
    if (us >= 0.07 && V <= vr) return k;
    if (js_log(V * alpha / (a / (us * us) + b)) <= h - log_factorial(k) - log_factorial(n - k) + (k - m) * lpq) return k;
  }
  return CUDART_NAN;
}

__host__ __device__ inline bool finite(double x) { return x - x == 0.0; }

// one replicated observation of family `fam` with parameters a[0 .. arity(fam) - 1]; NaN outside the domain
template <class S> __device__ double draw(int fam, const double* a, S& s) {
  const int n = arity(fam);
  for (int k = 0; k < n; ++k)
    if (!finite(a[k])) return CUDART_NAN;
  const double a0 = a[0], a1 = n > 1 ? a[1] : 0.0, a2 = n > 2 ? a[2] : 0.0;
  double x;
  switch (fam) {
    case kNorm: case kLnorm:
      if (!(a1 > 0.0)) return CUDART_NAN;
      x = s.z() * a1 + a0;
      if (fam == kLnorm) x = js_exp(x);
      break;
    case kCauchy: {
      if (!(a1 > 0.0)) return CUDART_NAN;
      const double z1 = s.z(), z2 = s.z();
      x = a0 + a1 * z1 / z2;
      break;
    }
    case kLaplace: {
      if (!(a1 > 0.0)) return CUDART_NAN;
      const double e1 = expo(s), e2 = expo(s);
      x = a0 + a1 * (e1 - e2);
      break;
    }
    case kLogis: {
      if (!(a1 > 0.0)) return CUDART_NAN;
      double U;
      do { U = s.u(); } while (U == 0.0 && !s.spent());
      x = a0 + a1 * (js_log(U) - js_log(1.0 - U));
      break;
    }
    case kExp:
      if (!(a0 > 0.0)) return CUDART_NAN;
      x = expo(s) / a0;
      break;
    case kWeibull:
      if (!(a0 > 0.0 && a1 > 0.0)) return CUDART_NAN;
      x = a1 * js_exp(js_log(expo(s)) / a0);
      break;
    case kPareto:
      if (!(a0 > 0.0 && a1 > 0.0)) return CUDART_NAN;
      x = a0 * js_exp(expo(s) / a1);
      break;
    case kUnif:
      if (!(a0 < a1)) return CUDART_NAN;
      x = a0 + (a1 - a0) * s.u();
      break;
    case kGamma:
      if (!(a0 > 0.0 && a1 > 0.0)) return CUDART_NAN;
      x = gamma1(s, a0) / a1;
      break;
    case kInvgamma:
      if (!(a0 > 0.0 && a1 > 0.0)) return CUDART_NAN;
      x = a1 / gamma1(s, a0);
      break;
    case kBeta: {
      if (!(a0 > 0.0 && a1 > 0.0)) return CUDART_NAN;
      const double X = gamma1(s, a0), Y = gamma1(s, a1);
      x = X / (X + Y);
      break;
    }
    case kT: {
      if (!(a1 > 0.0 && a2 > 0.0)) return CUDART_NAN;
      const double z = s.z(), g = gamma1(s, a2 / 2.0);
      x = a0 + a1 * z / sqrt(2.0 * g / a2);
      break;
    }
    case kBern:
      if (!(a0 >= 0.0 && a0 <= 1.0)) return CUDART_NAN;
      x = s.u() < a0 ? 1.0 : 0.0;
      break;
    case kPois:
      if (!(a0 >= 0.0)) return CUDART_NAN;
      x = pois(s, a0);
      break;
    case kBinom: {
      if (!(a0 >= 0.0 && a0 == floor(a0) && a1 >= 0.0 && a1 <= 1.0)) return CUDART_NAN;
      const bool flip = a1 > 0.5;
      const double k = binom_low(s, a0, flip ? 1.0 - a1 : a1);
      x = flip ? a0 - k : k;
      break;
    }
    case kNbinom: {
      if (!(a0 > 0.0 && a1 > 0.0 && a1 <= 1.0)) return CUDART_NAN;
      const double lam = gamma1(s, a0) / (a1 / (1.0 - a1));
      x = pois(s, lam);
      break;
    }
    default: return CUDART_NAN;
  }
  return s.spent() ? CUDART_NAN : x;
}

}  // namespace ppc
