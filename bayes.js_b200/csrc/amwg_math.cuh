// amwg_math.cuh -- device-side JS number semantics: Math.log / Math.exp / Math.round / Math.max,
// the Philox4x32-10 "Math.random()" stream and rnorm (mcmc.js:43-54).
//
// This translation unit is compiled with --fmad=false: every *, +, -, / below is one IEEE-754 fp64
// operation, as in a JS engine.  Fused multiply-adds appear only where written as fma() (the
// factorised likelihood plates in amwg_kernels.cu).
#pragma once
#ifdef __CUDACC_RTC__
// run-time compilation (NVRTC, amwg_jit.cuh): no host headers; the few names this file needs from them
typedef unsigned int uint32_t;
typedef unsigned long long uint64_t;
#define CUDART_INF __longlong_as_double(0x7ff0000000000000LL)
#define CUDART_NAN __longlong_as_double(0xfff8000000000000LL)
#else
#include <cstdint>
#include <cuda_runtime.h>
#include <math_constants.h>
#endif

namespace amwg {

// ---- Math.log : the fdlibm e_log algorithm (what V8's ieee754::log implements) -------------------
__device__ __noinline__ double js_log(double x) {
  const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10,
               two54 = 1.80143985094819840000e+16,
               Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
               Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
               Lg7 = 1.479819860511658591e-01;
  int hx = __double2hiint(x);
  unsigned lx = (unsigned)__double2loint(x);
  int k = 0;
  if (hx < 0x00100000) {
    if (((hx & 0x7fffffff) | lx) == 0) return -CUDART_INF;
    if (hx < 0) return CUDART_NAN;
    k -= 54; x *= two54; hx = __double2hiint(x);
  }
  if (hx >= 0x7ff00000) return x + x;
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  int i = (hx + 0x95f64) & 0x100000;
  x = __hiloint2double(hx | (i ^ 0x3ff00000), __double2loint(x));
  k += (i >> 20);
  double f = x - 1.0;
  if ((0x000fffff & (2 + hx)) < 3) {
    if (f == 0.0) { if (k == 0) return 0.0; double dk = (double)k; return dk * ln2_hi + dk * ln2_lo; }
    double R = f * f * (0.5 - 0.33333333333333333 * f);
    if (k == 0) return f - R;
    double dk = (double)k; return dk * ln2_hi - ((R - dk * ln2_lo) - f);
  }
  double s = f / (2.0 + f);
  double dk = (double)k;
  double z = s * s;
  i = hx - 0x6147a;
  double w = z * z;
  int j = 0x6b851 - hx;
  double t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  double t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  i |= j;
  double R = t2 + t1;
  if (i > 0) {
    double hfsq = 0.5 * f * f;
    if (k == 0) return f - (hfsq - s * (hfsq + R));
    return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
  }
  if (k == 0) return f - s * (f - R);
  return dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f);
}

// ---- Math.exp : the fdlibm e_exp algorithm ---------------------------------------------------------
__device__ __noinline__ double js_exp(double x) {
  const double huge = 1.0e+300, twom1000 = 9.33263618503218878990e-302,
               o_threshold = 7.09782712893383973096e+02, u_threshold = -7.45133219101941108420e+02,
               ln2HI = 6.93147180369123816490e-01, ln2LO = 1.90821492927058770002e-10,
               invln2 = 1.44269504088896338700e+00,
               P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
               P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
  double hi = 0.0, lo = 0.0;
  int k = 0;
  unsigned hx = (unsigned)__double2hiint(x);
  int xsb = (int)((hx >> 31) & 1);
  hx &= 0x7fffffff;
  if (hx >= 0x40862E42) {
    if (hx >= 0x7ff00000) {
      if (((hx & 0xfffff) | (unsigned)__double2loint(x)) != 0) return x + x;
      return (xsb == 0) ? x : 0.0;
    }
    if (x > o_threshold) return huge * huge;
    if (x < u_threshold) return twom1000 * twom1000;
  }
  if (hx > 0x3fd62e42) {
    if (hx < 0x3FF0A2B2) {
      hi = x - (xsb ? -ln2HI : ln2HI); lo = xsb ? -ln2LO : ln2LO; k = 1 - xsb - xsb;
    } else {
      k = (int)(invln2 * x + (xsb ? -0.5 : 0.5));
      double t = (double)k;
      hi = x - t * ln2HI;
      lo = t * ln2LO;
    }
    x = hi - lo;
  } else if (hx < 0x3e300000) {
    if (huge + x > 1.0) return 1.0 + x;
  }
  double t = x * x;
  double c = x - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  if (k == 0) return 1.0 - ((x * c) / (c - 2.0) - x);
  double y = 1.0 - ((lo - (x * c) / (2.0 - c)) - hi);
  if (k >= -1021) {
    if (k == 1024) return y * 2.0 * 8.98846567431157953865e+307;
    return __hiloint2double(__double2hiint(y) + (k << 20), __double2loint(y));
  }
  y = __hiloint2double(__double2hiint(y) + ((k + 1000) << 20), __double2loint(y));
  return y * twom1000;
}

// Math.pow: pow(d, 2) == d*d on the in-scope path (distributions.js:120); general case defers to CUDA pow.
__device__ __forceinline__ double js_pow(double x, double y) { return (y == 2.0) ? x * x : pow(x, y); }

// Math.round: halves toward +inf (mcmc.js:597).  V8 Float64Round: ceil, step down if it overshoots by > 0.5.
__device__ __forceinline__ double js_round(double x) {
  double r = ceil(x);
  if (r - 0.5 > x) r -= 1.0;
  return r;
}
// Math.max / Math.min: NaN-propagating (mcmc.js:758, :541)
__device__ __forceinline__ double js_max(double a, double b) { if (a != a || b != b) return CUDART_NAN; return a > b ? a : b; }
__device__ __forceinline__ double js_min(double a, double b) { if (a != a || b != b) return CUDART_NAN; return a < b ? a : b; }

// ---- Math.random() := Philox4x32-10 stream (DESIGN.md "RNG contract") -------------------------------
// call #n of chain g: block = n>>1; counter = (blk_lo, blk_hi, g_lo, g_hi); key = (seed_lo, seed_hi);
// words (r0..r3): n even -> (r0,r1), n odd -> (r2,r3);  u = ((a>>5)*2^26 + (b>>6)) * 2^-53.
struct Philox4 { uint32_t r0, r1, r2, r3; };

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}

// (double)v for a 32-bit v without an integer-to-double conversion (a quarter-rate instruction on sm_90): the double whose high
// word is 0x43300000 and whose low word is v is 2^52 + v, and subtracting 2^52 leaves v. Both steps are exact.
__device__ __forceinline__ double u32_to_double(uint32_t v) {
  return __hiloint2double(0x43300000, (int)v) - 4503599627370496.0;
}

__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  return (u32_to_double(a >> 5) * 67108864.0 + u32_to_double(b >> 6)) * (1.0 / 9007199254740992.0);
}

// one Philox block = uniforms #2*blk and #2*blk+1 of chain (g0,g1). Kept out of line by default: it is ~80 instructions and
// is needed at several points of a sweep; inlining it everywhere bloats the kernel past the instruction cache. The specialised
// statistics sweep defines AMWG_PHILOX_INLINE (amwg_jit.cuh): its step code is short, and there the call's overhead is the
// larger cost (config 2: 6 % less per-sweep O(1) time on an H100, DESIGN.md section 4.1).
#ifndef AMWG_PHILOX_INLINE
#define AMWG_PHILOX_INLINE 0
#endif
#if AMWG_PHILOX_INLINE
__device__ __forceinline__
#else
__device__ __noinline__
#endif
double2 philox_uniform_pair(uint32_t blk_lo, uint32_t blk_hi, uint32_t g0, uint32_t g1, uint32_t k0, uint32_t k1) {
  Philox4 p = philox4x32_10(blk_lo, blk_hi, g0, g1, k0, k1);
  return make_double2(u53(p.r0, p.r1), u53(p.r2, p.r3));
}

// The chain's position in its Math.random() stream plus the Philox block that contains it.  Lanes of a warp sit at
// different positions (rnorm consumes a data-dependent number of uniforms), so the block is fetched at ONE call site per
// draw with a per-lane block index: divergence in stream position never multiplies the Philox work.
struct RandomStream {
  // The key (seed) and the chain id are not stored: they live in the kernel's parameters / the thread's chain index, and
  // every register kept alive across the log_post evaluation is one more spill at the sweep kernel's register cap.
  uint64_t n;          // index of the next Math.random() call of this chain
  uint64_t cb;         // index of the cached block (uniforms #2*cb, #2*cb+1), ~0 if none
  double c0, c1;

  __device__ __forceinline__ void init(uint64_t pos) { n = pos; cb = ~0ull; c0 = c1 = 0.0; }
  __device__ __forceinline__ void load(uint64_t seed, uint64_t chain, uint64_t blk) {
    double2 p = philox_uniform_pair((uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)chain, (uint32_t)(chain >> 32), (uint32_t)seed, (uint32_t)(seed >> 32));
    cb = blk; c0 = p.x; c1 = p.y;
  }
  // one uniform
  __device__ __forceinline__ double next(uint64_t seed, uint64_t chain) {
    uint64_t blk = n >> 1;
    if (cb != blk) load(seed, chain, blk);
    double u = (n & 1) ? c1 : c0;
    ++n;
    return u;
  }
  // two consecutive uniforms (#n, #n+1) with exactly one block fetch: for odd n the first one is the cached block's
  // second word and the new block provides the second one.
  __device__ __forceinline__ void next2(uint64_t seed, uint64_t chain, double& u, double& v) {
    if ((n & 1) && cb != (n >> 1)) load(seed, chain, n >> 1);          // only right after a kernel (re)start
    double first_odd = c1;
    uint64_t blk = (n + 1) >> 1;                          // even n: the block of n; odd n: the next block
    bool odd = (n & 1);
    load(seed, chain, blk);
    u = odd ? first_odd : c0;
    v = odd ? c0 : c1;
    n += 2;
  }
};

// rnorm -- mcmc.js:43-54 (Leva ratio-of-uniforms; two uniforms per trial). js_rnorm_ratio is the accepted v / u: the draw is
// (v / u) * sd + mean, and a caller that does not have sd and mean at hand yet can finish it later with the same two operations.
__device__ __forceinline__ double js_rnorm_ratio(RandomStream& g, uint64_t seed, uint64_t chain) {
  double u, v, x, y, q;
  do {
    double r;
    g.next2(seed, chain, u, r);
    v = 1.7156 * (r - 0.5);
    x = u - 0.449871;
    y = fabs(v) + 0.386595;
    q = x * x + y * (0.19600 * y - 0.25472 * x);
  } while (q > 0.27597 && (q > 0.27846 || v * v > -4 * js_log(u) * u * u));
  return v / u;
}
__device__ __forceinline__ double js_rnorm(RandomStream& g, uint64_t seed, uint64_t chain, double mean, double sd) {
  return js_rnorm_ratio(g, seed, chain) * sd + mean;
}

}  // namespace amwg
