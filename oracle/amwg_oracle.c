/*
 * amwg_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C, fp64) of the one hot path of rasmusab/bayes.js:
 *   mcmc.AmwgSampler(params, log_post, data).burn()/sample()  +  the ld.* log densities.
 * It is the parity checker for the CUDA path. Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this file's shared object.
 * The product (bayes.js_b200/) never includes, links or calls anything in oracle/.
 *
 * Pinning status (see DESIGN.md "Oracle"):
 *   - pinned DRAW FOR DRAW against the UNMODIFIED /root/reference/mcmc.js + distributions.js + tests/test_data.js, executed
 *     by oracle/minijs (an ES5 interpreter written for this purpose, because no JS engine exists in the image) with
 *     Math.random replaced by the Philox stream below: 32 sampler scenarios covering every stepper kind, options, thin,
 *     monitor and adaptation toggles, plus every ld.* function, complete_params, param_init_fixed and the helpers.
 *     Vectors: tests/golden/reference_js.json; generator: oracle/minijs/make_golden.py; check: tests/test_golden.py;
 *   - pinned against the reference's only deterministic fixtures (complete_params goldens, tests/test_data.js:20-35,50-74)
 *     and the closed-form known answers of SURVEY.md 8(c) (tests/test_oracle.py);
 *   - exact equality with V8's own Math.log/Math.exp/Math.pow is "parity unpinned": V8 is not runnable here;
 *     orc_log/orc_exp restate the fdlibm algorithms V8's ieee754::log/exp are ports of (<= 1 ulp from glibc, checked).
 *
 * Every function cites the reference lines it follows (paths under /root/reference/).
 * Build: oracle/Makefile  (gcc -O2 -ffp-contract=off -fno-fast-math).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * Math.log / Math.exp : fdlibm e_log.c / e_exp.c algorithms (Sun Microsystems, 1993), which
 * V8's base/ieee754.cc ports. Written with explicit word access; no FMA contraction.
 * ---------------------------------------------------------------------------------------- */
static inline uint32_t hi_word(double x) { uint64_t u; memcpy(&u, &x, 8); return (uint32_t)(u >> 32); }
static inline uint32_t lo_word(double x) { uint64_t u; memcpy(&u, &x, 8); return (uint32_t)u; }
static inline double set_hi(double x, uint32_t hi) {
  uint64_t u; memcpy(&u, &x, 8); u = ((uint64_t)hi << 32) | (u & 0xffffffffu); memcpy(&x, &u, 8); return x;
}

ORC_API double orc_log(double x) {
  static const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10,
                      two54 = 1.80143985094819840000e+16,
                      Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01,
                      Lg3 = 2.857142874366239149e-01, Lg4 = 2.222219843214978396e-01,
                      Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
                      Lg7 = 1.479819860511658591e-01;
  double hfsq, f, s, z, R, w, t1, t2, dk;
  int32_t k, hx, i, j;
  uint32_t lx;
  hx = (int32_t)hi_word(x); lx = lo_word(x);
  k = 0;
  if (hx < 0x00100000) {                       /* x < 2**-1022 */
    if (((hx & 0x7fffffff) | lx) == 0) return -INFINITY;   /* log(+-0) = -inf */
    if (hx < 0) return NAN;                    /* log(-#) = NaN */
    k -= 54; x *= two54; hx = (int32_t)hi_word(x);
  }
  if (hx >= 0x7ff00000) return x + x;
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  i = (hx + 0x95f64) & 0x100000;
  x = set_hi(x, (uint32_t)(hx | (i ^ 0x3ff00000)));   /* normalize x or x/2 */
  k += (i >> 20);
  f = x - 1.0;
  if ((0x000fffff & (2 + hx)) < 3) {           /* |f| < 2**-20 */
    if (f == 0.0) { if (k == 0) return 0.0; dk = (double)k; return dk * ln2_hi + dk * ln2_lo; }
    R = f * f * (0.5 - 0.33333333333333333 * f);
    if (k == 0) return f - R;
    dk = (double)k; return dk * ln2_hi - ((R - dk * ln2_lo) - f);
  }
  s = f / (2.0 + f);
  dk = (double)k;
  z = s * s;
  i = hx - 0x6147a;
  w = z * z;
  j = 0x6b851 - hx;
  t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  i |= j;
  R = t2 + t1;
  if (i > 0) {
    hfsq = 0.5 * f * f;
    if (k == 0) return f - (hfsq - s * (hfsq + R));
    return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
  } else {
    if (k == 0) return f - s * (f - R);
    return dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f);
  }
}

ORC_API double orc_exp(double x) {
  static const double one = 1.0, halF[2] = {0.5, -0.5}, huge = 1.0e+300,
                      twom1000 = 9.33263618503218878990e-302,
                      o_threshold = 7.09782712893383973096e+02, u_threshold = -7.45133219101941108420e+02,
                      ln2HI[2] = {6.93147180369123816490e-01, -6.93147180369123816490e-01},
                      ln2LO[2] = {1.90821492927058770002e-10, -1.90821492927058770002e-10},
                      invln2 = 1.44269504088896338700e+00,
                      P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03,
                      P3 = 6.61375632143793436117e-05, P4 = -1.65339022054652515390e-06,
                      P5 = 4.13813679705723846039e-08;
  double y, hi = 0.0, lo = 0.0, c, t;
  int32_t k = 0, xsb;
  uint32_t hx;
  hx = hi_word(x);
  xsb = (int32_t)((hx >> 31) & 1);
  hx &= 0x7fffffff;
  if (hx >= 0x40862E42) {                      /* |x| >= 709.78... */
    if (hx >= 0x7ff00000) {
      if (((hx & 0xfffff) | lo_word(x)) != 0) return x + x;     /* NaN */
      return (xsb == 0) ? x : 0.0;             /* exp(+-inf) = {inf,0} */
    }
    if (x > o_threshold) return huge * huge;   /* overflow */
    if (x < u_threshold) return twom1000 * twom1000; /* underflow */
  }
  if (hx > 0x3fd62e42) {                       /* |x| > 0.5 ln2 */
    if (hx < 0x3FF0A2B2) {                     /* and |x| < 1.5 ln2 */
      hi = x - ln2HI[xsb]; lo = ln2LO[xsb]; k = 1 - xsb - xsb;
    } else {
      k = (int32_t)(invln2 * x + halF[xsb]);
      t = k;
      hi = x - t * ln2HI[0];
      lo = t * ln2LO[0];
    }
    x = hi - lo;
  } else if (hx < 0x3e300000) {                /* |x| < 2**-28 */
    if (huge + x > one) return one + x;
  } else {
    k = 0;
  }
  t = x * x;
  c = x - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  if (k == 0) return one - ((x * c) / (c - 2.0) - x);
  y = one - ((lo - (x * c) / (2.0 - c)) - hi);
  if (k >= -1021) {
    if (k == 1024) return y * 2.0 * 8.98846567431157953865e+307;  /* 2^1023 */
    return set_hi(y, hi_word(y) + ((uint32_t)k << 20));
  }
  y = set_hi(y, hi_word(y) + ((uint32_t)(k + 1000) << 20));
  return y * twom1000;
}

/* Math.pow: only pow(d,2) occurs on the in-scope ld.* (ld.norm, distributions.js:120), and
 * that is d*d exactly-rounded in every engine's fast path; general pow defers to libm. */
static inline double js_pow(double x, double y) { return (y == 2.0) ? x * x : pow(x, y); }

/* Math.round (V8 Float64Round): ceil, then step down if the ceiling overshoots by > 0.5.
 * Rounds halves toward +inf: round(-2.5) == -2, round(2.5) == 3.  (mcmc.js:597, :335) */
ORC_API double orc_js_round(double x) {
  double r = ceil(x);
  if (r - 0.5 > x) r -= 1.0;
  return r;
}
/* Math.max semantics: NaN if either is NaN (C fmax would drop the NaN). (mcmc.js:758) */
static inline double js_max(double a, double b) { if (a != a || b != b) return NAN; return a > b ? a : b; }
static inline double js_min(double a, double b) { if (a != a || b != b) return NAN; return a < b ? a : b; }

/* ------------------------------------------------------------------------------------------
 * Matched counter RNG ("Math.random() := Philox stream"), DESIGN.md "RNG contract".
 *   n  = index of this Math.random() call in the chain's own history (0-based)
 *   Philox4x32-10( counter = (blk_lo, blk_hi, chain_lo, chain_hi), key = (seed_lo, seed_hi) ), blk = n>>1
 *   words (r0,r1,r2,r3); call n uses (r0,r1) if n even else (r2,r3):
 *   u = ((a>>5) * 2^26 + (b>>6)) * 2^-53   in [0,1), 53 bits.
 * ---------------------------------------------------------------------------------------- */
ORC_API void orc_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

ORC_API double orc_stream_uniform(uint64_t seed, uint64_t chain, uint64_t n) {
  uint64_t blk = n >> 1;
  uint32_t ctr[4] = {(uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)chain, (uint32_t)(chain >> 32)};
  uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)}, r[4];
  orc_philox4x32_10(ctr, key, r);
  uint32_t a = (n & 1) ? r[2] : r[0], b = (n & 1) ? r[3] : r[1];
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

typedef struct {
  uint64_t seed, chain, n;           /* Philox stream position */
  const double* replay; uint64_t replay_len;   /* optional: explicit uniform tape (tests) */
} orc_rng;

static double rng_next(orc_rng* g) {
  if (g->replay) { double u = g->replay[g->n % g->replay_len]; g->n++; return u; }
  return orc_stream_uniform(g->seed, g->chain, g->n++);
}

/* runif / runif_discrete -- mcmc.js:31-38 */
static double runif_(orc_rng* g, double mn, double mx) { return rng_next(g) * (mx - mn) + mn; }
static double runif_discrete_(orc_rng* g, double mn, double mx) { return floor(rng_next(g) * (mx - mn + 1)) + mn; }

/* rnorm -- mcmc.js:43-54 (Leva ratio-of-uniforms; 2 uniforms per trial) */
static double rnorm_(orc_rng* g, double mean, double sd) {
  double u, v, x, y, q;
  do {
    u = rng_next(g);
    v = 1.7156 * (rng_next(g) - 0.5);
    x = u - 0.449871;
    y = fabs(v) + 0.386595;
    q = x * x + y * (0.19600 * y - 0.25472 * x);
  } while (q > 0.27597 && (q > 0.27846 || v * v > -4 * orc_log(u) * u * u));
  return (v / u) * sd + mean;
}

/* shuffle_array -- mcmc.js:228-236 (Durstenfeld, in place, len-1 uniforms) */
static void shuffle_ints(orc_rng* g, int* a, int len) {
  for (int i = len - 1; i > 0; i--) {
    int j = (int)floor(rng_next(g) * (i + 1));
    int t = a[i]; a[i] = a[j]; a[j] = t;
  }
}

/* stand-alone entry points for unit tests of the helpers */
ORC_API double orc_runif(uint64_t seed, uint64_t chain, uint64_t* n, double mn, double mx) {
  orc_rng g = {seed, chain, *n, 0, 0}; double r = runif_(&g, mn, mx); *n = g.n; return r; }
ORC_API double orc_runif_discrete(uint64_t seed, uint64_t chain, uint64_t* n, double mn, double mx) {
  orc_rng g = {seed, chain, *n, 0, 0}; double r = runif_discrete_(&g, mn, mx); *n = g.n; return r; }
ORC_API double orc_rnorm(uint64_t seed, uint64_t chain, uint64_t* n, double mean, double sd) {
  orc_rng g = {seed, chain, *n, 0, 0}; double r = rnorm_(&g, mean, sd); *n = g.n; return r; }
ORC_API void orc_shuffle(uint64_t seed, uint64_t chain, uint64_t* n, int* a, int len) {
  orc_rng g = {seed, chain, *n, 0, 0}; shuffle_ints(&g, a, len); *n = g.n; }

/* ------------------------------------------------------------------------------------------
 * ld.*  -- distributions.js:63-284, same operation order as the JS source.
 * ---------------------------------------------------------------------------------------- */
#define JS_PI 3.141592653589793

ORC_API double orc_ld_lgamma(double x) {                                 /* distributions.js:63-76 */
  static const double cof[6] = {76.18009172947146, -86.50532032941677, 24.01409824083091,
                                -1.231739572450155, 0.1208650973866179e-2, -0.5395239384953e-5};
  double ser = 1.000000000190015, xx, y, tmp;
  tmp = (y = xx = x) + 5.5;
  tmp -= (xx + 0.5) * orc_log(tmp);
  for (int j = 0; j < 6; j++) ser += cof[j] / ++y;
  return orc_log(2.5066282746310005 * ser / xx) - tmp;
}
ORC_API double orc_ld_lfactorial(double n) { return n < 0 ? NAN : orc_ld_lgamma(n + 1); }          /* :79-81 */
ORC_API double orc_ld_lchoose(double n, double k) {                                              /* :84-86 */
  return orc_ld_lfactorial(n) - orc_ld_lfactorial(k) - orc_ld_lfactorial(n - k); }
ORC_API double orc_ld_lbeta(double a, double b) {                                                /* :89-91 */
  return orc_ld_lgamma(a) + orc_ld_lgamma(b) - orc_ld_lgamma(a + b); }

ORC_API double orc_ld_beta(double x, double shape1, double shape2) {                             /* :104-113 */
  if (x > 1 || x < 0) return -INFINITY;
  if (shape1 == 1 && shape2 == 1) return 0;
  return (shape1 - 1) * orc_log(x) + (shape2 - 1) * orc_log(1 - x) - orc_ld_lbeta(shape1, shape2);
}
ORC_API double orc_ld_cauchy(double x, double location, double scale) {                          /* :115-117 */
  return orc_log(scale) - orc_log(js_pow(x - location, 2) + js_pow(scale, 2)) - orc_log(JS_PI); }
ORC_API double orc_ld_norm(double x, double mean, double sd) {                                   /* :119-121 */
  return -0.5 * orc_log(2 * JS_PI) - orc_log(sd) - js_pow(x - mean, 2) / (2 * sd * sd); }
ORC_API double orc_ld_bivarnorm(const double* x, const double* mean, const double* sd, double corr) { /* :125-133 */
  double z = js_pow(x[0] - mean[0], 2) / js_pow(sd[0], 2) + js_pow(x[1] - mean[1], 2) / js_pow(sd[1], 2) -
             (2 * corr * (x[0] - mean[0]) * (x[1] - mean[1])) / (sd[0] * sd[1]);
  double nf = -(orc_log(2) + orc_log(JS_PI) + orc_log(sd[0]) + orc_log(sd[1]) + 0.5 * orc_log(1 - js_pow(corr, 2)));
  return nf - z / (2 * (1 - js_pow(corr, 2)));
}
ORC_API double orc_ld_laplace(double x, double location, double scale) {                         /* :136-138 */
  return (-fabs(x - location) / scale) - orc_log(2 * scale); }
ORC_API double orc_ld_gamma(double x, double shape, double rate) {                               /* :142-152 */
  double scale = 1 / rate;
  if (x < 0) return -INFINITY;
  if (x == 0 && shape == 1) return -orc_log(scale);
  return (shape - 1) * orc_log(x) - x / scale - orc_ld_lgamma(shape) - shape * orc_log(scale);
}
ORC_API double orc_ld_invgamma(double x, double shape, double scale) {                           /* :154-159 */
  if (x <= 0) return -INFINITY;
  return -(shape + 1) * orc_log(x) - scale / x - orc_ld_lgamma(shape) + shape * orc_log(scale);
}
ORC_API double orc_ld_lnorm(double x, double meanlog, double sdlog) {                            /* :161-167 */
  if (x <= 0) return -INFINITY;
  return -orc_log(x) - 0.5 * orc_log(2 * JS_PI) - orc_log(sdlog) - js_pow(orc_log(x) - meanlog, 2) / (2 * sdlog * sdlog);
}
ORC_API double orc_ld_pareto(double x, double scale, double shape) {                             /* :169-174 */
  if (x < scale) return -INFINITY;
  return orc_log(shape) + shape * orc_log(scale) - (shape + 1) * orc_log(x);
}
ORC_API double orc_ld_t(double x, double location, double scale, double df) {                    /* :176-180 */
  df = df > 1e100 ? 1e100 : df;
  return orc_ld_lgamma((df + 1) / 2) - orc_ld_lgamma(df / 2) - orc_log(sqrt(JS_PI * df) * scale) +
         orc_log(js_pow(1 + (1 / df) * js_pow((x - location) / scale, 2), -(df + 1) / 2));
}
ORC_API double orc_ld_weibull(double x, double shape, double scale) {                            /* :185-191 */
  if (x < 0) return -INFINITY;
  if (x == 0 && shape < 1) return INFINITY;
  double tmp1 = js_pow(x / scale, shape - 1);
  double tmp2 = tmp1 * (x / scale);
  return -tmp2 + orc_log(shape * tmp1 / scale);
}
ORC_API double orc_ld_logis(double x, double location, double scale) {                           /* :196-201 */
  x = fabs((x - location) / scale);
  double e = orc_exp(-x), f = 1.0 + e;
  return -(x + orc_log(scale * f * f));
}
ORC_API double orc_ld_dirichlet(const double* x, const double* alpha, int n) {                   /* :203-214 */
  double sum_alpha = 0, sum_lgamma_alpha = 0, s = 0;
  for (int i = 0; i < n; i++) {
    sum_alpha += alpha[i];
    sum_lgamma_alpha += orc_ld_lgamma(alpha[i]);
    s += (alpha[i] - 1) * orc_log(x[i]);
  }
  return orc_ld_lgamma(sum_alpha) - sum_lgamma_alpha + s;
}
ORC_API double orc_ld_exp(double x, double rate) { return x < 0 ? -INFINITY : orc_log(rate) - rate * x; }  /* :217-219 */
ORC_API double orc_ld_unif(double x, double mn, double mx) {                                     /* :221-223 */
  return (x < mn || x > mx) ? -INFINITY : orc_log(1 / (mx - mn)); }
ORC_API double orc_ld_bern(double x, double prob) {                                              /* :228-230 */
  return !(x == 0 || x == 1) ? -INFINITY : orc_log(x * prob + (1 - x) * (1 - prob)); }
ORC_API double orc_ld_cat(double x, const double* probs, int n) {                                /* :232-238 */
  if (x < 1 || x > n) return -INFINITY;
  return orc_log(probs[(int)x - 1]);
}
ORC_API double orc_ld_binom(double x, double size, double prob) {                                /* :240-248 */
  if (x > size || x < 0) return -INFINITY;
  if (prob == 0 || prob == 1) return (size * prob) == x ? 0 : -INFINITY;
  return orc_ld_lchoose(size, x) + x * orc_log(prob) + (size - x) * orc_log(1 - prob);
}
ORC_API double orc_ld_nbinom(double x, double size, double prob) {                               /* :267-272 */
  if (x < 0) return -INFINITY;
  return orc_ld_lchoose(x + size - 1, size - 1) + x * orc_log(1 - prob) + size * orc_log(prob);
}
ORC_API double orc_ld_hyper(double x, double m, double n, double k) {                            /* :274-280 */
  if (x < 0 || x > k) return -INFINITY;
  return orc_ld_lchoose(m, x) + orc_ld_lchoose(n, k - x) - orc_ld_lchoose(m + n, k);
}
ORC_API double orc_ld_pois(double x, double lambda) {                                            /* :282-284 */
  return x < 0 ? -INFINITY : orc_log(lambda) * x - lambda - orc_ld_lfactorial(x); }

/* param_init_fixed -- mcmc.js:313-341.  type: 0 real, 1 int, 2 binary.  Returns NaN where JS throws. */
ORC_API double orc_param_init_fixed(int type, double lower, double upper) {
  if (lower > upper) return NAN;
  if (type == 0) {
    if (lower == -INFINITY && upper == INFINITY) return 0.5;
    if (lower == -INFINITY) return upper - 0.5;
    if (upper == INFINITY) return lower + 0.5;
    if (lower <= upper) return (lower + upper) / 2;
  } else if (type == 1) {
    if (lower == -INFINITY && upper == INFINITY) return 1;
    if (lower == -INFINITY) return upper - 1;
    if (upper == INFINITY) return lower + 1;
    if (lower <= upper) return orc_js_round((lower + upper) / 2);
  } else if (type == 2) {
    return 1;
  }
  return NAN;
}

/* ------------------------------------------------------------------------------------------
 * Steppers and Sampler -- mcmc.js:433-1099.
 * The state is a flat fp64 vector: the D parameter components in Object.keys(params) order,
 * multi-dim params flattened row-major, followed by the model's derived quantities.
 * log_post(state, data, user) may write the derived slots (mcmc.js:961-963, test_data.js:89).
 * ---------------------------------------------------------------------------------------- */
typedef double (*orc_logpost_fn)(double* state, const void* data, void* user);

typedef struct {                      /* one entry of `params`, completed (mcmc.js:357-403) */
  int32_t type;                       /* 0 real, 1 int, 2 binary */
  int32_t n_comp;                     /* prod(dim) */
  int32_t dim0;                       /* dim[0]: the only level visited in random order (mcmc.js:244-263) */
  int32_t comp_offset;                /* first flat component */
  double lower, upper;
} orc_param;

typedef struct {                      /* per scalar component: resolved stepper options (mcmc.js:500-505) */
  double prop_log_scale;
  double batch_size;
  double max_adaptation;
  double initial_adaptation;
  double target_accept_rate;
  int32_t is_adapting;
  int32_t _pad;
} orc_comp_options;

typedef struct {                      /* OnedimMetropolisStepper -- mcmc.js:485-512 */
  int comp, is_int;
  double lower, upper;
  double prop_log_scale, batch_size, max_adaptation, initial_adaptation, target_accept_rate;
  int is_adapting;
  double acceptance_count, batch_count, iterations_since_adaption;
} onedim_t;

typedef struct {                      /* one substepper of AmwgStepper (mcmc.js:844-879) */
  int param_index;                    /* which named param it was built for */
  int kind;                           /* 0 onedim, 1 multidim metropolis, 2 binary, 3 binary component */
  int comp_offset, n_comp, dim0;
  onedim_t* subs;                     /* kind 0/1 */
} substepper_t;

typedef struct orc_sampler {
  int n_params, D, n_derived;
  orc_param* params;
  double* state;
  orc_logpost_fn fn; const void* data; void* user;
  substepper_t** substeppers;         /* shuffled IN PLACE every sweep (mcmc.js:887) */
  substepper_t* storage;
  orc_rng rng;
  int64_t thinning_interval;
  int64_t n_logpost_calls;            /* instrumentation: how many evals the reference does */
  int* scratch;
  double* trace; int64_t trace_cap, trace_len;   /* optional step trace (orc_trace) */
} orc_sampler;

static double call_log_post(orc_sampler* s) { s->n_logpost_calls++; return s->fn(s->state, s->data, s->user); }

/* OnedimMetropolisStepper.prototype.step -- mcmc.js:517-553 */
static void onedim_step(orc_sampler* s, onedim_t* st) {
  double param_state = s->state[st->comp];
  /* generate_proposal: normal_proposal (:577-579) / discrete_normal_proposal (:596-598) */
  double param_proposal = rnorm_(&s->rng, param_state, orc_exp(st->prop_log_scale));
  if (st->is_int) param_proposal = orc_js_round(param_proposal);
  double* rec = (s->trace && s->trace_len < s->trace_cap) ? s->trace + 6 * s->trace_len : NULL;
  if (s->trace) s->trace_len++;
  if (rec) { rec[0] = st->comp; rec[1] = param_state; rec[2] = param_proposal; rec[3] = -1.0; rec[4] = NAN; rec[5] = NAN; }
  if (param_proposal < st->lower || param_proposal > st->upper) {
    /* outside the limits: reject, no log_post, no accept uniform (:520-522) */
  } else {
    double curr_log_dens = call_log_post(s);
    s->state[st->comp] = param_proposal;
    double prop_log_dens = call_log_post(s);
    double accept_prob = orc_exp(prop_log_dens - curr_log_dens);
    double u = rng_next(&s->rng);
    if (rec) { rec[3] = u; rec[4] = curr_log_dens; rec[5] = prop_log_dens; }
    if (accept_prob > u) {
      if (st->is_adapting) st->acceptance_count++;
    } else {
      s->state[st->comp] = param_state;
    }
  }
  if (st->is_adapting) {
    st->iterations_since_adaption++;
    if (st->iterations_since_adaption >= st->batch_size) {
      st->batch_count++;
      double log_sd_adjustment = js_min(st->max_adaptation, st->initial_adaptation / sqrt(st->batch_count));
      if (st->acceptance_count / st->batch_size > st->target_accept_rate) st->prop_log_scale += log_sd_adjustment;
      else st->prop_log_scale -= log_sd_adjustment;
      st->acceptance_count = 0;
      st->iterations_since_adaption = 0;
    }
  }
}

/* BinaryStepper.prototype.step -- mcmc.js:753-767 */
static void binary_step(orc_sampler* s, int comp) {
  s->state[comp] = 0;
  double zero_log_dens = call_log_post(s);
  s->state[comp] = 1;
  double one_log_dens = call_log_post(s);
  double max_log_dens = js_max(zero_log_dens, one_log_dens);
  zero_log_dens -= max_log_dens;
  one_log_dens -= max_log_dens;
  double zero_prob = orc_exp(zero_log_dens - orc_log(orc_exp(zero_log_dens) + orc_exp(one_log_dens)));
  if (rng_next(&s->rng) < zero_prob) s->state[comp] = 0;
}

/* nested_array_random_apply over the top level, in-order below -- mcmc.js:244-263, :685-688, :817-820 */
static void multidim_step(orc_sampler* s, substepper_t* ss) {
  int len = ss->dim0, inner = ss->n_comp / ss->dim0;
  int* array_is = s->scratch;
  for (int i = 0; i < len; i++) array_is[i] = i;
  shuffle_ints(&s->rng, array_is, len);
  for (int i = 0; i < len; i++) {
    int array_i = array_is[i];
    for (int r = 0; r < inner; r++) {
      int c = array_i * inner + r;
      if (ss->kind == 1) onedim_step(s, &ss->subs[c]);
      else binary_step(s, ss->comp_offset + c);
    }
  }
}

/* AmwgStepper.prototype.step -- mcmc.js:886-892 */
static void amwg_step(orc_sampler* s) {
  /* shuffle_array(this.substeppers): in place, persists across sweeps */
  for (int i = s->n_params - 1; i > 0; i--) {
    int j = (int)floor(rng_next(&s->rng) * (i + 1));
    substepper_t* t = s->substeppers[i]; s->substeppers[i] = s->substeppers[j]; s->substeppers[j] = t;
  }
  for (int i = 0; i < s->n_params; i++) {
    substepper_t* ss = s->substeppers[i];
    switch (ss->kind) {
      case 0: onedim_step(s, &ss->subs[0]); break;
      case 2: binary_step(s, ss->comp_offset); break;
      default: multidim_step(s, ss); break;
    }
  }
}

/* Sampler.prototype.step -- mcmc.js:985-997.  shuffle_array(this.steppers) has length 1: no RNG use. */
ORC_API void orc_step(orc_sampler* s) {
  amwg_step(s);
  if (s->n_derived > 0) call_log_post(s);      /* refresh derived quantities (:990-995) */
}

/* Sampler ctor + AmwgSampler + AmwgStepper ctor -- mcmc.js:940-966, 1090-1099, 837-881.
 * `init` is params[*].init flattened (complete_params is host logic and is tested directly
 * against the reference's golden fixtures); `opts` are the per-component resolved options. */
ORC_API orc_sampler* orc_create(int n_params, const orc_param* params, const double* init,
                                const orc_comp_options* opts, int n_derived,
                                orc_logpost_fn fn, const void* data, void* user,
                                uint64_t seed, uint64_t chain) {
  orc_sampler* s = (orc_sampler*)calloc(1, sizeof(orc_sampler));
  s->n_params = n_params;
  s->params = (orc_param*)malloc(sizeof(orc_param) * (size_t)n_params);
  memcpy(s->params, params, sizeof(orc_param) * (size_t)n_params);
  int D = 0, maxdim = 1;
  for (int p = 0; p < n_params; p++) { D += params[p].n_comp; if (params[p].dim0 > maxdim) maxdim = params[p].dim0; }
  s->D = D; s->n_derived = n_derived;
  s->state = (double*)calloc((size_t)(D + n_derived), sizeof(double));
  memcpy(s->state, init, sizeof(double) * (size_t)D);
  s->fn = fn; s->data = data; s->user = user;
  s->rng.seed = seed; s->rng.chain = chain; s->rng.n = 0;
  s->thinning_interval = 1;
  s->scratch = (int*)malloc(sizeof(int) * (size_t)maxdim);
  call_log_post(s);                              /* mcmc.js:963 */
  s->storage = (substepper_t*)calloc((size_t)n_params, sizeof(substepper_t));
  s->substeppers = (substepper_t**)malloc(sizeof(substepper_t*) * (size_t)n_params);
  for (int p = 0; p < n_params; p++) {
    substepper_t* ss = &s->storage[p];
    const orc_param* pa = &params[p];
    ss->param_index = p; ss->comp_offset = pa->comp_offset; ss->n_comp = pa->n_comp; ss->dim0 = pa->dim0;
    int scalar = (pa->n_comp == 1 && pa->dim0 == 1);      /* array_equal(param.dim, [1]) */
    if (pa->type == 2) ss->kind = scalar ? 2 : 3;
    else ss->kind = scalar ? 0 : 1;
    if (pa->type != 2) {
      ss->subs = (onedim_t*)calloc((size_t)pa->n_comp, sizeof(onedim_t));
      for (int c = 0; c < pa->n_comp; c++) {
        onedim_t* o = &ss->subs[c];
        const orc_comp_options* q = &opts[pa->comp_offset + c];
        o->comp = pa->comp_offset + c; o->is_int = (pa->type == 1);
        o->lower = pa->lower; o->upper = pa->upper;
        o->prop_log_scale = q->prop_log_scale; o->batch_size = q->batch_size;
        o->max_adaptation = q->max_adaptation; o->initial_adaptation = q->initial_adaptation;
        o->target_accept_rate = q->target_accept_rate; o->is_adapting = q->is_adapting;
      }
    }
    s->substeppers[p] = ss;
  }
  return s;
}

ORC_API void orc_destroy(orc_sampler* s) {
  if (!s) return;
  for (int p = 0; p < s->n_params; p++) free(s->storage[p].subs);
  free(s->storage); free(s->substeppers); free(s->params); free(s->state); free(s->scratch); free(s);
}

ORC_API void orc_set_replay(orc_sampler* s, const double* tape, uint64_t len) { s->rng.replay = tape; s->rng.replay_len = len; s->rng.n = 0; }
/* Step trace (tests): from now on every OnedimMetropolisStepper step appends one row of six doubles to buf (room for cap rows):
 * component, current value, proposal, accept uniform (-1 when the proposal is out of bounds and none is drawn), curr_log_dens,
 * prop_log_dens (both NaN without evaluation). Steps beyond cap are counted but not written; buf NULL switches the trace off.
 * Returns the number of rows so far. */
ORC_API int64_t orc_trace(orc_sampler* s, double* buf, int64_t cap) {
  if (buf != s->trace) s->trace_len = 0;
  s->trace = buf; s->trace_cap = buf ? cap : 0;
  return s->trace_len;
}
ORC_API int64_t orc_trace_len(const orc_sampler* s) { return s->trace_len; }
ORC_API uint64_t orc_rng_position(const orc_sampler* s) { return s->rng.n; }
ORC_API int64_t orc_logpost_calls(const orc_sampler* s) { return s->n_logpost_calls; }
ORC_API void orc_thin(orc_sampler* s, int64_t k) { s->thinning_interval = k; }          /* mcmc.js:1053-1055 */
ORC_API const double* orc_state(const orc_sampler* s) { return s->state; }

/* Sampler.prototype.burn -- mcmc.js:1035-1039 */
ORC_API void orc_burn(orc_sampler* s, int64_t n) { for (int64_t i = 0; i < n; i++) orc_step(s); }

/* Sampler.prototype.sample -- mcmc.js:1005-1030.  monitor = flat state indices (components and/or
 * derived slots); out is [ceil(n/thin)][n_monitor], row recorded BEFORE the step. Returns rows. */
ORC_API int64_t orc_sample(orc_sampler* s, int64_t n, const int32_t* monitor, int n_monitor, double* out) {
  int64_t rows = 0;
  for (int64_t i = 0; i < n; i++) {
    if (i % s->thinning_interval == 0) {
      for (int j = 0; j < n_monitor; j++) out[rows * n_monitor + j] = s->state[monitor[j]];
      rows++;
    }
    orc_step(s);
  }
  return rows;
}

/* start_adaptation / stop_adaptation -- mcmc.js:1060-1073 -> :894-904 -> :555-561, :690-696 */
ORC_API void orc_set_adapting(orc_sampler* s, int flag) {
  for (int p = 0; p < s->n_params; p++) {
    substepper_t* ss = &s->storage[p];
    if (ss->subs) for (int c = 0; c < ss->n_comp; c++) ss->subs[c].is_adapting = flag;
  }
}

/* info() -- mcmc.js:563-571 per component, flat order. out[c*5 + {0..4}] =
 * prop_log_scale, is_adapting, acceptance_count, iterations_since_adaption, batch_count (NaN for binary) */
ORC_API void orc_info(const orc_sampler* s, double* out) {
  for (int p = 0; p < s->n_params; p++) {
    const substepper_t* ss = &s->storage[p];
    for (int c = 0; c < ss->n_comp; c++) {
      double* o = out + (size_t)(ss->comp_offset + c) * 5;
      if (!ss->subs) { for (int k = 0; k < 5; k++) o[k] = NAN; continue; }
      const onedim_t* q = &ss->subs[c];
      o[0] = q->prop_log_scale; o[1] = q->is_adapting; o[2] = q->acceptance_count;
      o[3] = q->iterations_since_adaption; o[4] = q->batch_count;
    }
  }
}
/* current substepper order (param indices), to check the in-place cumulative shuffle */
ORC_API void orc_substepper_order(const orc_sampler* s, int32_t* out) {
  for (int p = 0; p < s->n_params; p++) out[p] = s->substeppers[p]->param_index;
}

/* ------------------------------------------------------------------------------------------
 * Models (the user's log_post closures), written as the reference's README/tests write them.
 * ---------------------------------------------------------------------------------------- */
typedef struct { const double* x; int64_t n; } orc_vec;

/* README.md:26-36 (configs 1 and 2): state = [mu, sigma] */
ORC_API double orc_model_norm_readme(double* st, const void* data, void* user) {
  (void)user; const orc_vec* d = (const orc_vec*)data;
  double log_post = 0;
  log_post += orc_ld_norm(st[0], 0, 100);
  log_post += orc_ld_unif(st[1], 0, 100);
  for (int64_t i = 0; i < d->n; i++) log_post += orc_ld_norm(d->x[i], st[0], st[1]);
  return log_post;
}
/* tests/test_data.js:80-91: as above plus the derived quantity par.var; state = [mu, sigma, var] */
ORC_API double orc_model_norm_test(double* st, const void* data, void* user) {
  double lp = orc_model_norm_readme(st, data, user);
  st[2] = st[1] * st[1];
  return lp;
}
/* README.md:149-164: beta-Bernoulli; state = [theta] */
ORC_API double orc_model_beta_bern(double* st, const void* data, void* user) {
  (void)user; const orc_vec* d = (const orc_vec*)data;
  double log_post = 0;
  log_post += orc_ld_beta(st[0], 2, 2);
  for (int64_t i = 0; i < d->n; i++) log_post += orc_ld_bern(d->x[i], st[0]);
  return log_post;
}
/* config 3 with the binary indicator (SURVEY 8(d).3, pattern of test_data.js:154-171):
 * state = [theta, m]; m ~ bern(0.5); y_i ~ bern(m === 0 ? 0.5 : theta) */
ORC_API double orc_model_spike_bern(double* st, const void* data, void* user) {
  (void)user; const orc_vec* d = (const orc_vec*)data;
  double theta = st[0], m = st[1];
  double log_post = 0;
  log_post += orc_ld_beta(theta, 2, 2);
  log_post += orc_ld_bern(m, 0.5);
  for (int64_t i = 0; i < d->n; i++) {
    if (m == 0) log_post += orc_ld_bern(d->x[i], 0.5);
    else log_post += orc_ld_bern(d->x[i], theta);
  }
  return log_post;
}
/* config 4: hierarchical normal; data: y[n], group[n]; state = [mu_0..mu_{J-1}, sigma] */
typedef struct { const double* y; const int32_t* g; int64_t n; int32_t J; } orc_hier;
ORC_API double orc_model_hier_norm(double* st, const void* data, void* user) {
  (void)user; const orc_hier* d = (const orc_hier*)data;
  double sigma = st[d->J];
  double log_post = 0;
  for (int j = 0; j < d->J; j++) log_post += orc_ld_norm(st[j], 0, 100);
  log_post += orc_ld_unif(sigma, 0, 100);
  for (int64_t i = 0; i < d->n; i++) log_post += orc_ld_norm(d->y[i], st[d->g[i]], sigma);
  return log_post;
}
/* config 5: Poisson regression; data: y[n], X[n][K] row-major; state = beta[K] */
typedef struct { const double* y; const double* X; int64_t n; int32_t K; } orc_poisreg;
ORC_API double orc_model_pois_reg(double* st, const void* data, void* user) {
  (void)user; const orc_poisreg* d = (const orc_poisreg*)data;
  double log_post = 0;
  for (int k = 0; k < d->K; k++) log_post += orc_ld_norm(st[k], 0, 10);
  for (int64_t i = 0; i < d->n; i++) {
    double eta = 0;
    for (int k = 0; k < d->K; k++) eta += d->X[i * d->K + k] * st[k];
    log_post += orc_ld_pois(d->y[i], orc_exp(eta));
  }
  return log_post;
}
/* tests/test_data.js:93-95, 109-111, 125-127: one-parameter densities used by the stepper tests */
ORC_API double orc_model_norm_dens(double* st, const void* d, void* u) { (void)d; (void)u; return orc_ld_norm(st[0], 10, 5); }
ORC_API double orc_model_poisson_dens(double* st, const void* d, void* u) { (void)d; (void)u; return orc_ld_pois(st[0], 10); }
ORC_API double orc_model_bern_dens(double* st, const void* d, void* u) { (void)d; (void)u; return orc_ld_bern(st[0], 0.85); }
/* tests/test_data.js:97-107, 113-123, 129-136: 2x2 multi-dim targets; state = x[0][0],x[0][1],x[1][0],x[1][1] */
ORC_API double orc_model_multivar_norm_dens(double* st, const void* d, void* u) { (void)d; (void)u;
  return orc_ld_norm(st[0], 1000, 50) + orc_ld_norm(st[1], 10, 5) + orc_ld_norm(st[2], 0.1, 0.5) + orc_ld_norm(st[3], 0.001, 0.05); }
ORC_API double orc_model_multivar_poisson_dens(double* st, const void* d, void* u) { (void)d; (void)u;
  return orc_ld_pois(st[0], 0.1) + orc_ld_pois(st[1], 10) + orc_ld_pois(st[2], 1000) + orc_ld_pois(st[3], 100000); }
ORC_API double orc_model_multi_bern_dens(double* st, const void* d, void* u) { (void)d; (void)u;
  double x1 = st[0], x2 = st[1], x3 = st[2], x4 = st[3];
  return orc_log(x1 * x2 * 0.85 + (1 - x1 * x2) * 0.15) + orc_log(x3 * x4 * 0.75 + (1 - x3 * x4) * 0.25); }
/* tests/test_data.js:154-171: real p1 in [0,1], int n1 >= 1, binary m; data x[] ; state = [p1, n1, m] */
ORC_API double orc_model_complex(double* st, const void* data, void* user) {
  (void)user; const orc_vec* d = (const orc_vec*)data;
  double p1 = st[0], n1 = st[1], m = st[2];
  double log_post = 0;
  log_post += orc_ld_bern(m, 0.4);
  log_post += orc_ld_beta(p1, 2, 2);
  log_post += orc_ld_nbinom(n1, 2, 0.1);
  for (int64_t i = 0; i < d->n; i++) {
    if (m == 0) log_post += orc_ld_nbinom(d->x[i], 21, 0.5);
    else log_post += orc_ld_nbinom(d->x[i], n1, p1);
  }
  return log_post;
}
/* tests/test_data.js:199-211: p dim [1,6], mu_logit_p, sigma_logit_p; data x[6], n[6];
 * state = [p_0..p_5, mu_logit_p, sigma_logit_p] */
typedef struct { const double* x; const double* n; int64_t len; } orc_binom_data;
ORC_API double orc_model_hier_binom(double* st, const void* data, void* user) {
  (void)user; const orc_binom_data* d = (const orc_binom_data*)data;
  double mu = st[d->len], sg = st[d->len + 1];
  double log_post = 0;
  log_post += orc_ld_norm(mu, 0, 10);
  log_post += orc_ld_norm(sg, 0, 10);
  for (int64_t i = 0; i < d->len; i++) {
    double p = st[i];
    log_post += orc_ld_norm(orc_log(p / (1 - p)), mu, sg);
    log_post += orc_ld_binom(d->x[i], d->n[i], p);
  }
  return log_post;
}

/* Many independent chains of one built-in model, optionally threaded by the caller (bench.py's CPU
 * baseline): runs chains [chain0, chain0+n_chains) burn + sample and writes out[chain][row][n_monitor], and, when final is not
 * NULL, each chain's state at the end, final[chain][D + n_derived]. */
ORC_API void orc_run_chains(int n_params, const orc_param* params, const double* init, const orc_comp_options* opts,
                            int n_derived, orc_logpost_fn fn, const void* data, uint64_t seed,
                            uint64_t chain0, int64_t n_chains, int64_t n_burn, int64_t n_sample, int64_t thin,
                            const int32_t* monitor, int n_monitor, double* out, double* final) {
  int64_t rows = (n_sample + thin - 1) / thin;
  for (int64_t c = 0; c < n_chains; c++) {
    orc_sampler* s = orc_create(n_params, params, init, opts, n_derived, fn, data, 0, seed, chain0 + (uint64_t)c);
    orc_thin(s, thin);
    orc_burn(s, n_burn);
    if (n_sample > 0) orc_sample(s, n_sample, monitor, n_monitor, out + (size_t)c * (size_t)rows * (size_t)n_monitor);
    if (final) memcpy(final + (size_t)c * (size_t)(s->D + n_derived), s->state, sizeof(double) * (size_t)(s->D + n_derived));
    orc_destroy(s);
  }
}

/* The same, on `n_threads` host threads (bench.py --impl reference: the reference is single-threaded JavaScript, mcmc.js has no
 * parallelism; independent chains are the only way to occupy a many-core host with it). Chains are dealt out in contiguous
 * blocks; every chain is the same computation as in orc_run_chains, so the output does not depend on n_threads. */
#include <pthread.h>
typedef struct {
  int n_params; const orc_param* params; const double* init; const orc_comp_options* opts; int n_derived; orc_logpost_fn fn;
  const void* data; uint64_t seed, chain0; int64_t c_lo, c_hi, n_burn, n_sample, thin; const int32_t* monitor; int n_monitor; double* out;
  double* final; int width;
} orc_mt_job;
static void* orc_mt_worker(void* arg) {
  orc_mt_job* j = (orc_mt_job*)arg;
  int64_t rows = (j->n_sample + j->thin - 1) / j->thin;
  if (j->c_hi > j->c_lo)
    orc_run_chains(j->n_params, j->params, j->init, j->opts, j->n_derived, j->fn, j->data, j->seed, j->chain0 + (uint64_t)j->c_lo,
                   j->c_hi - j->c_lo, j->n_burn, j->n_sample, j->thin, j->monitor, j->n_monitor,
                   j->out ? j->out + (size_t)j->c_lo * (size_t)rows * (size_t)j->n_monitor : NULL,
                   j->final ? j->final + (size_t)j->c_lo * (size_t)j->width : NULL);
  return NULL;
}
ORC_API int orc_run_chains_mt(int n_params, const orc_param* params, const double* init, const orc_comp_options* opts,
                              int n_derived, orc_logpost_fn fn, const void* data, uint64_t seed,
                              uint64_t chain0, int64_t n_chains, int64_t n_burn, int64_t n_sample, int64_t thin,
                              const int32_t* monitor, int n_monitor, double* out, double* final, int n_threads) {
  int width = n_derived;
  for (int p = 0; p < n_params; p++) width += params[p].n_comp;
  if (n_threads < 1) n_threads = 1;
  if ((int64_t)n_threads > n_chains) n_threads = (int)n_chains;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)n_threads);
  orc_mt_job* jobs = (orc_mt_job*)malloc(sizeof(orc_mt_job) * (size_t)n_threads);
  int started = 0;
  for (int t = 0; t < n_threads; t++) {
    orc_mt_job j = { n_params, params, init, opts, n_derived, fn, data, seed, chain0,
                     n_chains * t / n_threads, n_chains * (t + 1) / n_threads, n_burn, n_sample, thin, monitor, n_monitor, out,
                     final, width };
    jobs[t] = j;
    if (pthread_create(&th[t], NULL, orc_mt_worker, &jobs[t]) != 0) break;
    started++;
  }
  for (int t = 0; t < started; t++) pthread_join(th[t], NULL);
  for (int t = started; t < n_threads; t++) orc_mt_worker(&jobs[t]);      /* could not start a thread: run its block here */
  free(th); free(jobs);
  return started;
}
