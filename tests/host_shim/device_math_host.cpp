// Test infrastructure: the product's device arithmetic (csrc/amwg_math.cuh, csrc/amwg_ld.cuh -- the same files nvcc and NVRTC compile
// for sm_90a) compiled for the host behind a C ABI. Built by tests/test_device_math_on_host.py with -ffp-contract=off (the GPU build
// uses --fmad=false): every operation is one IEEE-754 fp64 operation on both sides.
#include "amwg_math.cuh"
#include "amwg_ld.cuh"

using namespace amwg;
extern "C" {
double hs_js_log(double x) { return js_log(x); }
double hs_js_exp(double x) { return js_exp(x); }
double hs_js_round(double x) { return js_round(x); }
double hs_js_max(double a, double b) { return js_max(a, b); }
double hs_js_min(double a, double b) { return js_min(a, b); }
double hs_uniform(uint64_t seed, uint64_t chain, uint64_t n) { RandomStream g; g.init(n); return g.next(seed, chain); }
double hs_rnorm(uint64_t seed, uint64_t chain, uint64_t* n, double mean, double sd) {
  RandomStream g; g.init(*n);
  const double v = js_rnorm(g, seed, chain, mean, sd);
  *n = g.n;
  return v;
}
double hs_lgamma(double a) { return ld_lgamma(a); }
double hs_lfactorial(double a) { return ld_lfactorial(a); }
double hs_lchoose(double a, double b) { return ld_lchoose(a, b); }
double hs_lbeta(double a, double b) { return ld_lbeta(a, b); }
#define HS3(name) double hs_##name(double a, double b, double c) { return ld_##name(a, b, c); }
#define HS2(name) double hs_##name(double a, double b) { return ld_##name(a, b); }
#define HS4(name) double hs_##name(double a, double b, double c, double d) { return ld_##name(a, b, c, d); }
HS3(beta) HS3(cauchy) HS3(norm) HS3(laplace) HS3(gamma) HS3(invgamma) HS3(lnorm) HS3(pareto) HS4(t) HS3(weibull) HS3(logis)
HS2(exp) HS3(unif) HS2(bern) HS3(binom) HS3(nbinom) HS4(hyper) HS2(pois)
}
