// Test infrastructure: the samplers of csrc/amwg_ppc.cuh (the file nvcc compiles for sm_90a) compiled for the HOST behind a C ABI,
// for tests/test_summary_ppc_host.py. Built with -ffp-contract=off (the GPU build uses --fmad=false).
#include "cuda_runtime.h"
#include "math_constants.h"
#include "amwg_ppc.cuh"

namespace {
// a fixed tape of uniforms, to force a branch (logis's U = 0 redraw); z() is mcmc.js's Leva rnorm over the tape
struct TapeSource {
  const double* t;
  uint64_t n, len;
  double u() { const double v = n < len ? t[n] : 0.5; ++n; return v; }
  double z() {
    double u0, v, x, y, q;
    do {
      u0 = u();
      v = 1.7156 * (u() - 0.5);
      x = u0 - 0.449871;
      y = fabs(v) + 0.386595;
      q = x * x + y * (0.19600 * y - 0.25472 * x);
    } while (q > 0.27597 && (q > 0.27846 || v * v > -4 * amwg::js_log(u0) * u0 * u0));
    return v / u0;
  }
  bool spent() const { return n > len; }
};
}  // namespace

extern "C" {

uint64_t hs_ppc_position(uint64_t row, uint64_t points, uint64_t i) { return ppc::stream_position(row, points, i); }

// the draw of (row, point i of `points`) for global chain `chain`; *used = the uniforms it took
double hs_ppc_draw(int fam, const double* a, uint64_t seed, uint64_t chain, uint64_t row, uint64_t points, uint64_t i, uint64_t* used) {
  ppc::PhiloxSource s;
  const uint64_t pos = ppc::stream_position(row, points, i);
  s.init(seed, chain, pos);
  const double x = ppc::draw(fam, a, s);
  *used = s.g.n - pos;
  return x;
}

// n draws at consecutive stream positions (for the distribution tests: draw j at row 0, point j of n); returns the largest number
// of uniforms any of them took
uint64_t hs_ppc_draws(int fam, const double* a, uint64_t seed, uint64_t chain, uint64_t n, double* out) {
  uint64_t most = 0;
  for (uint64_t j = 0; j < n; ++j) {
    ppc::PhiloxSource s;
    const uint64_t pos = ppc::stream_position(0, n, j);
    s.init(seed, chain, pos);
    out[j] = ppc::draw(fam, a, s);
    if (s.g.n - pos > most) most = s.g.n - pos;
  }
  return most;
}

double hs_ppc_draw_tape(int fam, const double* a, const double* tape, uint64_t len, uint64_t* used) {
  TapeSource s{tape, 0, len};
  const double x = ppc::draw(fam, a, s);
  *used = s.n;
  return x;
}

double hs_ppc_log_factorial(double k) { return ppc::log_factorial(k); }
double hs_ppc_log1p(double x) { return ppc::log1p_g(x); }
double hs_ppc_log_factorial_diff(double i, double e) { return ppc::log_factorial_diff(i, e); }

}
