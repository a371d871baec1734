// amwg_init.cuh -- over-dispersed starting points (amwg_disperse_state, DESIGN.md §2 "Dispersed starting points").
//
// One attempt for one component of one chain: a uniform from a reserved part of the chain's own Philox stream, a step of
// +-radius around the component's init on the unconstrained scale, and the map back to the parameter's support. Everything is
// js_log / js_exp / js_round and single IEEE-754 operations, so a host restatement (tests/test_inits_host.py compiles this very
// file with g++ through tests/host_shim) reproduces it bit for bit.
#pragma once
#include "amwg_math.cuh"

namespace amwg {

constexpr int kDisperseAttempts = 100;                 // attempts per chain before amwg_disperse_state gives up
constexpr uint64_t kInitStreamBase = 1ull << 63;       // uniform #(2^63 + a*n_comp + c): Math.random() never gets there

// The chain whose stream draws the attempts of global chain `chain` when superchains of `superchain_size` consecutive chains
// start together (amwg_disperse_state_superchains): the superchain's first chain, superchain_size * floor(chain /
// superchain_size). Every chain of a superchain then draws the same attempts and keeps the same point; superchain_size = 1 is
// the chain itself.
__device__ __forceinline__ uint64_t superchain_leader(uint64_t chain, uint64_t superchain_size) {
  return chain - chain % superchain_size;
}

// uniform of attempt `attempt` for component `c` of global chain `chain`
__device__ __forceinline__ double disperse_uniform(uint64_t seed, uint64_t chain, int attempt, int n_comp, int c) {
  RandomStream g;
  g.init(kInitStreamBase + (uint64_t)attempt * (uint64_t)n_comp + (uint64_t)c);
  return g.next(seed, chain);
}

// The value an attempt proposes for a component of type `type` (0 real, 1 int, 2 binary: amwg.h AMWG_*) with bounds
// [lower, upper] and init `init`, given the attempt's uniform U. Returns whether the value is a valid starting value of the
// component (inside [lower, upper]; binary values always are). Whether log_post is finite there is the kernel's part.
__device__ __forceinline__ bool disperse_component(int type, double lower, double upper, double init, double radius, double U, double* out) {
  if (type == 2) { *out = U < 0.5 ? 0.0 : 1.0; return true; }
  const bool lo = lower != -CUDART_INF, hi = upper != CUDART_INF;
  double z0 = init;                                     // the centre on the unconstrained scale
  if (lo && hi) z0 = js_log(init - lower) - js_log(upper - init);
  else if (lo) z0 = js_log(init - lower);
  else if (hi) z0 = js_log(upper - init);
  if (!(z0 - z0 == 0.0)) z0 = 0.0;                      // init on or outside a bound (or not a number): centre at 0
  const double u = (2.0 * U - 1.0) * radius;
  const double z = z0 + u;
  double x = z;
  if (lo && hi) x = lower + (upper - lower) / (1.0 + js_exp(-z));
  else if (lo) x = lower + js_exp(z);
  else if (hi) x = upper - js_exp(z);
  if (type == 1) x = js_round(x);
  *out = x;
  return x >= lower && x <= upper;
}

}  // namespace amwg
