// Test infrastructure: the dispersal transform of amwg_disperse_state (csrc/amwg_init.cuh, the file nvcc compiles for sm_90a)
// compiled for the HOST behind a C ABI, for tests/test_inits_host.py. Built with -ffp-contract=off (the GPU build uses --fmad=false).
#include "amwg_init.cuh"

using namespace amwg;
extern "C" {
double hs_disperse_uniform(uint64_t seed, uint64_t chain, int attempt, int n_comp, int c) { return disperse_uniform(seed, chain, attempt, n_comp, c); }
int hs_disperse_component(int type, double lower, double upper, double init, double radius, double U, double* out) {
  return disperse_component(type, lower, upper, init, radius, U, out) ? 1 : 0;
}
int hs_disperse_attempts(void) { return kDisperseAttempts; }
}
