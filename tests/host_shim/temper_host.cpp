// Test infrastructure: the swap decision of tempered ladders (csrc/amwg_temper.cuh, the file nvcc compiles for sm_90a) compiled for
// the HOST behind a C ABI, for tests/test_temper_host.py. Built with -ffp-contract=off (the GPU build uses --fmad=false).
#include "amwg_temper.cuh"

using namespace amwg;
extern "C" {
double hs_swap_uniform(uint64_t seed, uint64_t chain_a, uint64_t round) { return swap_uniform(seed, chain_a, round); }
int hs_swap_accept(double beta_a, double beta_b, double lp_a, double lp_b, double u) { return swap_accept(beta_a, beta_b, lp_a, lp_b, u) ? 1 : 0; }
int hs_swap_pairs(int K, uint64_t round) { return swap_pairs(K, round); }
int hs_max_rungs(void) { return kMaxRungs; }
}
