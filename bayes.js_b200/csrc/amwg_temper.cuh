// amwg_temper.cuh -- parallel tempering (DESIGN.md §2 "Tempered ladders"): the swap decision and the swap kernel.
//
// Global chain g is rung g mod K of ladder floor(g / K); a rung-r chain targets exp(beta_r * log_post). After every sweep, swap
// round k pairs, in every ladder, each rung r with r = k (mod 2) and r + 1 < K with rung r + 1 (the deterministic even/odd scheme of
// non-reversible parallel tempering, Syed, Bouchard-Cote, Deligiannidis & Doucet, JRSS-B 2022). The pair's uniform is
// #(2^63 + 2^62 + k) of the lower chain's own stream, above the dispersal range (amwg_init.cuh) and the predictive-check positions
// (amwg_ppc.cuh). The decision is one subtraction, one multiplication, js_exp and a strict comparison, so a host restatement
// (tests/test_temper_host.py compiles this very file with g++ through tests/host_shim) reproduces it bit for bit.
#pragma once
#include "amwg_math.cuh"

namespace amwg {

constexpr int kMaxRungs = 256;                                       // K <= 256 temperatures per ladder
constexpr uint64_t kSwapStreamBase = (1ull << 63) + (1ull << 62);     // uniform #(2^63 + 2^62 + k) decides round k

// the ladder a tempered sweep and the swap kernel read: beta[r] = 1 / T_r, computed once on the host
struct LadderDev {
  const double* beta;      // [K] global
  int K;                   // 0: untempered
};

// the uniform of swap round `round` of the pair whose lower chain is global chain `chain_a`
__device__ __forceinline__ double swap_uniform(uint64_t seed, uint64_t chain_a, uint64_t round) {
  RandomStream g;
  g.init(kSwapStreamBase + round);
  return g.next(seed, chain_a);
}

// accept the exchange of chains a (rung r, beta_a) and b (rung r + 1, beta_b) with untempered log_post lp_a, lp_b: strict >, so a NaN
// ratio rejects
__device__ __forceinline__ bool swap_accept(double beta_a, double beta_b, double lp_a, double lp_b, double u) {
  return js_exp((beta_a - beta_b) * (lp_b - lp_a)) > u;
}

// pairs per ladder in round `round`: rungs r = round (mod 2) with r + 1 < K
__host__ __device__ __forceinline__ int swap_pairs(int K, uint64_t round) { return (K - (int)(round & 1ull)) / 2; }

#ifdef __CUDACC__
// One thread per (ladder, pair) of round `round`, over the handle's C chains (C and first_chain are multiples of K). The pair's two
// chains are adjacent columns of every [.][C] array. On acceptance they exchange what is a function of the state: the state columns,
// curr_lp and the term cache (n_terms rows of tval). Proposal scales, acceptance counts, permutations and stream positions stay with
// the chain. accepts is [ladders][K - 1]: one thread owns each counter of a round, so no atomics.
__global__ void __launch_bounds__(256) amwg_swap_kernel(double* __restrict__ state, double* __restrict__ curr_lp, double* __restrict__ tval,
                                                        int D, int n_terms, unsigned long long C, unsigned long long first_chain,
                                                        unsigned long long seed, LadderDev ld, unsigned long long round,
                                                        unsigned long long* __restrict__ accepts) {
  const int K = ld.K;
  const int per = swap_pairs(K, round);
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long ladders = C / (unsigned long long)K;
  if (per == 0 || t >= ladders * (unsigned long long)per) return;
  const unsigned long long ladder = t / (unsigned long long)per;
  const int r = (int)(round & 1ull) + 2 * (int)(t - ladder * (unsigned long long)per);
  const unsigned long long ca = ladder * (unsigned long long)K + (unsigned long long)r, cb = ca + 1;
  const double lpa = curr_lp[ca], lpb = curr_lp[cb];
  const double u = swap_uniform(seed, first_chain + ca, round);
  if (!swap_accept(ld.beta[r], ld.beta[r + 1], lpa, lpb, u)) return;
  curr_lp[ca] = lpb; curr_lp[cb] = lpa;
  for (int c = 0; c < D; ++c) {
    double* p = state + (unsigned long long)c * C + ca;
    const double x = p[0]; p[0] = p[1]; p[1] = x;
  }
  for (int k = 0; k < n_terms; ++k) {
    double* p = tval + (unsigned long long)k * C + ca;
    const double x = p[0]; p[0] = p[1]; p[1] = x;
  }
  accepts[ladder * (unsigned long long)(K - 1) + (unsigned long long)r] += 1ull;
}
#endif

}  // namespace amwg
