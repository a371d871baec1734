// amwg_tma.cuh -- device helpers shared by the ahead-of-time kernels (amwg_kernels.cu) and the run-time specialised sweep
// (amwg_jit_kernel.cuh, compiled by NVRTC): 1-D bulk TMA + mbarrier, warp-broadcast shared-memory loads, and the inner loop of
// every Normal likelihood sum, sum_i (x_i - mean)^2.
#pragma once

namespace amwg {

// ---- per-chain arrays and the arguments of one sweep launch (passed by value to every sweep kernel) --------------------
struct ChainArrays {
  double* state;          // [D][C]
  double* pls;            // [D][C] prop_log_scale
  double* psd;            // [D][C] exp(prop_log_scale): the proposal sd, recomputed only when pls changes (same bits as mcmc.js:578)
  int* acc;               // [D][C] acceptance_count of the current batch
  double* curr_lp;        // [C]   cached log_post(state)
  double* tval;           // [n_terms][C] term cache: value of every value-term of log_post at the chain's current state
  double* tcand;          // [n_terms][C] candidates written while a proposal is evaluated; committed on acceptance
  double* bprop;          // [D][C] block steps: the proposal of every component of the block (its current value when out of bounds)
  double* bcoin;          // [D][C] block steps: the accept uniform drawn for it (-1: proposal out of bounds, no uniform drawn)
  unsigned short* vseq;   // [D][C] pre-evaluated statistics: the components in this sweep's visiting order
  unsigned long long* perm;   // [C] substepper order, 4 bits per named parameter (persists: mcmc.js:887 shuffles in place)
  unsigned char* perm_ext;    // [P][C] the same order, one byte per entry, for models with more than 16 named parameters (else nullptr)
  unsigned short* order_ext;  // [max dim0][C] visiting order of a multi-dim parameter whose dim[0] exceeds 256 (else nullptr)
  unsigned long long* rng_n;  // [C] Math.random() calls consumed so far
  unsigned long long C;
  unsigned long long first_chain;
  unsigned long long seed;
};

struct SweepArgs {
  long long n_sweeps;
  long long sample_i0;     // index i of the first sweep within the current sample() call
  long long thin;
  int record;              // 0: burn, 1: sample
  int n_monitor;
  const int* monitor;      // global [n_monitor]
  double* out;             // [row][monitor][chain]
};

// ---- the two permutations of a sweep ------------------------------------------------------------------------------------------
// AmwgStepper shuffles its substeppers IN PLACE every sweep (mcmc.js:887): the order persists. Up to 16 named parameters it is one
// 64-bit word per chain, kept in a register; beyond that a byte per entry in global memory. A multi-dim parameter's visiting order
// (mcmc.js:246-252, a fresh shuffle every sweep) is a 256-byte local array, or 16-bit rows in global memory for dim[0] > 256.
// Threads that shadow the last chain (CTA-uniform data passes) never write the global forms; what they read is the owner's array
// at some moment -- always valid indices, and a shadow's results are discarded.
constexpr int kLocalOrder = 256;
__device__ __forceinline__ int perm_get(const ChainArrays& a, unsigned long long perm, unsigned long long chain, int i) {
  return a.perm_ext ? (int)a.perm_ext[(unsigned long long)i * a.C + chain] : (int)((perm >> (4 * i)) & 15ull);
}
__device__ __forceinline__ void perm_swap(const ChainArrays& a, unsigned long long& perm, unsigned long long chain, int i, int j, bool wr) {
  if (a.perm_ext) {
    if (!wr) return;
    unsigned char* pi = a.perm_ext + (unsigned long long)i * a.C + chain;
    unsigned char* pj = a.perm_ext + (unsigned long long)j * a.C + chain;
    const unsigned char t = *pi; *pi = *pj; *pj = t;
    return;
  }
  const unsigned long long vi = (perm >> (4 * i)) & 15ull, vj = (perm >> (4 * j)) & 15ull;
  perm = (perm & ~(15ull << (4 * i))) | (vj << (4 * i));
  perm = (perm & ~(15ull << (4 * j))) | (vi << (4 * j));
}
__device__ __forceinline__ int ord_get(const ChainArrays& a, const unsigned char* loc, unsigned long long chain, int dim0, int i) {
  return dim0 <= kLocalOrder ? (int)loc[i] : (int)a.order_ext[(unsigned long long)i * a.C + chain];
}
__device__ __forceinline__ void ord_set(const ChainArrays& a, unsigned char* loc, unsigned long long chain, int dim0, int i, int v, bool wr) {
  if (dim0 <= kLocalOrder) loc[i] = (unsigned char)v;
  else if (wr) a.order_ext[(unsigned long long)i * a.C + chain] = (unsigned short)v;
}

// ---- TMA 1-D bulk copy + mbarrier (sm_90+; SASS: UBLKCP / SYNCS) -------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(
          smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ double2 lds_f64x2(unsigned saddr) {
  double2 v;
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(saddr));
  return v;
}

__device__ __forceinline__ double lds_f64_sa(unsigned saddr) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(saddr)); return v; }

// ---- plates: the O(N) likelihood sums -----------------------------------------------------------------------------
// sum_i (x_i - mean)^2 : 2 fp64-pipe instructions per point (DADD + DFMA), four independent accumulators, eight points
// per block read as four 16-byte warp-broadcast loads (ld.shared.v2.f64 when `saddr` != 0, i.e. the column sits in shared
// memory; else the same loop over global/L2 addresses). From shared memory the next block is loaded while the current one is summed.
#define AMWG_ACC8(P0, P1, P2, P3)                                                                              \
  {                                                                                                            \
    double d0 = P0.x - mean, d1 = P0.y - mean, d2 = P1.x - mean, d3 = P1.y - mean;                             \
    double d4 = P2.x - mean, d5 = P2.y - mean, d6 = P3.x - mean, d7 = P3.y - mean;                             \
    s0 = fma(d0, d0, s0); s1 = fma(d1, d1, s1); s2 = fma(d2, d2, s2); s3 = fma(d3, d3, s3);                     \
    s0 = fma(d4, d4, s0); s1 = fma(d5, d5, s1); s2 = fma(d6, d6, s2); s3 = fma(d7, d7, s3);                     \
  }
__device__ __forceinline__ double sum_sq_dev(const double* __restrict__ x, unsigned saddr, int n, double mean) {
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
  int i = 0;
  if ((reinterpret_cast<unsigned long long>(x) & 15ull) && n > 0) { double d = x[0] - mean; s3 = fma(d, d, s3); i = 1; }   // 16B-align the vector loads
  const int nb = (n - i) >> 3;                 // blocks of eight points
  if (nb > 0) {
    if (saddr) {
      unsigned a = saddr + 8u * (unsigned)i;
      double2 p0 = lds_f64x2(a), p1 = lds_f64x2(a + 16u), p2 = lds_f64x2(a + 32u), p3 = lds_f64x2(a + 48u);
#pragma unroll 2
      for (int b = 1; b < nb; ++b) {
        a += 64u;
        double2 q0 = lds_f64x2(a), q1 = lds_f64x2(a + 16u), q2 = lds_f64x2(a + 32u), q3 = lds_f64x2(a + 48u);
        AMWG_ACC8(p0, p1, p2, p3)
        p0 = q0; p1 = q1; p2 = q2; p3 = q3;
      }
      AMWG_ACC8(p0, p1, p2, p3)
    } else {
      const double2* g = reinterpret_cast<const double2*>(x + i);
#pragma unroll 2
      for (int b = 0; b < nb; ++b, g += 4) {
        double2 p0 = g[0], p1 = g[1], p2 = g[2], p3 = g[3];
        AMWG_ACC8(p0, p1, p2, p3)
      }
    }
    i += nb << 3;
  }
  for (; i < n; ++i) { double d = x[i] - mean; s0 = fma(d, d, s0); }
  return (s0 + s1) + (s2 + s3);
}
#undef AMWG_ACC8

}  // namespace amwg
