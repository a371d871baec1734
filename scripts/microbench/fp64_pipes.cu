// Micro-benchmark behind DESIGN.md's Poisson-plate and statistics-sweep notes: how fast are DFMA, DMMA (mma.sync m8n8k4 f64),
// broadcast LDS.128 and quad-pattern LDS.64 (four distinct 8-byte words per warp, one per lane & 3, in a 32-byte window: the loads
// of a plate sum whose quads of lanes share every value, DESIGN.md section 4.1) on this GPU, alone and together? A loaded value is
// folded into one of four integer XOR accumulators (one LOP3 on the integer pipe): no fp64 instruction and no long dependency chain
// rides on the loads.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_pipes fp64_pipes.cu && ./fp64_pipes
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <int NF, int NM, int NL, int W>
__global__ void __launch_bounds__(256) k(double* out, long long iters, double x) {
  __shared__ __align__(16) double tab[512];
  for (int i = threadIdx.x; i < 512; i += blockDim.x) tab[i] = 1.0 + 1e-9 * i;
  __syncthreads();
  double f[8]; double c[8][2];
#pragma unroll
  for (int j = 0; j < 8; ++j) { f[j] = x + j; c[j][0] = x; c[j][1] = x; }
  const double a = 1.0 + 1e-12 * threadIdx.x, b = 1.0 - 1e-12 * threadIdx.x;
  unsigned ix[4] = {0u, 0u, 0u, 0u};
  const unsigned sa = (unsigned)__cvta_generic_to_shared(tab);
  for (long long it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < NF; ++j) f[j & 7] = fma(f[j & 7], a, b);
#pragma unroll
    for (int j = 0; j < NM; ++j) dmma(c[j & 7][0], c[j & 7][1], a, b);
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      double2 v;
      if (W == 16) {
        asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(sa + 16u * (unsigned)((j + (int)it) & 31)));
        ix[j & 3] ^= (unsigned)__double2loint(v.x) ^ (unsigned)__double2hiint(v.y);
      } else {
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v.x) : "r"(sa + 8u * (threadIdx.x & 3u) + 32u * (unsigned)((j + (int)it) & 15)));
        ix[j & 3] ^= (unsigned)__double2loint(v.x) ^ (unsigned)__double2hiint(v.x);
      }
    }
  }
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) s += f[j] + c[j][0] + c[j][1];
  if (s == 1.2345 || (ix[0] ^ ix[1] ^ ix[2] ^ ix[3]) == 0x12345u) out[0] = s;
}

template <int NF, int NM, int NL, int W = 16>
static void run(const char* name, int warps_per_sm_target) {
  int dev = 0; cudaDeviceProp p; cudaGetDeviceProperties(&p, dev);
  const int threads = 256, blocks = p.multiProcessorCount * (warps_per_sm_target * 32 / threads);
  double* out; cudaMalloc(&out, 8);
  const long long iters = 20000;
  k<NF, NM, NL, W><<<blocks, threads>>>(out, 100, 1.0);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    cudaEventRecord(e0); k<NF, NM, NL, W><<<blocks, threads>>>(out, iters, 1.0); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
  }
  const double warps = (double)blocks * threads / 32, sec = best * 1e-3;
  const double clk = 1.965e9;   // nominal boost; the cycles below are per SM sub-partition at that clock
  const double per_sched_warps = warps / (p.multiProcessorCount * 4.0);
  const double cyc_per_iter_per_sched = sec * clk / iters;
  printf("%-28s warps/SM %2d  %8.3f ms  cycles/iteration/scheduler %7.1f  (per warp %6.2f)", name, warps_per_sm_target, best, cyc_per_iter_per_sched,
         cyc_per_iter_per_sched / per_sched_warps);
  if (NF) printf("  DFMA %.1f TF", warps * 32 * iters * NF * 2 / sec * 1e-12);
  if (NM) printf("  DMMA %.1f TF", warps * iters * NM * 512.0 / sec * 1e-12);
  if (NL) printf("  LDS.%d %.2f /clk/SM", 8 * W, warps * iters * NL / sec / clk / p.multiProcessorCount);
  printf("\n");
  cudaFree(out);
}

int main() {
  for (int w : {16, 32}) {
    run<16, 0, 0>("dfma x16", w);
    run<0, 8, 0>("dmma x8", w);
    run<0, 2, 0>("dmma x2 (dependent-ish)", w);
    run<16, 2, 0>("dfma x16 + dmma x2", w);
    run<20, 2, 0>("dfma x20 + dmma x2", w);
    run<16, 8, 0>("dfma x16 + dmma x8", w);
    run<0, 0, 16>("lds.128 broadcast x16", w);
    run<16, 0, 4>("dfma x16 + lds.128 x4", w);
    run<16, 0, 8>("dfma x16 + lds.128 x8", w);
    run<34, 0, 8>("dfma x34 + lds.128 x8", w);
    run<0, 0, 16, 8>("lds.64 quad x16", w);
    run<16, 0, 4, 8>("dfma x16 + lds.64 x4", w);
  }
  return 0;
}
