// amwg_peak.cuh -- the measured roof of the sweep kernels: non-tensor fp64 FMA throughput of this GPU.
//
// MEASURED_PEAKS.json (driver-written) holds HBM and bf16 tensor peaks only; the AMWG hot path is bound by the fp64 pipe
// (DADD + DFMA per data point, DESIGN.md section 4), so bench.py measures that roof itself, in the same process and at the
// same clocks as the timed region: a grid of (SM count) x 8 CTAs x 256 threads, every thread running 8 independent DFMA chains
// (enough ILP and resident warps to keep the pipe issuing back to back), timed with CUDA events on the launching stream.
// Included at the end of amwg_kernels.cu (same translation unit: shares CUDA_TRY / fail()).
#pragma once

namespace peak {

__global__ void __launch_bounds__(256) amwg_fp64_fma_kernel(double* __restrict__ out, long long iters, double seed) {
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
  double a0 = seed + tid * 1e-9, a1 = a0 + 0.125, a2 = a0 + 0.25, a3 = a0 + 0.375;
  double a4 = a0 + 0.5, a5 = a0 + 0.625, a6 = a0 + 0.75, a7 = a0 + 0.875;
  const double m = 0.999999999, c = 1e-9;
  for (long long i = 0; i < iters; ++i) {
#pragma unroll 8
    for (int u = 0; u < 8; ++u) {
      a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
      a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
  }
  out[tid] = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));     // keeps the chains alive
}

}  // namespace peak

// Measured non-tensor fp64 throughput of `device` in TFLOP/s (2 flop per DFMA), best of `reps` launches of about `ms_target` ms.
extern "C" int amwg_peak_fp64(int device, int reps, double* tflops_out, double* ms_out) {
  if (!tflops_out) return fail("amwg_peak_fp64: tflops_out is NULL");
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop{};
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  const int threads = 256, grid = prop.multiProcessorCount * 8;
  double* d_out = nullptr;
  CUDA_TRY(cudaMalloc(&d_out, sizeof(double) * (size_t)grid * threads));
  cudaEvent_t e0, e1;
  CUDA_TRY(cudaEventCreate(&e0));
  CUDA_TRY(cudaEventCreate(&e1));
  const long long iters = 20000;                       // x 64 DFMA per thread per iteration
  double best = 0.0, best_ms = 0.0;
  cudaError_t err = cudaSuccess;
  for (int r = 0; r < (reps < 1 ? 1 : reps) + 1 && err == cudaSuccess; ++r) {      // first launch is the warm-up
    cudaEventRecord(e0, 0);
    peak::amwg_fp64_fma_kernel<<<grid, threads>>>(d_out, iters, 1.0 + r);
    cudaEventRecord(e1, 0);
    err = cudaEventSynchronize(e1);
    if (err != cudaSuccess) break;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    const double flop = 2.0 * 64.0 * (double)iters * (double)grid * threads;
    const double tf = flop / (ms * 1e-3) / 1e12;
    if (r > 0 && tf > best) { best = tf; best_ms = ms; }
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d_out);
  if (err != cudaSuccess) return fail(std::string("amwg_peak_fp64: ") + cudaGetErrorString(err));
  *tflops_out = best;
  if (ms_out) *ms_out = best_ms;
  return 0;
}
