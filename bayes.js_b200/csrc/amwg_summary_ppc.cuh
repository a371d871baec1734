// Posterior predictive checks in sample_summary(..., ppc=...) (DESIGN.md §4.8): replicated data y_rep[row][point][chain] drawn
// where the draws are, each draw's test statistics, and exact comparison counts.
//   K_p1  amwg_ppc_pointwise_kernel        : one thread per (row, chain) over a chunk of points: the K parameter programs of the
//                                            traced ld.* call, run by the model's interpreter (run_program_t) at the point index,
//                                            then the family's sampler (amwg_ppc.cuh) on the chain's stream. Writes y_rep in the
//                                            sample-block layout with points as entries (coalesced over chains) and carries the
//                                            draw's Welford record T[row][4][chain] = (m, M2, min, max) across chunks; the last
//                                            chunk replaces M2 by sd, which makes T a sample block of (mean, sd, min, max).
//   K_p2  amwg_threshold_counts_kernel     : grid (chain groups, entries): per entry the draws <, ==, > a threshold and NaN, summed
//                                            in 64-bit integers (warp shuffles, then one atomic per warp): exact in any order.
// Included at the end of amwg_kernels.cu, after amwg_summary_loo.cuh (the staging of pointwise programs, LooColumns).
#pragma once

#include "amwg_ppc.cuh"

namespace summary {

struct PpcPrograms { int pc[3]; };

// K_p1. Dynamic shared memory: the program words (padded to 8 bytes), then the folded constants (as K_l1).
__global__ void __launch_bounds__(kThreads) amwg_ppc_pointwise_kernel(const int* __restrict__ code, int n_code, const double* __restrict__ consts,
                                                                      int n_consts, int family, int K, PpcPrograms progs,
                                                                      const LooColumns* __restrict__ cols, const double* __restrict__ x,
                                                                      int entries, long long rows, long long C, unsigned long long first_chain,
                                                                      unsigned long long seed, long long N, int p0, int P, bool last,
                                                                      double* __restrict__ out, double* __restrict__ T) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ Ctx ctx;
  int* s_code = reinterpret_cast<int*>(smem);
  double* s_consts = reinterpret_cast<double*>(smem + (((unsigned)n_code * 4u + 7u) & ~7u));
  for (int i = threadIdx.x; i < n_code; i += blockDim.x) s_code[i] = code[i];
  for (int i = threadIdx.x; i < n_consts; i += blockDim.x) s_consts[i] = consts[i];
  for (int k = threadIdx.x; k < kMaxColumns; k += blockDim.x) ctx.col[k] = cols->col[k];
  __syncthreads();
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long r = (long long)blockIdx.z * 65535 + blockIdx.y;
  if (c >= C || r >= rows) return;
  const unsigned code_sa = smem_u32(s_code), consts_sa = smem_u32(s_consts);
  const EvalStateT<false> es{x + (size_t)r * entries * C + c, (unsigned long long)C, -1, 0.0};
  double* t = T + (size_t)r * 4 * C + c;
  double m = 0.0, M2 = 0.0, mn = CUDART_NAN, mx = CUDART_NAN;
  if (p0 > 0) { m = t[0]; M2 = t[C]; mn = t[2 * C]; mx = t[3 * C]; }
  double* o = out + (size_t)r * P * C + c;
  const unsigned long long g = first_chain + (unsigned long long)c;
  for (int i = p0; i < p0 + P; ++i, o += C) {
    double a[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < K; ++k) a[k] = run_program_t<false>(code_sa, consts_sa, ctx, es, progs.pc[k], nullptr, true, i);
    ppc::PhiloxSource src;
    src.init(seed, g, ppc::stream_position((unsigned long long)r, (unsigned long long)N, (unsigned long long)i));
    const double y = ppc::draw(family, a, src);
    *o = y;
    const double d = y - m;
    m += d / (double)(i + 1);
    M2 += d * (y - m);
    mn = i == 0 ? y : amwg::js_min(mn, y);
    mx = i == 0 ? y : amwg::js_max(mx, y);
  }
  t[0] = m;
  t[C] = last ? sqrt(M2 / (double)(N - 1)) : M2;
  t[2 * C] = mn;
  t[3 * C] = mx;
}

// K_p2. counts[entry][4] = { <, ==, > threshold, NaN }, zeroed by the caller.
__global__ void __launch_bounds__(256) amwg_threshold_counts_kernel(const double* __restrict__ x, long long rows, int E, long long C,
                                                                    const double* __restrict__ thr, unsigned long long* __restrict__ counts) {
  const int e = blockIdx.y;
  const double th = thr[e];
  unsigned long long lt = 0, eq = 0, gt = 0, nan = 0;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* q = x + (size_t)e * C + c;
    for (long long r = 0; r < rows; ++r) {
      const double v = q[(size_t)r * E * C];
      if (v != v) ++nan;
      else if (v < th) ++lt;
      else if (v == th) ++eq;
      else if (v > th) ++gt;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    lt += __shfl_xor_sync(0xffffffffu, lt, o);
    eq += __shfl_xor_sync(0xffffffffu, eq, o);
    gt += __shfl_xor_sync(0xffffffffu, gt, o);
    nan += __shfl_xor_sync(0xffffffffu, nan, o);
  }
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* ce = counts + 4 * (size_t)e;
    if (lt) atomicAdd(ce, lt);
    if (eq) atomicAdd(ce + 1, eq);
    if (gt) atomicAdd(ce + 2, gt);
    if (nan) atomicAdd(ce + 3, nan);
  }
}

}  // namespace summary

extern "C" int amwg_ppc_pointwise(amwg_sampler* s, const int32_t* host_code, int32_t n_code, const double* host_consts, int32_t n_consts,
                                  int32_t family, const int32_t* host_arg_progs, int32_t n_args, const int32_t* host_fold_prog,
                                  const int32_t* host_fold_dst, int32_t n_fold, const double* dev_samples, int64_t rows, int32_t entries,
                                  int64_t points, int64_t p0, int32_t n_points, double* dev_out, double* dev_stats) {
  const char* who = "amwg_ppc_pointwise";
  if (!s) return fail("amwg_ppc_pointwise: NULL handle");
  if (s->K) return fail("amwg_ppc_pointwise: predictive checks of tempered ladders (options.temperatures) are not supported yet");
  if (!host_code || !host_consts || !host_arg_progs || !dev_samples || !dev_out || !dev_stats || (n_fold > 0 && (!host_fold_prog || !host_fold_dst)))
    return fail("amwg_ppc_pointwise: null pointer");
  if (family < 0 || family >= ppc::kFamilies) return fail("amwg_ppc_pointwise: unknown family");
  if (n_args != ppc::arity(family)) return fail("amwg_ppc_pointwise: the family takes " + std::to_string(ppc::arity(family)) + " parameter programs");
  if (rows <= 0 || entries <= 0 || n_points <= 0 || n_code <= 0 || n_consts <= 0 || n_fold < 0) return fail("amwg_ppc_pointwise: empty program or block");
  if (p0 < 0 || points > ((int64_t)1 << 31) - 1 || p0 + n_points > points) return fail("amwg_ppc_pointwise: point range out of bounds");
  if ((double)rows * (double)points >= 70368744177664.0) return fail("amwg_ppc_pointwise: rows x points must stay below 2^46 (the stream region)");
  const size_t smem = (((size_t)n_code * 4 + 7) & ~(size_t)7) + (size_t)n_consts * 8;
  if (smem > kSmemBudget) return fail("amwg_ppc_pointwise: the program and its constants exceed the shared memory budget");
  std::vector<int> bodies(host_arg_progs, host_arg_progs + n_args);
  if (check_pointwise_programs(s, who, host_code, n_code, n_consts, bodies, host_fold_prog, host_fold_dst, n_fold, entries, p0, n_points))
    return -1;
  if (summary::select_device(s->device, who)) return -1;
  CUDA_TRY(cudaStreamSynchronize(s->stream));               // the sampler's stream wrote the block
  int* d_code = nullptr;
  double* d_consts = nullptr;
  summary::LooColumns* d_cols = nullptr;
  summary::Scratch sc;
  if (stage_pointwise_program(s, sc, who, (const void*)summary::amwg_ppc_pointwise_kernel, smem, host_code, n_code, host_consts, n_consts,
                              host_fold_prog, host_fold_dst, n_fold, &d_code, &d_consts, &d_cols))
    return -1;
  summary::PpcPrograms progs{{0, 0, 0}};
  for (int k = 0; k < n_args; ++k) progs.pc[k] = host_arg_progs[k];
  const long long C = (long long)s->a.C;
  const dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)std::min<int64_t>(rows, 65535), (unsigned)((rows + 65534) / 65535));
  summary::amwg_ppc_pointwise_kernel<<<grid, kThreads, smem>>>(d_code, n_code, d_consts, n_consts, family, n_args, progs, d_cols, dev_samples,
                                                               entries, rows, C, (unsigned long long)s->a.first_chain,
                                                               (unsigned long long)s->a.seed, points, (int)p0, n_points,
                                                               p0 + n_points == points, dev_out, dev_stats);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  s->launches += 1;
  return 0;
}

extern "C" int amwg_summary_threshold_counts(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                             const double* host_thresholds, int64_t* dev_counts) {
  if (rows <= 0 || entries <= 0 || chains <= 0) return fail("amwg_summary_threshold_counts: empty block");
  if (entries > 65535) return fail("amwg_summary_threshold_counts: at most 65535 entries per call");
  if (!dev_samples || !host_thresholds || !dev_counts) return fail("amwg_summary_threshold_counts: null pointer");
  if (summary::select_device(device, "amwg_summary_threshold_counts")) return -1;
  summary::Scratch sc;
  if (sc.acquire(device, "amwg_summary_threshold_counts", {(size_t)entries * 8})) return -1;
  double* d_thr = sc.part<double>(0);
  CUDA_TRY(cudaMemcpy(d_thr, host_thresholds, (size_t)entries * 8, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(dev_counts, 0, (size_t)entries * 4 * sizeof(int64_t)));
  const unsigned bx = (unsigned)summary::chain_ctas(chains);
  summary::amwg_threshold_counts_kernel<<<dim3(bx, (unsigned)entries), 256>>>(dev_samples, rows, entries, chains, d_thr,
                                                                              reinterpret_cast<unsigned long long*>(dev_counts));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}
