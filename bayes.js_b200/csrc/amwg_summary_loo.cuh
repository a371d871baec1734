// PSIS-LOO and WAIC in sample_summary(..., loo=...) (DESIGN.md §4.7): the pointwise log-likelihood ll[row][point][chain] of
// every kept draw, formed where the draws are, and the per-point reductions that the base summary kernels do not already give.
//   K_l0  amwg_loo_fold_kernel      : the body's constant sub-expressions, folded on the device as amwg_fold_kernel folds the
//                                     model's (same interpreter, one thread)
//   K_l1  amwg_loo_pointwise_kernel : one thread per (row, chain) over a chunk of points: the traced log_lik body, run by the
//                                     model's interpreter (run_program_t) entered at the point index, on the draw's column of the
//                                     sample block. Writes coalesced over chains: the sample-block layout with points as entries.
//   K_l2  amwg_loo_reduce_kernel    : one pass over the chunk per (chain group, point): sum exp(ll - llmax) over all draws and
//                                     sum exp(lw), sum exp(lw + ll - llmin) over the draws outside the Pareto tail
//                                     (lw = llmin - ll <= cut), fixed CTA trees then amwg_merge_sums_kernel; the tail draws' ll
//                                     appended to the point's tail buffer through a slot counter (their order does not matter:
//                                     K_l3 sorts them)
//   K_l3  amwg_loo_fit_kernel       : one CTA per point: the shards' tails gathered and sorted (bitonic, in global scratch), the
//                                     generalised Pareto fit of amwg_loo.cuh, the smoothed tail weights and their two sums
// Included at the end of amwg_kernels.cu, after amwg_summary.cuh (cta_sum, amwg_merge_sums_kernel, kChainCtas).
#pragma once

#include "amwg_loo.cuh"

namespace summary {

constexpr int kFitThreads = 512;

struct LooColumns { const double* col[kMaxColumns]; };

// K_l0: the fold programs, in order (later folds may use earlier ones), into the constants in global memory: one thread, as
// amwg_fold_kernel folds the model's. A fold program may read data at a fixed index (DATA: a parameter-free `data.s[0]`), so the
// data columns are set up as for K_l1. Dynamic shared memory as K_l1's.
__global__ void amwg_loo_fold_kernel(const int* __restrict__ code, int n_code, double* __restrict__ consts, int n_consts,
                                     const int* __restrict__ fold_prog, const int* __restrict__ fold_dst, int n_fold,
                                     const LooColumns* __restrict__ cols) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ Ctx ctx;
  int* s_code = reinterpret_cast<int*>(smem);
  double* s_consts = reinterpret_cast<double*>(smem + (((unsigned)n_code * 4u + 7u) & ~7u));
  for (int i = 0; i < n_code; ++i) s_code[i] = code[i];
  for (int i = 0; i < n_consts; ++i) s_consts[i] = consts[i];
  for (int k = 0; k < kMaxColumns; ++k) ctx.col[k] = cols->col[k];
  EvalStateT<false> none{nullptr, 0, -1, 0.0};
  for (int k = 0; k < n_fold; ++k) {
    const double v = run_program_t<false>(smem_u32(s_code), smem_u32(s_consts), ctx, none, fold_prog[k], nullptr, true);
    s_consts[fold_dst[k]] = v;
    consts[fold_dst[k]] = v;
  }
}

// K_l1. Dynamic shared memory: the program words (padded to 8 bytes), then the folded constants.
__global__ void __launch_bounds__(kThreads) amwg_loo_pointwise_kernel(const int* __restrict__ code, int n_code, const double* __restrict__ consts,
                                                                      int n_consts, int body_pc, const LooColumns* __restrict__ cols,
                                                                      const double* __restrict__ x, int entries, long long rows, long long C,
                                                                      int p0, int P, double* __restrict__ out) {
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
  double* o = out + (size_t)r * P * C + c;
  const double* const end = o + (size_t)P * C;
  for (int i = p0; o != end; o += C, ++i) *o = run_program_t<false>(code_sa, consts_sa, ctx, es, body_pc, nullptr, true, i);
}

// K_l2. Grid (chain groups, points). partial[point][3][gridDim.x]; tail[point][cap], count[point] (zeroed by the caller).
__global__ void __launch_bounds__(256) amwg_loo_reduce_kernel(const double* __restrict__ x, long long rows, int P, long long C,
                                                              const double* __restrict__ llmin, const double* __restrict__ llmax,
                                                              const double* __restrict__ cut, int cap, double* __restrict__ tail,
                                                              int* __restrict__ count, double* __restrict__ partial) {
  __shared__ double sh[256];
  const int p = blockIdx.y;
  const double mn = llmin[p], mx = llmax[p], ct = cut[p];
  const size_t stride = (size_t)P * C;
  double s_all = 0.0, s_w = 0.0, s_wl = 0.0;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const double* q = x + (size_t)p * C + c;
    for (long long r = 0; r < rows; ++r) {
      const double v = q[r * stride];
      s_all += exp(v - mx);
      const double lw = mn - v;                         // the reference's lw, in the same fp64 operation
      if (lw > ct) {
        const int slot = atomicAdd(&count[p], 1);
        if (slot < cap) tail[(size_t)p * cap + slot] = v;
      } else {
        s_w += exp(lw);
        s_wl += exp((lw + v) - mn);
      }
    }
  }
  const double a = cta_sum<256>(sh, s_all), b = cta_sum<256>(sh, s_w), d = cta_sum<256>(sh, s_wl);
  if (threadIdx.x == 0) {
    partial[((size_t)p * 3 + 0) * gridDim.x + blockIdx.x] = a;
    partial[((size_t)p * 3 + 1) * gridDim.x + blockIdx.x] = b;
    partial[((size_t)p * 3 + 2) * gridDim.x + blockIdx.x] = d;
  }
}

// K_l3. One CTA per point. tails[shard][point][cap] with counts[shard][point]; work and xs: [point][cap] scratch, cap a power of two.
// out[point][4] = { k (+inf for a tail of <= 4 draws or one where no candidate of the fit has a finite profile value, NaN for a
// skipped point), sum exp(lw), sum exp(lw + ll - llmin) over the
// tail with lw smoothed when k is finite, the number of tail draws over all shards }.
__global__ void __launch_bounds__(kFitThreads) amwg_loo_fit_kernel(const double* __restrict__ tails, const int* __restrict__ counts, int shards,
                                                                   int P, int cap, const double* __restrict__ llmin, const double* __restrict__ cut,
                                                                   const int* __restrict__ skip, double* __restrict__ work, double* __restrict__ xs,
                                                                   double* __restrict__ out) {
  __shared__ double sh[kFitThreads];
  __shared__ double sb[loo::kMaxM], sL[loo::kMaxM], sw[loo::kMaxM];
  __shared__ double s_bp;
  const int p = blockIdx.x, t = threadIdx.x, T = blockDim.x;
  double* a = work + (size_t)p * cap;
  double* xp = xs + (size_t)p * cap;
  long long total = 0;
  for (int r = 0; r < shards; ++r) {
    const long long cnt = counts[(size_t)r * P + p];
    const long long have = cnt < cap ? cnt : cap;
    for (long long i = t; i < have; i += T)
      if (total + i < cap) a[total + i] = tails[((size_t)r * P + p) * cap + i];
    total += cnt;
  }
  const int n = (int)(total < cap ? total : cap);
  if (skip[p]) {
    if (t == 0) { out[4 * p] = CUDART_NAN; out[4 * p + 1] = CUDART_NAN; out[4 * p + 2] = CUDART_NAN; out[4 * p + 3] = (double)total; }
    return;
  }
  for (int i = n + t; i < cap; i += T) a[i] = -CUDART_INF;
  __syncthreads();
  for (int k = 2; k <= cap; k <<= 1) {                        // bitonic sort, descending ll = ascending lw
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < cap; i += T) {
        const int l = i ^ j;
        if (l > i) {
          const double ai = a[i], al = a[l];
          if ((i & k) == 0 ? (ai < al) : (ai > al)) { a[i] = al; a[l] = ai; }
        }
      }
      __syncthreads();
    }
  }
  const double mn = llmin[p], ct = cut[p], expcut = exp(ct);
  double k = CUDART_INF, sigma = CUDART_NAN;
  if (n > 4) {
    for (int i = t; i < n; i += T) xp[i] = exp(mn - a[i]) - expcut;
    __syncthreads();
    const int m = loo::fit_m(n);
    const double xq = xp[loo::fit_quartile(n)], xmax = xp[n - 1];
    const int warp = t >> 5, lane = t & 31;
    for (int j = warp; j < m; j += T >> 5) {                  // one warp per candidate: lanes stride the tail, then a fixed shuffle tree
      const double b = loo::fit_b(j + 1, m, xq, xmax);
      double s = 0.0;
      for (int i = lane; i < n; i += 32) s += loo::fit_term(b, xp[i]);
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) { sb[j] = b; sL[j] = loo::fit_profile(n, b, s / (double)n); }
    }
    __syncthreads();
    for (int j = t; j < m; j += T) sw[j] = loo::fit_weight(sL, m, j);
    __syncthreads();
    if (t == 0) s_bp = loo::fit_b_post(sb, sw, m);
    __syncthreads();
    const double bp = s_bp;
    if (bp == bp) {                                           // NaN: no candidate with a finite profile value, k stays +inf
      double s = 0.0;
      for (int i = t; i < n; i += T) s += loo::fit_term(bp, xp[i]);
      const double kh = cta_sum<kFitThreads>(sh, s) / (double)n;
      sigma = -kh / bp;
      k = loo::fit_prior_k(kh, n);
    }
  }
  const bool smooth = isfinite(k);
  double s_w = 0.0, s_wl = 0.0;
  for (int i = t; i < n; i += T) {
    const double lw = smooth ? loo::smoothed(i, n, k, sigma, expcut) : mn - a[i];
    s_w += exp(lw);
    s_wl += exp((lw + a[i]) - mn);
  }
  const double tw = cta_sum<kFitThreads>(sh, s_w), twl = cta_sum<kFitThreads>(sh, s_wl);
  if (t == 0) { out[4 * p] = k; out[4 * p + 1] = tw; out[4 * p + 2] = twl; out[4 * p + 3] = (double)total; }
}

// per-device scratch that lives as long as the process, grown on demand (as amwg_summary_moments')
struct LooScratch { void* p = nullptr; size_t bytes = 0; };
inline int loo_scratch(int device, size_t need, void** out, const char* who) {
  static LooScratch pool[64];
  if (device < 0 || device >= 64) return fail(std::string(who) + ": device index out of range");
  LooScratch& sc = pool[device];
  if (sc.bytes < need) {
    if (sc.p) cudaFree(sc.p);
    sc.p = nullptr; sc.bytes = 0;
    CUDA_TRY(cudaMalloc(&sc.p, need));
    sc.bytes = need;
  }
  *out = sc.p;
  return 0;
}

}  // namespace summary

static std::mutex g_loo_mu;               // the calls below share one scratch pool per device

// The checks of amwg_loo_pointwise and amwg_ppc_pointwise, before anything runs: every program well formed and an expression (no
// sum, plate, loop, store or cache word), each index inside its table and, for the body programs `bodies`, each data read inside
// its column at every point of p0 .. p0 + n_points - 1; each program leaves one value.
static int check_pointwise_programs(amwg_sampler* s, const char* who, const int32_t* host_code, int32_t n_code, int32_t n_consts,
                                    const std::vector<int>& bodies, const int32_t* host_fold_prog, const int32_t* host_fold_dst,
                                    int32_t n_fold, int32_t entries, int64_t p0, int32_t n_points) {
  amwg_model md{};
  md.code = host_code; md.n_code = n_code;
  std::vector<int> progs(bodies);
  const size_t n_bodies = bodies.size();
  for (int k = 0; k < n_fold; ++k) {
    if (host_fold_dst[k] < 0 || host_fold_dst[k] >= n_consts) return fail(std::string(who) + ": constant-folding table out of range");
    progs.push_back(host_fold_prog[k]);
  }
  const int64_t p1 = p0 + n_points - 1;
  for (size_t q = 0; q < progs.size(); ++q) {
    const bool fold = q >= n_bodies;
    std::vector<jit::Insn> ins;
    std::string err;
    int depth = 0;
    if (!jit::decode_program(&md, progs[q], ins, &depth, err)) return fail(std::string(who) + ": malformed program: " + err);
    if (depth > kStack) return fail(std::string(who) + ": the program nests deeper than the device's operand stack");
    int left = 0;
    for (const jit::Insn& in : ins) {
      left += in.pushes - in.pops;
      if (in.acc || in.store) return fail(std::string(who) + ": the program must be an expression");
      for (int k = 0; k < 4; ++k) {
        if (in.mode[k] == AMWG_MODE_CONST && (in.inl[k] < 0 || in.inl[k] >= n_consts)) return fail(std::string(who) + ": constant index out of range");
        if (in.mode[k] == AMWG_MODE_COMP && (fold || in.inl[k] < 0 || in.inl[k] >= entries)) return fail(std::string(who) + ": entry index out of range");
      }
      switch (in.op) {
        case AMWG_OP_END: break;
        case AMWG_OP_CONST: if (in.a >= n_consts) return fail(std::string(who) + ": constant index out of range"); break;
        case AMWG_OP_COMP: if (fold || in.a >= entries) return fail(std::string(who) + ": entry index out of range"); break;
        case AMWG_OP_DATA:
          if (in.a >= (int)s->col_n.size() || in.extra[0] < 0 || in.extra[0] >= s->col_n[in.a]) return fail(std::string(who) + ": data index out of range");
          break;
        case AMWG_OP_DATA_I: case AMWG_OP_COMP_I: {
          if (fold || in.a >= (int)s->col_n.size()) return fail(std::string(who) + ": data column out of range");
          const int64_t off = in.extra[0], stride = in.extra[1], lo = off + stride * p0, hi = off + stride * p1, n = s->col_n[in.a];
          if (lo < 0 || lo >= n || hi < 0 || hi >= n) return fail(std::string(who) + ": a point index runs past the end of a data column");
          if (in.op == AMWG_OP_COMP_I) {                     // entries[base + data[i]] must stay inside the block's entries
            std::vector<double> col((size_t)n);
            CUDA_TRY(cudaSetDevice(s->device));
            CUDA_TRY(cudaMemcpy(col.data(), s->m.col_global[in.a], (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
            for (int64_t i = p0; i <= p1; ++i) {
              const double v = col[(size_t)(off + stride * i)];
              if (!(v == std::floor(v)) || in.extra[2] + v < 0 || in.extra[2] + v >= entries)
                return fail(std::string(who) + ": the program indexes the block's entries with a data value outside them");
            }
          }
          break;
        }
        case AMWG_OP_ACC: case AMWG_OP_ACC_RANGE: case AMWG_OP_PLATE: case AMWG_OP_PLATE_SS: case AMWG_OP_NORM_SS: case AMWG_OP_CACHED:
        case AMWG_OP_CAND: case AMWG_OP_STORE: case AMWG_OP_LOOP_BEGIN: case AMWG_OP_LOOP_END:
          return fail(std::string(who) + ": the program must be an expression");
        default: break;
      }
    }
    if (left != 1) return fail(std::string(who) + ": the program must leave exactly one value");
  }
  return 0;
}

// Copies the checked program, its constants, the fold table and the handle's data column pointers into the per-device pool and
// folds the constants on the device (K_l0), for a pointwise kernel with `smem` bytes of dynamic shared memory. The caller holds
// g_loo_mu and has selected the handle's device.
static int stage_pointwise_program(amwg_sampler* s, const char* who, const void* kernel, size_t smem, const int32_t* host_code,
                                   int32_t n_code, const double* host_consts, int32_t n_consts, const int32_t* host_fold_prog,
                                   const int32_t* host_fold_dst, int32_t n_fold, int** d_code_out, double** d_consts_out,
                                   summary::LooColumns** d_cols_out) {
  const size_t b_code = ((size_t)n_code * 4 + 15) & ~(size_t)15, b_consts = ((size_t)n_consts * 8 + 15) & ~(size_t)15;
  const size_t b_fold = (((size_t)std::max(n_fold, 1) * 4) + 15) & ~(size_t)15;
  void* base = nullptr;
  const size_t b_cols = (sizeof(summary::LooColumns) + 15) & ~(size_t)15;
  if (summary::loo_scratch(s->device, b_code + b_consts + 2 * b_fold + b_cols, &base, who)) return -1;
  char* cb = reinterpret_cast<char*>(base);
  int* d_code = reinterpret_cast<int*>(cb);
  double* d_consts = reinterpret_cast<double*>(cb + b_code);
  int* d_fp = reinterpret_cast<int*>(cb + b_code + b_consts);
  int* d_fd = reinterpret_cast<int*>(cb + b_code + b_consts + b_fold);
  auto* d_cols = reinterpret_cast<summary::LooColumns*>(cb + b_code + b_consts + 2 * b_fold);
  CUDA_TRY(cudaMemcpy(d_code, host_code, (size_t)n_code * 4, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_consts, host_consts, (size_t)n_consts * 8, cudaMemcpyHostToDevice));
  if (n_fold > 0) {
    CUDA_TRY(cudaMemcpy(d_fp, host_fold_prog, (size_t)n_fold * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(d_fd, host_fold_dst, (size_t)n_fold * 4, cudaMemcpyHostToDevice));
  }
  summary::LooColumns cols{};
  for (int k = 0; k < (int)s->col_n.size(); ++k) cols.col[k] = s->m.col_global[k];
  CUDA_TRY(cudaMemcpy(d_cols, &cols, sizeof cols, cudaMemcpyHostToDevice));
  if (smem > 48 * 1024) {
    CUDA_TRY(cudaFuncSetAttribute(summary::amwg_loo_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  if (n_fold > 0) summary::amwg_loo_fold_kernel<<<1, 1, smem>>>(d_code, n_code, d_consts, n_consts, d_fp, d_fd, n_fold, d_cols);
  *d_code_out = d_code; *d_consts_out = d_consts; *d_cols_out = d_cols;
  return 0;
}

extern "C" int amwg_loo_pointwise(amwg_sampler* s, const int32_t* host_code, int32_t n_code, const double* host_consts, int32_t n_consts,
                                  int32_t body_prog, const int32_t* host_fold_prog, const int32_t* host_fold_dst, int32_t n_fold,
                                  const double* dev_samples, int64_t rows, int32_t entries, int64_t p0, int32_t n_points, double* dev_out) {
  const char* who = "amwg_loo_pointwise";
  if (!s) return fail("amwg_loo_pointwise: NULL handle");
  if (!host_code || !host_consts || !dev_samples || !dev_out || (n_fold > 0 && (!host_fold_prog || !host_fold_dst)))
    return fail("amwg_loo_pointwise: null pointer");
  if (rows <= 0 || entries <= 0 || n_points <= 0 || n_code <= 0 || n_consts <= 0 || n_fold < 0) return fail("amwg_loo_pointwise: empty program or block");
  if (p0 < 0 || p0 + n_points > ((int64_t)1 << 31) - 1) return fail("amwg_loo_pointwise: point range out of bounds");
  const size_t smem = (((size_t)n_code * 4 + 7) & ~(size_t)7) + (size_t)n_consts * 8;
  if (smem > kSmemBudget) return fail("amwg_loo_pointwise: the program and its constants exceed the shared memory budget");
  if (check_pointwise_programs(s, who, host_code, n_code, n_consts, {body_prog}, host_fold_prog, host_fold_dst, n_fold, entries, p0, n_points))
    return -1;
  std::lock_guard<std::mutex> lock(g_loo_mu);
  CUDA_TRY(cudaSetDevice(s->device));
  CUDA_TRY(cudaStreamSynchronize(s->stream));               // the sampler's stream wrote the block
  int* d_code = nullptr;
  double* d_consts = nullptr;
  summary::LooColumns* d_cols = nullptr;
  if (stage_pointwise_program(s, who, (const void*)summary::amwg_loo_pointwise_kernel, smem, host_code, n_code, host_consts, n_consts,
                              host_fold_prog, host_fold_dst, n_fold, &d_code, &d_consts, &d_cols))
    return -1;
  const long long C = (long long)s->a.C;
  const dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)std::min<int64_t>(rows, 65535), (unsigned)((rows + 65534) / 65535));
  summary::amwg_loo_pointwise_kernel<<<grid, kThreads, smem>>>(d_code, n_code, d_consts, n_consts, body_prog, d_cols, dev_samples, entries, rows,
                                                               C, (int)p0, n_points, dev_out);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  s->launches += 1;
  return 0;
}

extern "C" int amwg_loo_reduce(int device, const double* dev_ll, int64_t rows, int32_t points, int64_t chains, const double* host_llmin,
                               const double* host_llmax, const double* host_cut, int32_t tail_cap, double* dev_tail, int32_t* dev_count,
                               double* host_sums) {
  if (rows <= 0 || points <= 0 || chains <= 0) return fail("amwg_loo_reduce: empty block");
  if (points > 65535) return fail("amwg_loo_reduce: at most 65535 points per call");
  if (tail_cap < 1 || tail_cap > loo::kMaxTail) return fail("amwg_loo_reduce: tail_cap must be 1.." + std::to_string(loo::kMaxTail));
  if (!dev_ll || !host_llmin || !host_llmax || !host_cut || !dev_tail || !dev_count || !host_sums) return fail("amwg_loo_reduce: null pointer");
  std::lock_guard<std::mutex> lock(g_loo_mu);
  CUDA_TRY(cudaSetDevice(device));
  const unsigned bx = (unsigned)std::min<int64_t>((chains + 255) / 256, summary::kChainCtas);     // depends on `chains` only: a fixed merge order
  auto up = [](size_t b) { return ((b + 255) / 256) * 256; };
  const size_t b_vec = up((size_t)points * 8), b_part = up((size_t)points * 3 * bx * 8), b_sums = up((size_t)points * 3 * 8);
  void* base = nullptr;
  if (summary::loo_scratch(device, 3 * b_vec + b_part + b_sums, &base, "amwg_loo_reduce")) return -1;
  char* cb = reinterpret_cast<char*>(base);
  double* d_min = reinterpret_cast<double*>(cb);
  double* d_max = reinterpret_cast<double*>(cb + b_vec);
  double* d_cut = reinterpret_cast<double*>(cb + 2 * b_vec);
  double* d_part = reinterpret_cast<double*>(cb + 3 * b_vec);
  double* d_sums = reinterpret_cast<double*>(cb + 3 * b_vec + b_part);
  CUDA_TRY(cudaMemcpy(d_min, host_llmin, (size_t)points * 8, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_max, host_llmax, (size_t)points * 8, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_cut, host_cut, (size_t)points * 8, cudaMemcpyHostToDevice));
  summary::amwg_loo_reduce_kernel<<<dim3(bx, (unsigned)points), 256>>>(dev_ll, rows, points, chains, d_min, d_max, d_cut, tail_cap, dev_tail,
                                                                       dev_count, d_part);
  summary::amwg_merge_sums_kernel<<<(unsigned)points * 3, 256>>>(d_part, (int)bx, d_sums);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpy(host_sums, d_sums, (size_t)points * 3 * 8, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int amwg_loo_fit(int device, const double* dev_tails, const int32_t* dev_counts, int32_t shards, int32_t points, int32_t tail_cap,
                            const double* host_llmin, const double* host_cut, const int32_t* host_skip, double* host_out) {
  if (shards < 1 || points < 1) return fail("amwg_loo_fit: shards and points must be >= 1");
  if (tail_cap < 8 || tail_cap > loo::kMaxTail || (tail_cap & (tail_cap - 1))) return fail("amwg_loo_fit: tail_cap must be a power of two in 8.." + std::to_string(loo::kMaxTail));
  if (!dev_tails || !dev_counts || !host_llmin || !host_cut || !host_skip || !host_out) return fail("amwg_loo_fit: null pointer");
  std::lock_guard<std::mutex> lock(g_loo_mu);
  CUDA_TRY(cudaSetDevice(device));
  auto up = [](size_t b) { return ((b + 255) / 256) * 256; };
  const size_t b_vec = up((size_t)points * 8), b_work = up((size_t)points * tail_cap * 8), b_out = up((size_t)points * 4 * 8);
  void* base = nullptr;
  if (summary::loo_scratch(device, 3 * b_vec + 2 * b_work + b_out, &base, "amwg_loo_fit")) return -1;
  char* cb = reinterpret_cast<char*>(base);
  double* d_min = reinterpret_cast<double*>(cb);
  double* d_cut = reinterpret_cast<double*>(cb + b_vec);
  int* d_skip = reinterpret_cast<int*>(cb + 2 * b_vec);
  double* d_work = reinterpret_cast<double*>(cb + 3 * b_vec);
  double* d_xs = reinterpret_cast<double*>(cb + 3 * b_vec + b_work);
  double* d_out = reinterpret_cast<double*>(cb + 3 * b_vec + 2 * b_work);
  CUDA_TRY(cudaMemcpy(d_min, host_llmin, (size_t)points * 8, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_cut, host_cut, (size_t)points * 8, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_skip, host_skip, (size_t)points * 4, cudaMemcpyHostToDevice));
  summary::amwg_loo_fit_kernel<<<(unsigned)points, summary::kFitThreads>>>(dev_tails, dev_counts, shards, points, tail_cap, d_min, d_cut, d_skip,
                                                                          d_work, d_xs, d_out);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpy(host_out, d_out, (size_t)points * 4 * 8, cudaMemcpyDeviceToHost));
  return 0;
}
