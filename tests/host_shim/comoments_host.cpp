// Test infrastructure: the covariance reduction of amwg_summary_comoments run on the HOST with the kernels' addressing
// (csrc/amwg_comoments.cuh, the text the Gram kernel indexes with) and a scalar emulation of mma.sync.m8n8k4.f64 over 32
// emulated lanes in the PTX fragment layouts, for tests/test_summary_covariance_host.py. Every global, shared and partial index
// the schedule forms is checked against its buffer, and every fragment read against what was staged; hs_comoments returns the
// number of violations. Build with -ffp-contract=off, as the library is built with --fmad=false.
#include "cuda_runtime.h"
#include "amwg_comoments.cuh"

#include <cmath>
#include <vector>

using namespace summary;

namespace {

long long g_bad = 0;
inline void check(bool ok) { if (!ok) ++g_bad; }

// D = A B + C for one DMMA.8x8x4: lane l holds A[l >> 2][l & 3] in a[l], B[l & 3][l >> 2] in b[l] and C[l >> 2][2 (l & 3) + i] in
// c[l][i]; each output element adds its four products in k order, one rounding per fma
void mma_m8n8k4(double (*c)[2], const double* a, const double* b) {
  for (int l = 0; l < 32; ++l)
    for (int i = 0; i < 2; ++i) {
      const int m = co_acc_row(l, i), n = co_acc_col(l, i);
      double d = c[l][i];
      for (int k = 0; k < 4; ++k) d = std::fma(a[4 * m + k], b[4 * n + k], d);
      c[l][i] = d;
    }
}

// K_c3 + K_c4 with the kernel's grid, stages, warps, reps, slots and partial layout: out[tile][64] (tile-major, 8 x 8 row-major)
void gram(const double* x, long long x_len, long long rows, int entries, long long C, const int* sel, int n_sel, const double* cen,
          long long cen_len, long long cen_se, long long cen_sc, std::vector<double>& out) {
  const int nb = co_blocks(n_sel), n_tiles = co_tiles(nb), srows = co_stage_rows(nb), reps = co_reps(nb);
  const int per_stage = srows * 8 * nb * kCoChains;
  check(per_stage <= kCoStageValues);
  const long long gx = co_ctas(C);
  std::vector<double> partial((size_t)gx * reps * n_tiles * 64, NAN);
  std::vector<int> writes(partial.size(), 0);
  std::vector<double> st(kCoSmem);
  std::vector<char> staged(kCoSmem);
  for (long long cta = 0; cta < gx; ++cta) {
    std::vector<double> acc((size_t)kCoWarps * kCoSlots * 32 * 2, 0.0);
    for (long long g = cta; g * kCoChains < C; g += gx) {
      const long long c0 = g * kCoChains;
      const int nq = (int)((C - c0 < kCoChains ? C - c0 + 3 : kCoChains) / 4);
      for (long long r0 = 0; r0 < rows; r0 += srows) {
        std::fill(staged.begin(), staged.end(), 0);
        for (int thread = 0; thread < kCoThreads; ++thread)
          for (int u = 0; u < kCoStageValues / kCoThreads; ++u) {
            const int i = thread + u * kCoThreads;
            if (i >= per_stage) continue;
            const CoStageElem el = co_stage_elem(i, nb);
            const long long r = r0 + el.rr, c = c0 + el.cc;
            double v = 0.0;
            if (co_loads(r, el.s, c, rows, n_sel, C)) {
              check(el.s >= 0 && el.s < n_sel && sel[el.s] >= 0 && sel[el.s] < entries && r >= 0 && c >= 0);
              const long long xi = co_x_index(r, sel[el.s], c, entries, C), ci = co_cen_index(el.s, c, cen_se, cen_sc);
              check(xi >= 0 && xi < x_len);
              check(ci >= 0 && ci < cen_len);
              if (xi >= 0 && xi < x_len && ci >= 0 && ci < cen_len) v = x[xi] - cen[ci];
            }
            const int si = co_smem_index(el.rr, el.s, el.cc, nb);
            check(si >= 0 && si < kCoSmem);
            if (si >= 0 && si < kCoSmem) { check(!staged[si]); st[si] = v; staged[si] = 1; }
          }
        const int nr = (int)(rows - r0 < srows ? rows - r0 : srows);
        for (int w = 0; w < kCoWarps; ++w)
          for (int k = co_warp_rep(w, nb); k < nr * nq; k += reps) {
            const int base = co_frag_base(k % nq, k / nq, nb);
            for (int s = 0; s < kCoSlots; ++s) {
              const int t = co_slot_tile(w, s, nb);
              if (t < 0) continue;
              int bi = 0, bj = 0;
              co_tile(t, nb, bi, bj);
              check(bi <= bj && bj < nb);
              double a[32], b[32];
              for (int l = 0; l < 32; ++l) {
                const int ia = base + co_frag_lane(l, bi), ib = base + co_frag_lane(l, bj);
                check(ia >= 0 && ia < kCoSmem && ib >= 0 && ib < kCoSmem);
                const bool ok = ia >= 0 && ia < kCoSmem && ib >= 0 && ib < kCoSmem;
                if (ok) check(staged[ia] && staged[ib]);
                a[l] = ok ? st[ia] : NAN;
                b[l] = ok ? st[ib] : NAN;
              }
              mma_m8n8k4(reinterpret_cast<double(*)[2]>(&acc[(((size_t)w * kCoSlots + s) * 32) * 2]), a, b);
            }
          }
      }
    }
    for (int w = 0; w < kCoWarps; ++w)
      for (int s = 0; s < kCoSlots; ++s) {
        const int t = co_slot_tile(w, s, nb);
        if (t < 0) continue;
        for (int l = 0; l < 32; ++l)
          for (int i = 0; i < 2; ++i) {
            const long long pi = co_partial_index(cta, co_warp_rep(w, nb), t, nb, l, i);
            check(pi >= 0 && pi < (long long)partial.size());
            if (pi >= 0 && pi < (long long)partial.size()) { partial[pi] = acc[(((size_t)w * kCoSlots + s) * 32 + l) * 2 + i]; ++writes[pi]; }
          }
      }
  }
  for (int wcount : writes) check(wcount == 1);                  // every partial element written exactly once
  const int n_vals = n_tiles * 64;
  out.assign(n_vals, 0.0);
  for (int v = 0; v < n_vals; ++v) {
    double a = 0.0;
    for (long long k = 0; k < gx * reps; ++k) a += partial[(size_t)k * n_vals + v];
    out[v] = a;
  }
}

}  // namespace

extern "C" {
// out[1 + n + 2 n^2] = { C, m, B, W } as amwg_summary_comoments forms it; -> the number of out-of-range or unstaged indices
long long hs_comoments(const double* x, long long rows, int entries, long long C, const int* sel, int n_sel, double* out) {
  g_bad = 0;
  const long long x_len = rows * entries * C;
  std::vector<double> xbar((size_t)n_sel * C), m(n_sel);
  for (int s = 0; s < n_sel; ++s)
    for (long long c = 0; c < C; ++c) {
      double sum = 0.0;
      for (long long r = 0; r < rows; ++r) sum += x[co_x_index(r, sel[s], c, entries, C)];
      xbar[(size_t)s * C + c] = sum / (double)rows;
    }
  for (int s = 0; s < n_sel; ++s) {
    double sum = 0.0;
    for (long long c = 0; c < C; ++c) sum += xbar[(size_t)s * C + c];
    m[s] = sum / (double)C;
  }
  std::vector<int> ident(n_sel);
  for (int i = 0; i < n_sel; ++i) ident[i] = i;
  std::vector<double> tw, tb;
  gram(x, x_len, rows, entries, C, sel, n_sel, xbar.data(), (long long)xbar.size(), C, 1, tw);
  gram(xbar.data(), (long long)xbar.size(), 1, n_sel, C, ident.data(), n_sel, m.data(), n_sel, 1, 0, tb);
  const int nb = co_blocks(n_sel), n = n_sel;
  double* oB = out + 1 + n;
  double* oW = oB + (size_t)n * n;
  out[0] = (double)C;
  for (int i = 0; i < n; ++i) out[1 + i] = m[i];
  for (int t = 0; t < co_tiles(nb); ++t) {
    int bi = 0, bj = 0;
    co_tile(t, nb, bi, bj);
    for (int r = 0; r < 8; ++r)
      for (int c = 0; c < 8; ++c) {
        const int i = 8 * bi + r, j = 8 * bj + c;
        if (i > j || j >= n) continue;
        oW[(size_t)i * n + j] = oW[(size_t)j * n + i] = tw[(size_t)t * 64 + r * 8 + c];
        oB[(size_t)i * n + j] = oB[(size_t)j * n + i] = tb[(size_t)t * 64 + r * 8 + c];
      }
  }
  return g_bad;
}
}
