// Addressing of the Gram kernel behind amwg_summary_comoments (sample_summary(..., covariance=...)): which tiles exist, which warp
// owns each, which (row, entry, chain) every thread stages, where a lane reads its mma.sync.m8n8k4.f64 fragments and which
// elements of a tile it accumulates, and where a CTA's partial tiles go. One __host__ __device__ text, so that the kernel
// (amwg_summary.cuh) and the host-compiled emulation the CPU tests run (tests/host_shim/comoments_host.cpp) index alike.
//
// The Gram matrix G[i][j] = sum_k d[i][k] d[j][k] of n_sel centred series over k = (row, chain) is cut into 8 x 8 tiles, i and j
// in 8-entry blocks b < nb = ceil(n_sel / 8); only the upper-triangle tiles (bi <= bj) are formed. One DMMA.8x8x4 step adds
// four k (four chains of one row). Per the PTX m8n8k4 f64 layouts, lane l holds A[l >> 2][l & 3] (row-major A, 8 x 4),
// B[l & 3][l >> 2] (column-major B, 4 x 8) and C[l >> 2][2 (l & 3) + i], i < 2. With A = d of block bi and B = d^T of block bj,
// a lane's A and B fragments are both the centred value of entry 8b + (l >> 2), chain c0 + (l & 3): one staged value serves as
// the A fragment of tiles (b, .) and the B fragment of tiles (., b).
#pragma once

namespace summary {

constexpr int kMaxSel = 128;                        // entries per call: 16 blocks, 136 tiles
constexpr int kCoWarps = 16;                        // warps per CTA of the Gram kernel
constexpr int kCoThreads = 32 * kCoWarps;
constexpr int kCoSlots = ((kMaxSel / 8) * (kMaxSel / 8 + 1) / 2 + kCoWarps - 1) / kCoWarps;   // tiles per warp at n_sel = 128: ceil(136 / 16) = 9
constexpr int kCoChains = 32;                       // chains per stage (eight quads)
constexpr int kCoPitch = 36;                        // doubles per staged (row, entry): 32 chains + 4 of padding, so that the
                                                    // eight entries of a fragment read fall in distinct bank groups
constexpr int kCoStageValues = 4096;                // staged values per stage at most (8 per thread)
constexpr int kCoStageRows = kCoStageValues / (8 * kCoChains);     // rows per stage at nb = 1; nb blocks stage kCoStageRows / nb
constexpr int kCoSmem = kCoStageRows * 8 * kCoPitch;               // shared doubles of one stage, for every nb (36 KB)

__host__ __device__ __forceinline__ int co_blocks(int n_sel) { return (n_sel + 7) / 8; }
__host__ __device__ __forceinline__ int co_tiles(int nb) { return nb * (nb + 1) / 2; }
__host__ __device__ __forceinline__ int co_stage_rows(int nb) { return kCoStageRows / nb > 0 ? kCoStageRows / nb : 1; }

// tile t < co_tiles(nb) -> (bi, bj), bi <= bj, row by row of the upper triangle: (0,0) (0,1) .. (0,nb-1) (1,1) ..
__host__ __device__ __forceinline__ void co_tile(int t, int nb, int& bi, int& bj) {
  int i = 0;
  while (t >= nb - i) { t -= nb - i; ++i; }
  bi = i;
  bj = i + t;
}

// Fewer tiles than warps (n_sel <= 40): co_reps(nb) warps share each tile, rep r of them taking the steps k (k = rr * nq + q
// within a stage) with k % reps == r into an accumulator of its own, so that no warp runs a long chain of dependent DMMAs alone.
__host__ __device__ __forceinline__ int co_reps(int nb) { return co_tiles(nb) >= kCoWarps ? 1 : kCoWarps / co_tiles(nb); }

// the tile in slot s of warp w (slots are compile-time register indices), or -1: with one rep the tiles are dealt round-robin
// over the warps; with several, warp w < reps * tiles holds tile w % tiles in slot 0 as rep w / tiles
__host__ __device__ __forceinline__ int co_slot_tile(int w, int s, int nb) {
  const int tiles = co_tiles(nb), reps = co_reps(nb);
  if (reps == 1) {
    const int t = w + kCoWarps * s;
    return t < tiles ? t : -1;
  }
  return s == 0 && w < reps * tiles ? w % tiles : -1;
}
__host__ __device__ __forceinline__ int co_warp_rep(int w, int nb) { return co_reps(nb) == 1 ? 0 : w / co_tiles(nb); }

// Staged value v < stage_rows * 8nb * kCoChains of the stage at (row r0, chain c0): chain fastest, then entry slot, then row.
struct CoStageElem { int rr, s, cc; };
__host__ __device__ __forceinline__ CoStageElem co_stage_elem(int v, int nb) {
  const int per_row = 8 * nb * kCoChains;
  return CoStageElem{v / per_row, (v % per_row) / kCoChains, v % kCoChains};
}

// whether the thread staging (r0 + rr, entry slot s, chain c0 + cc) loads: slots past n_sel, rows past the block and chains
// past C stage 0 and read nothing
__host__ __device__ __forceinline__ bool co_loads(long long row, int s, long long chain, long long rows, int n_sel, long long C) {
  return s < n_sel && row < rows && chain < C;
}

// element of the block x[row][entry][chain] (entries per row, C chains) and of the centre cen[entry * cen_se + chain * cen_sc]
__host__ __device__ __forceinline__ long long co_x_index(long long row, int entry, long long chain, int entries, long long C) {
  return (row * entries + entry) * C + chain;
}
__host__ __device__ __forceinline__ long long co_cen_index(int s, long long chain, long long cen_se, long long cen_sc) {
  return s * cen_se + chain * cen_sc;
}

// shared-memory place of staged (rr, entry slot s, chain cc)
__host__ __device__ __forceinline__ int co_smem_index(int rr, int s, int cc, int nb) { return (rr * 8 * nb + s) * kCoPitch + cc; }

// The value lane `lane` feeds as fragment of block b for quad q (chains 4q .. 4q+3 of the stage) of staged row rr sits at
// co_frag_base(q, rr, nb) + co_frag_lane(lane, b) = co_smem_index(rr, 8b + (lane >> 2), 4q + (lane & 3), nb): the kernel keeps
// the lane part of each of its tiles in registers and adds the base per step.
__host__ __device__ __forceinline__ int co_frag_base(int q, int rr, int nb) { return co_smem_index(rr, 0, 4 * q, nb); }
__host__ __device__ __forceinline__ int co_frag_lane(int lane, int b) { return (8 * b + (lane >> 2)) * kCoPitch + (lane & 3); }

// element i < 2 of the accumulator a lane holds for a tile: row and column inside the 8 x 8 tile
__host__ __device__ __forceinline__ int co_acc_row(int lane, int) { return lane >> 2; }
__host__ __device__ __forceinline__ int co_acc_col(int lane, int i) { return 2 * (lane & 3) + i; }

// partial[cta][rep][tile][8][8]: where rep `rep` of CTA `cta` writes element i of its accumulator of tile t; K_c4 sums the
// cta * reps + rep records in that order
__host__ __device__ __forceinline__ long long co_partial_index(long long cta, int rep, int t, int nb, int lane, int i) {
  return (((cta * co_reps(nb) + rep) * co_tiles(nb) + t) * 8 + co_acc_row(lane, i)) * 8 + co_acc_col(lane, i);
}

// CTAs of the Gram kernel: one per 32-chain group, at most kCoCtas (two waves of one CTA per SM on an H100 SXM). A function of the
// chain count only, never of the device, because it sets the order in which the partial tiles are summed and so their last bits.
constexpr long long kCoCtas = 264;
__host__ __device__ __forceinline__ long long co_ctas(long long C) {
  const long long g = (C + kCoChains - 1) / kCoChains;
  return g < kCoCtas ? g : kCoCtas;
}

}  // namespace summary
