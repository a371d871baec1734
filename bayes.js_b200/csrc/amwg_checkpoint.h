// amwg_checkpoint.h -- checkpoint images of a sampler handle (amwg_checkpoint_*, DESIGN.md §2 "Checkpoints"), and the model
// fingerprint that ties an image to the model it was taken with (amwg_model_fingerprint).
//
// Plain C++ (no CUDA): amwg_kernels.cu does the device copies around it, and tests/host_shim/checkpoint_host.cpp compiles this very
// file with g++ so that the layout, the checks and the assembly from several images are tested without a GPU. Everything here
// works on host bytes; every multi-byte field is little-endian and read with memcpy, so no alignment is assumed.
//
// Image layout, version 1 (C chains of a handle, D components, P named parameters):
//   offset      bytes   field
//   0           8       magic "AMWGCKPT"
//   8           4       u32 format version (1)
//   12          4       u32 P
//   16          4       u32 D
//   20          4       u32 K: 0, or the rungs per ladder of a tempered handle (amwg_set_ladder, 2..256)
//   24          8       u64 model fingerprint
//   32          8       u64 seed
//   40          8       u64 first_chain (global id of the image's first chain)
//   48          8       u64 C
//   56          24*D    per component: u64 is_adapting (0 or 1), f64 iterations since adaptation, f64 batch count
//   H = 56+24D  8*D*C   state            f64 [D][C]   (chain fastest, in every array)
//               8*D*C   prop_log_scale   f64 [D][C]
//               8*C     perm             u64 [C]      (P <= 16 only: the substepper order, 4 bits per named parameter)
//               8*C     rng_n            u64 [C]      (stream position: Math.random() calls consumed)
//               4*D*C   acceptance count i32 [D][C]
//               P*C     perm_ext         u8  [P][C]   (P > 16 only: the substepper order, one byte per named parameter)
//               8*K     beta             f64 [K]      (K > 0 only: the ladder; first_chain and C are multiples of K)
//               8       rounds           u64          (K > 0 only: swap rounds performed)
//               8*(C/K)*(K-1)  accepts   u64 [C/K][K-1] (K > 0 only: accepted swaps per ladder and rung pair)
//   end         8       u64 checksum (checksum() below) of bytes [0, end)
// Per chain: 20*D + 16 bytes when P <= 16, 20*D + 8 + P when P > 16. An untempered image (K = 0) is the same bytes as before the
// ladder section existed.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/amwg.h"

namespace amwg {
namespace ckpt {

constexpr char kMagic[8] = {'A', 'M', 'W', 'G', 'C', 'K', 'P', 'T'};
constexpr uint32_t kVersion = 1;
constexpr uint64_t kHashBasis = 0xcbf29ce484222325ull;   // FNV-1a's offset basis and prime, applied to 64-bit words
constexpr uint64_t kHashPrime = 0x100000001b3ull;

// ---- the 64-bit word hash of checksums and fingerprints ------------------------------------------------------------------------
// h <- (h xor w) * prime for every 64-bit little-endian word w. Each step is a bijection of h for a fixed w, so two inputs of the
// same length that differ in exactly one word (in particular by any change within one byte) always give different hashes.
inline uint64_t mix(uint64_t h, uint64_t w) { return (h ^ w) * kHashPrime; }
inline uint64_t load_u64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
// n bytes: the byte count, then the bytes as words, the last one zero-padded
inline uint64_t mix_bytes(uint64_t h, const void* data, uint64_t n) {
  const uint8_t* p = static_cast<const uint8_t*>(data);
  h = mix(h, n);
  uint64_t i = 0;
  for (; i + 8 <= n; i += 8) h = mix(h, load_u64(p + i));
  if (i < n) {
    uint64_t w = 0;
    std::memcpy(&w, p + i, (size_t)(n - i));
    h = mix(h, w);
  }
  return h;
}
inline uint64_t checksum(const uint8_t* p, uint64_t n) { return mix_bytes(kHashBasis, p, n); }
inline uint64_t dbits(double x) { uint64_t b; std::memcpy(&b, &x, 8); return b; }

// ---- model fingerprint (DESIGN.md §2): everything in amwg_model except init ------------------------------------------------------
inline uint64_t model_fingerprint(const amwg_model* md) {
  uint64_t h = kHashBasis;
  auto i64 = [&](int64_t v) { h = mix(h, (uint64_t)v); };
  auto f64 = [&](double v) { h = mix(h, dbits(v)); };
  auto i32s = [&](const int32_t* p, int64_t n) { h = mix_bytes(h, p, p ? sizeof(int32_t) * (uint64_t)std::max<int64_t>(n, 0) : 0); };
  i64(md->n_params);
  for (int p = 0; p < md->n_params; ++p) {
    const amwg_param& pa = md->params[p];
    i64(pa.type); i64(pa.n_comp); i64(pa.dim0); i64(pa.comp_offset); f64(pa.lower); f64(pa.upper);
  }
  i64(md->n_comp);
  for (int c = 0; c < md->n_comp; ++c) {
    const amwg_comp_options& o = md->comp_options[c];
    f64(o.prop_log_scale); f64(o.batch_size); f64(o.max_adaptation); f64(o.initial_adaptation); f64(o.target_accept_rate); i64(o.is_adapting);
  }
  i32s(md->code, md->n_code);
  i64(md->logpost_prog); i64(md->derived_prog); i64(md->n_derived);
  h = mix_bytes(h, md->consts, sizeof(double) * (uint64_t)std::max(md->n_consts, 0));
  i64(md->n_columns);
  for (int k = 0; k < md->n_columns; ++k) h = mix_bytes(h, md->columns[k].values, sizeof(double) * (uint64_t)std::max<int64_t>(md->columns[k].n, 0));
  i64(md->n_plates);
  for (int q = 0; q < md->n_plates; ++q) {
    const amwg_plate& pl = md->plates[q];
    i64(pl.kind); i64(pl.n);
    for (int j = 0; j < 4; ++j) { i64(pl.col[j]); i64(pl.iparam[j]); }
  }
  i64(md->n_fold);
  if (md->n_fold > 0) { i32s(md->fold_prog, md->n_fold); i32s(md->fold_dst, md->n_fold); }
  const bool cached = md->comp_prog && md->n_terms > 0;
  i64(cached ? md->n_terms : 0);
  if (cached) {
    i32s(md->comp_prog, md->n_comp);
    i32s(md->touch_off, md->n_comp + 1);
    i32s(md->touch_terms, md->touch_off[md->n_comp]);
    const bool blocks = md->n_block_params > 0 && md->block_params && md->term_block_comp;
    i64(blocks ? md->n_block_params : 0);
    if (blocks) { i32s(md->block_params, md->n_block_params); i32s(md->term_block_comp, (int64_t)md->n_block_params * md->n_terms); }
    i64(md->stat_prog); i64(md->n_sum_terms);
  }
  i64(md->n_variant_comps);
  if (md->n_variant_comps > 0) {
    const int nv = 1 << md->n_variant_comps;
    i32s(md->variant_comps, md->n_variant_comps);
    i32s(md->variant_logpost, nv);
    for (int v = 0; v < nv; ++v) i64(md->variant_derived ? md->variant_derived[v] : -1);
  }
  return h;
}

// Binary components hold 0 or 1 (the values BinaryStepper flips between, mcmc.js:753-767): the init at amwg_create, every chain's
// value at amwg_set_state and every restored chain. x is [n_comp][per_comp]; returns false at the first other value.
inline bool binary_values_ok(const amwg_param* params, int n_params, const double* x, size_t per_comp) {
  for (int p = 0; p < n_params; ++p) {
    if (params[p].type != AMWG_BINARY) continue;
    for (size_t k = (size_t)params[p].comp_offset * per_comp; k < (size_t)(params[p].comp_offset + params[p].n_comp) * per_comp; ++k)
      if (x[k] != 0.0 && x[k] != 1.0) return false;
  }
  return true;
}

// ---- layout ---------------------------------------------------------------------------------------------------------------------
constexpr uint64_t kFixedHeader = 56;
struct Layout {
  uint64_t state, pls, perm, rng_n, acc, perm_ext, ladder, accepts, sum, total;   // byte offsets; perm / perm_ext / ladder: ~0 when absent
};
constexpr uint64_t kAbsent = ~0ull;
constexpr uint32_t kMaxRungs = 256;
inline Layout layout(uint64_t D, uint64_t P, uint64_t C, uint64_t K = 0) {
  Layout L{};
  uint64_t o = kFixedHeader + 24 * D;
  L.state = o; o += 8 * D * C;
  L.pls = o; o += 8 * D * C;
  if (P <= 16) { L.perm = o; o += 8 * C; } else L.perm = kAbsent;
  L.rng_n = o; o += 8 * C;
  L.acc = o; o += 4 * D * C;
  if (P > 16) { L.perm_ext = o; o += P * C; } else L.perm_ext = kAbsent;
  if (K) { L.ladder = o; L.accepts = o + 8 * K + 8; o = L.accepts + 8 * (C / K) * (K - 1); } else L.ladder = L.accepts = kAbsent;
  L.sum = o;
  L.total = o + 8;
  return L;
}
inline uint64_t per_chain_bytes(uint64_t D, uint64_t P) { return 20 * D + 8 + (P > 16 ? P : 8); }

// Chain-invariant part of an image: what amwg_sampler keeps on the host.
struct Header {
  uint32_t version = kVersion, P = 0, D = 0;
  uint64_t fingerprint = 0, seed = 0, first_chain = 0, n_chains = 0;
  std::vector<uint64_t> is_adapting;
  std::vector<double> iter_since, batch_count;
  uint32_t K = 0;                      // tempered ladder: K rungs with beta[K], `rounds` swap rounds performed (0: untempered)
  std::vector<double> beta;
  uint64_t rounds = 0;
};

inline void put_u32(uint8_t* p, uint32_t v) { std::memcpy(p, &v, 4); }
inline void put_u64(uint8_t* p, uint64_t v) { std::memcpy(p, &v, 8); }
inline uint32_t get_u32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
inline double get_f64(const uint8_t* p) { double v; std::memcpy(&v, p, 8); return v; }

// The header of an image of layout(h.D, h.P, h.n_chains, h.K).total bytes, and with K > 0 the ladder's beta and rounds; the arrays
// (and the accepts) go to their sections (the caller's copies), then seal().
inline void write_header(uint8_t* out, const Header& h) {
  std::memcpy(out, kMagic, 8);
  put_u32(out + 8, h.version); put_u32(out + 12, h.P); put_u32(out + 16, h.D); put_u32(out + 20, h.K);
  put_u64(out + 24, h.fingerprint); put_u64(out + 32, h.seed); put_u64(out + 40, h.first_chain); put_u64(out + 48, h.n_chains);
  for (uint32_t c = 0; c < h.D; ++c) {
    uint8_t* r = out + kFixedHeader + 24 * (uint64_t)c;
    put_u64(r, h.is_adapting[c]);
    std::memcpy(r + 8, &h.iter_since[c], 8);
    std::memcpy(r + 16, &h.batch_count[c], 8);
  }
  if (h.K) {
    const Layout L = layout(h.D, h.P, h.n_chains, h.K);
    for (uint32_t r = 0; r < h.K; ++r) std::memcpy(out + L.ladder + 8 * (uint64_t)r, &h.beta[r], 8);
    put_u64(out + L.ladder + 8 * (uint64_t)h.K, h.rounds);
  }
}
inline void seal(uint8_t* out, const Layout& L) { put_u64(out + L.sum, checksum(out, L.sum)); }

// ---- reading ----------------------------------------------------------------------------------------------------------------------
struct View {
  Header h;
  Layout L;
  const uint8_t* p = nullptr;
};

// magic, version, sizes and checksum of one image. Returns "" or the refusal.
inline std::string parse(const uint8_t* p, int64_t n, View& v) {
  if (!p || n < (int64_t)kFixedHeader || std::memcmp(p, kMagic, 8) != 0) return "restore: not a checkpoint image";
  v.h.version = get_u32(p + 8);
  if (v.h.version != kVersion) return "restore: unsupported format version " + std::to_string(v.h.version) + " (this library reads version 1)";
  v.h.P = get_u32(p + 12); v.h.D = get_u32(p + 16);
  v.h.fingerprint = load_u64(p + 24); v.h.seed = load_u64(p + 32); v.h.first_chain = load_u64(p + 40); v.h.n_chains = load_u64(p + 48);
  v.h.K = get_u32(p + 20);
  const uint64_t D = v.h.D, P = v.h.P, C = v.h.n_chains, K = v.h.K;
  const uint64_t per = per_chain_bytes(D, P);
  if ((K != 0 && (K < 2 || K > kMaxRungs || C % K || v.h.first_chain % K)) || D == 0 || D > (1u << 24) || P == 0 || P > D || C == 0 ||
      C > ((uint64_t)1 << 40) / per || (uint64_t)n != layout(D, P, C, K).total)
    return "restore: the image is truncated or its size does not match its header";
  v.L = layout(D, P, C, K);
  if (load_u64(p + v.L.sum) != checksum(p, v.L.sum)) return "restore: the image is damaged (checksum mismatch)";
  v.h.is_adapting.resize(D); v.h.iter_since.resize(D); v.h.batch_count.resize(D);
  for (uint64_t c = 0; c < D; ++c) {
    const uint8_t* r = p + kFixedHeader + 24 * c;
    v.h.is_adapting[c] = load_u64(r); v.h.iter_since[c] = get_f64(r + 8); v.h.batch_count[c] = get_f64(r + 16);
  }
  v.h.beta.resize(K);
  for (uint64_t r = 0; r < K; ++r) v.h.beta[r] = get_f64(p + v.L.ladder + 8 * r);
  v.h.rounds = K ? load_u64(p + v.L.ladder + 8 * K) : 0;
  v.p = p;
  return "";
}

// What a restore must match: the handle's model and chain range.
struct Target {
  uint64_t fingerprint = 0, first_chain = 0, n_chains = 0;
  int D = 0, P = 0;
  std::vector<amwg_param> params;
  std::vector<double> batch_size;      // per component
  std::vector<double> beta;            // the handle's ladder (empty: untempered)
};

// Chains [dst, dst + count) of the handle (handle-local ids) come from chains [src, src + count) of image `img` (image-local ids).
struct Piece {
  int img;
  uint64_t src, dst, count;
};

inline bool is_count(double x) { return x >= 0 && x <= 9007199254740992.0 && x == (double)(int64_t)x; }

// Every check of a restore, on the host, before anything on the device changes. On success `pieces` (ordered by dst) cover the
// handle's chains exactly once. Returns "" or the refusal.
inline std::string check(const std::vector<View>& views, const Target& t, std::vector<Piece>& pieces) {
  pieces.clear();
  if (views.empty()) return "restore: no image given";
  const Header& h0 = views[0].h;
  for (const View& v : views)
    if (v.h.fingerprint != t.fingerprint || (int)v.h.D != t.D || (int)v.h.P != t.P)
      return "restore: the image was taken with a different model, data or options";
  for (const View& v : views) {
    if (v.h.K && t.beta.empty()) return "restore: the image is of a tempered ladder (options.temperatures) and this sampler is not tempered";
    if (!v.h.K && !t.beta.empty()) return "restore: this sampler is a tempered ladder (options.temperatures) and the image is not";
    bool same_ladder = v.h.K == t.beta.size();
    for (uint32_t r = 0; same_ladder && r < v.h.K; ++r) same_ladder = dbits(v.h.beta[r]) == dbits(t.beta[r]);
    if (!same_ladder) return "restore: the image was taken with other temperatures";
  }
  for (const View& v : views) {
    bool same = v.h.seed == h0.seed && v.h.rounds == h0.rounds;
    for (int c = 0; same && c < t.D; ++c)
      same = v.h.is_adapting[c] == h0.is_adapting[c] && dbits(v.h.iter_since[c]) == dbits(h0.iter_since[c]) &&
             dbits(v.h.batch_count[c]) == dbits(h0.batch_count[c]);
    if (!same) return "restore: the images come from different runs, or from different points of one run";
  }
  for (const amwg_param& pa : t.params)
    for (int c = pa.comp_offset; c < pa.comp_offset + pa.n_comp; ++c) {
      const uint64_t ad = h0.is_adapting[c];
      const double it = h0.iter_since[c], bc = h0.batch_count[c];
      if (ad > 1 || (pa.type == AMWG_BINARY && ad != 0) || !is_count(it) || !is_count(bc) || !(it == 0 || !(it >= t.batch_size[c])))
        return "restore: invalid adaptation counters";
    }
  // chain ranges: sorted by first global chain, no overlap, the handle's range covered
  std::vector<int> order(views.size());
  for (size_t k = 0; k < views.size(); ++k) order[k] = (int)k;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return views[a].h.first_chain < views[b].h.first_chain; });
  for (size_t k = 0; k + 1 < order.size(); ++k) {
    const Header& a = views[order[k]].h;
    const Header& b = views[order[k + 1]].h;
    if (a.first_chain > ~0ull - a.n_chains) return "restore: the image is truncated or its size does not match its header";
    if (b.first_chain < a.first_chain + a.n_chains) return "restore: images overlap at chain " + std::to_string(b.first_chain);
  }
  const uint64_t lo = t.first_chain, hi = t.first_chain + t.n_chains;
  uint64_t next = lo;
  for (int k : order) {
    const Header& a = views[k].h;
    const uint64_t a0 = a.first_chain, a1 = a.first_chain + a.n_chains;
    if (a1 <= next || a0 >= hi) continue;
    if (a0 > next) break;
    const uint64_t end = std::min(a1, hi);
    pieces.push_back(Piece{k, next - a0, next - lo, end - next});
    next = end;
    if (next == hi) break;
  }
  if (next < hi) {
    uint64_t gap_end = hi;
    for (int k : order) if (views[k].h.first_chain > next) { gap_end = std::min(gap_end, views[k].h.first_chain); break; }
    pieces.clear();
    return "restore: chains [" + std::to_string(next) + ", " + std::to_string(gap_end) + ") are not covered by the images";
  }
  const uint64_t K = t.beta.size();                 // whole ladders only (images and handles of a tempered run always hold whole ladders)
  for (const Piece& pc : pieces)
    if (K && (pc.src % K || pc.dst % K || pc.count % K)) { pieces.clear(); return "restore: the images split a ladder"; }
  // per chain, over the chains the handle takes
  const int D = t.D, P = t.P;
  std::vector<double> x(D);
  for (const Piece& pc : pieces) {
    const View& v = views[pc.img];
    const uint64_t C = v.h.n_chains;
    for (uint64_t j = pc.src; j < pc.src + pc.count; ++j) {
      const uint64_t g = v.h.first_chain + j;
      const std::string who = "restore: chain " + std::to_string(g);
      unsigned seen = 0;
      bool ok = true;
      if (P <= 16) {
        const uint64_t perm = load_u64(v.p + v.L.perm + 8 * j);
        if (P < 16 && (perm >> (4 * P)) != 0) ok = false;
        for (int i = 0; ok && i < P; ++i) {
          const unsigned e = (unsigned)((perm >> (4 * i)) & 15u);
          ok = e < (unsigned)P && !(seen & (1u << e));
          seen |= 1u << e;
        }
      } else {
        std::vector<unsigned char> mark(P, 0);
        for (int i = 0; ok && i < P; ++i) {
          const unsigned e = v.p[v.L.perm_ext + (uint64_t)i * C + j];
          ok = e < (unsigned)P && !mark[e];
          if (ok) mark[e] = 1;
        }
      }
      if (!ok) { pieces.clear(); return who + " has an invalid substepper order"; }
      for (int c = 0; c < D; ++c) {
        int32_t a;
        std::memcpy(&a, v.p + v.L.acc + 4 * ((uint64_t)c * C + j), 4);
        if (a < 0) { pieces.clear(); return who + " has a negative acceptance count"; }
        x[c] = get_f64(v.p + v.L.state + 8 * ((uint64_t)c * C + j));
      }
      if (!binary_values_ok(t.params.data(), P, x.data(), 1)) { pieces.clear(); return who + " has a binary parameter other than 0 or 1"; }
    }
  }
  return "";
}

// The per-chain arrays of an image: [rows][C] elements of `width` bytes at byte offset `off`.
enum Section { kState, kPls, kPerm, kRng, kAcc, kPermExt, kSections };
struct Span { uint64_t off, rows, width; };
inline Span span(const Layout& L, int D, int P, Section s) {
  switch (s) {
    case kState: return {L.state, (uint64_t)D, 8};
    case kPls: return {L.pls, (uint64_t)D, 8};
    case kPerm: return {L.perm, P <= 16 ? 1ull : 0ull, 8};
    case kRng: return {L.rng_n, 1, 8};
    case kAcc: return {L.acc, (uint64_t)D, 4};
    default: return {L.perm_ext, P > 16 ? (uint64_t)P : 0ull, 1};
  }
}

// Section `s` of the handle's chains, assembled from the pieces into dst ([rows][n_chains]): the host form of the upload that
// amwg_checkpoint_load does with one cudaMemcpy2D per piece and section.
inline void gather(const std::vector<View>& views, const std::vector<Piece>& pieces, int D, int P, Section s, uint64_t n_chains, uint8_t* dst) {
  for (const Piece& pc : pieces) {
    const View& v = views[pc.img];
    const Span sp = span(v.L, D, P, s);
    for (uint64_t r = 0; r < sp.rows; ++r)
      std::memcpy(dst + (r * n_chains + pc.dst) * sp.width, v.p + sp.off + (r * v.h.n_chains + pc.src) * sp.width, (size_t)(pc.count * sp.width));
  }
}

// The accepted-swap counters of a tempered handle's ladders ([n_chains / K][K - 1] u64), assembled from the pieces into dst.
inline void gather_accepts(const std::vector<View>& views, const std::vector<Piece>& pieces, uint64_t K, uint8_t* dst) {
  const uint64_t w = 8 * (K - 1);
  for (const Piece& pc : pieces) {
    const View& v = views[pc.img];
    std::memcpy(dst + pc.dst / K * w, v.p + v.L.accepts + pc.src / K * w, (size_t)(pc.count / K * w));
  }
}

}  // namespace ckpt
}  // namespace amwg
