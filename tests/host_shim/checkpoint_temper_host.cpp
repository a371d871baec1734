// Test infrastructure: the checkpoint image code (csrc/amwg_checkpoint.h) with the ladder section of tempered handles, compiled for
// the HOST behind a C ABI, for tests/test_temper_checkpoint_host.py.
#include <cstdio>

#include "amwg_checkpoint.h"

using namespace amwg::ckpt;
extern "C" {
uint64_t hs_image_size(uint64_t D, uint64_t P, uint64_t C, uint64_t K) { return layout(D, P, C, K).total; }

// an image from host arrays laid out as in the image; K = 0 writes an untempered image (beta, accepts ignored)
void hs_write_image(uint32_t P, uint32_t D, uint64_t fingerprint, uint64_t seed, uint64_t first_chain, uint64_t C, const uint64_t* is_adapting,
                    const double* iter_since, const double* batch_count, const double* state, const double* pls, const uint64_t* perm,
                    const uint64_t* rng_n, const int32_t* acc, const uint8_t* perm_ext, uint32_t K, const double* beta, uint64_t rounds,
                    const uint64_t* accepts, uint8_t* out) {
  Header h;
  h.P = P; h.D = D; h.fingerprint = fingerprint; h.seed = seed; h.first_chain = first_chain; h.n_chains = C;
  h.is_adapting.assign(is_adapting, is_adapting + D); h.iter_since.assign(iter_since, iter_since + D); h.batch_count.assign(batch_count, batch_count + D);
  h.K = K; if (K) h.beta.assign(beta, beta + K); h.rounds = rounds;
  const Layout L = layout(D, P, C, K);
  write_header(out, h);
  const void* src[kSections] = {state, pls, perm, rng_n, acc, perm_ext};
  for (int s = 0; s < kSections; ++s) {
    const Span sp = span(L, (int)D, (int)P, (Section)s);
    if (sp.rows) std::memcpy(out + sp.off, src[s], (size_t)(sp.rows * C * sp.width));
  }
  if (K) std::memcpy(out + L.accepts, accepts, (size_t)(8 * (C / K) * (K - 1)));
  seal(out, L);
}

// a restore into a handle over [first_chain, first_chain + n_chains) with the ladder beta[K] (K = 0: untempered): the checks, then
// state, rng_n, the rounds and the accepts ([n_chains / K][K - 1]). Returns 0, or -1 with the refusal in err.
int hs_restore(const uint8_t* const* images, const int64_t* sizes, int n_images, uint64_t fingerprint, uint64_t first_chain, uint64_t n_chains,
               int D, int P, const int32_t* types, const int32_t* comp_offset, const int32_t* n_comp, const double* batch_size, uint32_t K,
               const double* beta, double* state, uint64_t* rng_n, uint64_t* rounds, uint64_t* accepts, char* err, int64_t err_cap) {
  std::vector<View> views(n_images);
  std::string e;
  for (int k = 0; k < n_images && e.empty(); ++k) e = parse(images[k], sizes[k], views[k]);
  Target t;
  t.fingerprint = fingerprint; t.first_chain = first_chain; t.n_chains = n_chains; t.D = D; t.P = P;
  for (int p = 0; p < P; ++p) { amwg_param pa{}; pa.type = types[p]; pa.comp_offset = comp_offset[p]; pa.n_comp = n_comp[p]; pa.dim0 = 1; t.params.push_back(pa); }
  t.batch_size.assign(batch_size, batch_size + D);
  if (K) t.beta.assign(beta, beta + K);
  std::vector<Piece> pieces;
  if (e.empty()) e = check(views, t, pieces);
  if (!e.empty()) { snprintf(err, (size_t)err_cap, "%s", e.c_str()); return -1; }
  gather(views, pieces, D, P, kState, n_chains, (uint8_t*)state);
  gather(views, pieces, D, P, kRng, n_chains, (uint8_t*)rng_n);
  *rounds = views[0].h.rounds;
  if (K) gather_accepts(views, pieces, K, (uint8_t*)accepts);
  return 0;
}
}
