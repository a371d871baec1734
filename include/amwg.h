/*
 * amwg.h -- C ABI of the H100-native many-chain AMWG sampler (libamwg_b200.so).
 *
 * The reference (rasmusab/bayes.js) has no FFI: its boundary is the JavaScript object API
 *     new mcmc.AmwgSampler(params, log_post, data, options)   mcmc.js:1090-1092, 940-966
 *     .burn(n) .sample(n) .step() .thin(k) .monitor(names)     mcmc.js:985-1055
 *     .start_adaptation() .stop_adaptation() .info()           mcmc.js:1060-1073, 977-980
 * This header is what the Node N-API addon (js/amwg_napi.cc, see INTEGRATION.md), the Python host (bayes.js_b200/_ffi.py) or any other host
 * binds instead.  Plain pointers and sizes only; every call returns 0 or a negative status and
 * amwg_last_error() gives the message the JS shim re-throws as a bare string (the reference
 * throws strings, mcmc.js:165,299,315,340,445,490,495,636,746,790,867,972).
 *
 * Calls block until the result is usable; a handle is not thread-safe (the reference is
 * single-threaded); all per-chain state stays resident in HBM between calls, so successive
 * burn()/sample() calls continue the same chains (mcmc.js:964-965, 509-511).
 *
 * A handle owns `n_chains` independent chains with global ids [first_chain, first_chain+n_chains).
 * Chain g behaves exactly like one run of the reference with Math.random() replaced by the
 * Philox4x32-10 stream (seed, g) defined in DESIGN.md "RNG contract"; results therefore do not
 * depend on how chains are sharded over handles / GPUs.
 */
#ifndef AMWG_H_
#define AMWG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AMWG_ABI_VERSION 8
#define AMWG_MAX_BLOCK_PARAMS 4
#if defined(__GNUC__)
#define AMWG_API __attribute__((visibility("default")))
#else
#define AMWG_API
#endif

/* ---- parameters: one entry per key of the completed `params` object (mcmc.js:357-403) ---- */
enum { AMWG_REAL = 0, AMWG_INT = 1, AMWG_BINARY = 2 };

typedef struct {
  int32_t type;          /* AMWG_REAL | AMWG_INT | AMWG_BINARY                      (mcmc.js:844-868) */
  int32_t n_comp;        /* prod(dim): scalar components, flattened row-major                          */
  int32_t dim0;          /* dim[0]: the level visited in random order each sweep   (mcmc.js:244-263)  */
  int32_t comp_offset;   /* index of the first component in the flat state vector                     */
  double lower, upper;   /* bounds, +-inf allowed                                  (mcmc.js:497-498)  */
} amwg_param;

/* per scalar component: the options OnedimMetropolisStepper resolves (mcmc.js:500-505, 658-660) */
typedef struct {
  double prop_log_scale;       /* default 0    */
  double batch_size;           /* default 50   */
  double max_adaptation;       /* default 0.33 */
  double initial_adaptation;   /* default 1.0  */
  double target_accept_rate;   /* default 0.44 */
  int32_t is_adapting;         /* default 1    */
  int32_t _pad;
} amwg_comp_options;

/* ---- data: named fp64 columns (JS numbers); copied to the device at create ---- */
typedef struct {
  const double* values;
  int64_t n;
} amwg_column;

/* ---- log_post as a program --------------------------------------------------------------
 * log_post(state, data) (mcmc.js:958-960) arrives as a postfix program over an fp64 stack.
 * Instruction word (int32):
 *     bits  0-7   opcode
 *     bits  8-9   mode of operand A     0 = popped from the stack, 1 = consts[next word], 2 = state component [next word],
 *                                       3 = the opcode has no such operand
 *     bits 10-11  mode of operand B     (operands are named in source order: op(A, B, C, D))
 *     bits 12-13  mode of operand C
 *     bits 14-15  mode of operand D
 *     bit  16     ACC flag: the result is added to lp (lp = lp + result) instead of being pushed
 *     bit  17     STORE flag (only with ACC, or on PLATE): the value is also written to the chain's term cache; the term id
 *                 follows as the last extra word of the instruction
 *     bits 18-31  immediate `a` (const index, component, column, plate id ...)
 * Inline operand words follow the instruction word in consumption order: last operand first (D, C, B, A), which is
 * also the order stack operands are popped.  Further extra words are noted per opcode.
 * The accumulator `lp` starts at 0 and receives terms strictly in program order, so the sum is formed in the same
 * order as the JS `log_post += ...` statements.  Every arithmetic op is a single IEEE-754 fp64 operation (no FMA
 * contraction); LOG/EXP are the fdlibm algorithms V8's Math.log/Math.exp port; LD_* follow distributions.js operation
 * by operation (cited per opcode in csrc/amwg_ld.cuh).
 */
#define AMWG_MODE_STACK 0
#define AMWG_MODE_CONST 1
#define AMWG_MODE_COMP 2
#define AMWG_MODE_NONE 3
#define AMWG_WORD(op, mA, mB, mC, mD, acc, a) \
  ((int32_t)((uint32_t)(op) | ((uint32_t)(mA) << 8) | ((uint32_t)(mB) << 10) | ((uint32_t)(mC) << 12) | ((uint32_t)(mD) << 14) | \
             ((uint32_t)((acc) ? 1 : 0) << 16) | ((uint32_t)(a) << 18)))
#define AMWG_STORE_FLAG (1u << 17)
#define AMWG_MAX_IMMEDIATE 16383

enum {
  AMWG_OP_END = 0,
  AMWG_OP_CONST,        /* push consts[operand]                                             */
  AMWG_OP_COMP,         /* push state component `operand` (proposal value for the moved one) */
  AMWG_OP_DATA,         /* push columns[operand][next word]                                  */
  AMWG_OP_DATA_I,       /* push columns[operand][off + stride*i], i = plate point; next words: off, stride */
  AMWG_OP_COMP_I,       /* push state component base + (int)columns[operand][off + stride*i]; next words: off, stride, base */
  AMWG_OP_ADD, AMWG_OP_SUB, AMWG_OP_MUL, AMWG_OP_DIV, AMWG_OP_NEG,
  AMWG_OP_LOG, AMWG_OP_EXP, AMWG_OP_SQRT, AMWG_OP_ABS, AMWG_OP_POW,
  AMWG_OP_LT, AMWG_OP_LE, AMWG_OP_GT, AMWG_OP_GE, AMWG_OP_EQ, AMWG_OP_NE,   /* push 1.0 / 0.0 */
  AMWG_OP_AND, AMWG_OP_OR, AMWG_OP_NOT,
  AMWG_OP_SELECT,       /* pops b, a, c ; pushes c != 0 ? a : b                              */
  AMWG_OP_LGAMMA, AMWG_OP_LFACTORIAL, AMWG_OP_LCHOOSE, AMWG_OP_LBETA,   /* distributions.js:63-92 */
  AMWG_OP_LD_NORM, AMWG_OP_LD_UNIF, AMWG_OP_LD_BETA, AMWG_OP_LD_BERN, AMWG_OP_LD_POIS,
  AMWG_OP_LD_CAUCHY, AMWG_OP_LD_LAPLACE, AMWG_OP_LD_GAMMA, AMWG_OP_LD_INVGAMMA, AMWG_OP_LD_LNORM,
  AMWG_OP_LD_PARETO, AMWG_OP_LD_T, AMWG_OP_LD_WEIBULL, AMWG_OP_LD_LOGIS, AMWG_OP_LD_EXP,
  AMWG_OP_LD_BINOM, AMWG_OP_LD_NBINOM, AMWG_OP_LD_HYPER,
  AMWG_OP_ACC,          /* lp = lp + pop                                                     */
  AMWG_OP_PLATE,        /* lp = plate[operand](lp, popped operands): a recognised O(N) likelihood sum */
  AMWG_OP_STORE,        /* derived[operand] = pop   (derived-quantity program only)          */
  AMWG_OP_LOOP_BEGIN,   /* start of a GENERIC plate body: i = 0 (plate[a].n points); next word: offset to continue at when n == 0 */
  AMWG_OP_LOOP_END,     /* lp = lp + pop; if (++i < n) jump to the word offset in the next word (first word of the body) */
  /* ld.* with constant hyper-parameters, partially evaluated by the host: the constant parts are folded once on the device
   * (fold table), the rest is the same operations in the same order as distributions.js -> same bits as the LD_* opcode. */
  AMWG_OP_NORM_K,       /* (x, mean, K1, K2): K1 - pow(x-mean,2)/K2,  K1 = -0.5*log(2pi) - log(sd), K2 = 2*sd*sd   (:119-121) */
  AMWG_OP_UNIF_K,       /* (x, min, max, K):  (x<min || x>max) ? -inf : K,  K = log(1/(max-min))                    (:221-223) */
  AMWG_OP_BETA_K,       /* (x, a1, b1, K):    (x>1 || x<0) ? -inf : a1*log(x) + b1*log(1-x) - K, a1 = shape1-1, b1 = shape2-1, K = lbeta (:104-113) */
  AMWG_OP_ACC_RANGE,    /* lp = lp + cache[a] + cache[a+1] + ... (next word: count), one term at a time, in order: the terms of the
                           sum that do not read the moved component, taken from the chain's term cache (see amwg_model.comp_prog) */
  /* Pre-evaluated plate statistics (see amwg_model.stat_prog). A NORM_IID plate is  f(S, sd) = n*(-0.5*log(2pi) - log(sd)) - S/(2*sd*sd)
   * with S = sum_i (x_i - mean)^2 -- the O(N) part, which only depends on the mean operand. */
  AMWG_OP_PLATE_SS,     /* (mean): push S of plate `a`; next word: the statistic's slot in the term cache, S is stored there too */
  AMWG_OP_NORM_SS,      /* (S, sd): f(S, sd) of plate `a` (same operations as AMWG_PLATE_NORM_IID, given its S)                */
  AMWG_OP_CACHED,       /* push cache[a]      : the committed value of slot a (a statistic of the chain's current state)       */
  AMWG_OP_CAND,         /* push candidate[a]  : the value the last stat_prog evaluation computed for slot a (at the proposals)   */
  AMWG_OP__COUNT
};

/* A plate is a run of N structurally identical likelihood terms, `for (i...) log_post += ld.X(data[i], ...)`.
 * Recognised shapes get a hand-written inner loop (AMWG_OP_PLATE; their index-free operands are evaluated by
 * the program and popped from the stack); anything else is a bytecode loop over its body
 * (AMWG_OP_LOOP_BEGIN ... AMWG_OP_LOOP_END, body uses DATA_I / COMP_I), bit-faithful to the JS loop. */
enum {
  AMWG_PLATE_GENERIC = 0,   /* bytecode loop: lp += body(i), i = 0..n-1, in order                                   */
  AMWG_PLATE_NORM_IID,      /* operands A = mean, B = sd.  sum_i ld.norm(x_i, mean, sd), factorised:
                               N*(-0.5*log(2pi) - log(sd)) - sum_i (x_i-mean)^2 / (2*sd*sd)     (KS-level parity)   */
  AMWG_PLATE_BERN_IID,      /* operand A = p.  sum_i ld.bern(y_i, p), sequential, bit-faithful                       */
  AMWG_PLATE_NORM_GROUPED,  /* operand A = sd.  sum_i ld.norm(y_i, mu[g_i], sd); points sorted by group              */
  AMWG_PLATE_POIS_LOGLIN    /* sum_i ld.pois(y_i, exp(sum_k X_ik * beta_k)) = beta . (X^T y) - sum_i exp(X_i . beta) - sum_i lfactorial(y_i):
                               the linear part and the constant come precomputed (col[2]), the device sums the exponentials.
                               K in {1..8, 10, 12, 16}                                           (KS-level parity)   */
};

typedef struct {
  int32_t kind;          /* AMWG_PLATE_*                                                          */
  int32_t n;             /* number of points                                                       */
  int32_t col[4];        /* data columns: [0] x or y; GROUPED: [1] group start offsets (J+1);
                            POIS_LOGLIN: [1] X row-major n*K, [2] K+1 values filled by the host: X^T y, then sum_i lfactorial(y_i) */
  int32_t iparam[4];     /* GROUPED: [0] first mu component, [1] J;  POIS_LOGLIN: [0] first beta component, [1] K;
                            all specialised kinds: [2] offset of the plate's first point inside col[0]              */
} amwg_plate;

typedef struct {
  int32_t abi_version;                     /* AMWG_ABI_VERSION */
  int32_t n_params;   const amwg_param* params;
  int32_t n_comp;     const double* init;                  /* params[*].init flattened, length n_comp */
  const amwg_comp_options* comp_options;                   /* length n_comp (ignored for binary)      */
  int32_t n_code;     const int32_t* code;                 /* all programs, concatenated              */
  int32_t logpost_prog;                                    /* word offset of the log_post program     */
  int32_t derived_prog;                                    /* word offset of the derived program, -1  */
  int32_t n_derived;                                       /* derived quantities (state keys beyond params, mcmc.js:990) */
  int32_t n_consts;   const double* consts;
  int32_t n_columns;  const amwg_column* columns;
  int32_t n_plates;   const amwg_plate* plates;
  /* Constant sub-expressions (no parameter, no plate index) are evaluated ONCE on the device at create, with the
   * device's own arithmetic, and stored into consts[fold_dst[k]]: fold_prog[k] is the word offset of an
   * END-terminated expression program.  (log(2*pi), log(sd) of a constant sd, ... : same bits, computed once.) */
  int32_t n_fold;     const int32_t* fold_prog;  const int32_t* fold_dst;
  /* Control flow on binary parameters (`if (m === 0) ... else ...`, tests/test_data.js:163-168) cannot be recorded as one
   * expression, so the host records log_post once per configuration of up to AMWG_MAX_VARIANT_COMPS binary components.
   * Configuration v has bit k set when state component variant_comps[k] is non-zero (the proposal counts for the moved one);
   * its programs start at variant_logpost[v] / variant_derived[v]. n_variant_comps == 0: logpost_prog / derived_prog are used. */
  /* Dependency-aware evaluation (optional). log_post is a sum of terms; a step that moves component c only changes the terms
   * that read c. With comp_prog != NULL the sampler keeps every value-term of every chain in a term cache (n_terms doubles per
   * chain) and evaluates a proposal for component c with comp_prog[c]: the terms that read c are recomputed (STORE flag: the new
   * value goes to a candidate slot), the others are added from the cache by ACC_RANGE -- each in its original position, so the
   * sum is formed in the same order with the same values as the full program (bit-identical). On acceptance the candidates of
   * touch_terms[touch_off[c] .. touch_off[c+1]) are committed. logpost_prog is the full program (it stores every value-term). */
  int32_t n_terms;          const int32_t* comp_prog;      /* n_comp word offsets, or NULL */
  const int32_t* touch_off; const int32_t* touch_terms;    /* n_comp + 1 offsets into touch_terms */
  /* Block steps (optional, needs comp_prog). A multi-dim parameter whose components never share a term (every term reads at most
   * one of them: the group means of a hierarchical model) can be stepped with ONE evaluation of the full program: the proposals
   * (and accept uniforms) of all its components are drawn first, in the chain's random visiting order, the program is evaluated
   * with all of them in place (every term's candidate value lands in the term cache), and the accept decisions are then taken one
   * component at a time in visiting order from the cached terms -- the same sums, values and uniforms as stepping them one by
   * one. block_params lists such parameters (indices into params[]); term_block_comp[k * n_terms + t] is the component of
   * block_params[k] that term t reads, or -1. */
  int32_t n_block_params;   const int32_t* block_params;   const int32_t* term_block_comp;
  /* Pre-evaluated statistics (optional, needs comp_prog; no binary parameter, no variants). When every O(N) plate is a NORM_IID
   * plate whose mean reads exactly ONE component, the expensive part of a proposal's evaluation -- S at the proposed value of that
   * component -- does not depend on how the other steps of the sweep turn out, and neither do the sweep's random numbers (a step
   * consumes its rnorm trials and, if the proposal is in bounds, one uniform, whatever log_post says: mcmc.js:519-528). So a sweep
   * is run as: (a) draw every step's proposal and accept uniform, in the chain's visiting order; (b) ONE pass over the data:
   * stat_prog evaluates every statistic at the proposals (candidate slots n_sum_terms .. n_terms-1 of the term cache);
   * (c) the steps, in visiting order, each with comp_prog[c] -- which now contains no O(N) work: a plate term is NORM_SS of
   * CAND(slot) (the moved component is the plate's mean) or CACHED(slot) (it is not). Same values, same sums, same uniforms as
   * stepping with the full program, at one data pass per sweep instead of one per step. The term cache then has n_terms slots of
   * which the first n_sum_terms are terms of the sum (ACC_RANGE only ever covers those); without stat_prog n_sum_terms == n_terms. */
  int32_t stat_prog;        int32_t n_sum_terms;           /* stat_prog: word offset, -1 = not in use */
  int32_t n_variant_comps;  const int32_t* variant_comps;
  const int32_t* variant_logpost;  const int32_t* variant_derived;     /* 1 << n_variant_comps entries each (derived: -1 if none) */
} amwg_model;
#define AMWG_MAX_VARIANT_COMPS 4

typedef struct amwg_sampler amwg_sampler;

/* new mcmc.AmwgSampler(...) for n_chains chains on CUDA device `device` (mcmc.js:1090-1092, 940-966):
 * uploads the model, places every chain at params[*].init and evaluates log_post once. */
AMWG_API int amwg_create(const amwg_model* model, uint64_t n_chains, uint64_t first_chain, uint64_t seed,
                int device, amwg_sampler** out);
AMWG_API void amwg_destroy(amwg_sampler* s);

/* sampler.burn(n) -- mcmc.js:1035-1039 */
AMWG_API int amwg_burn(amwg_sampler* s, int64_t n);

/* sampler.sample(n) with thinning interval `thin` and the monitored entries `monitor[n_monitor]`
 * (index < n_comp: state component; n_comp + d: derived quantity d) -- mcmc.js:1005-1030.
 * Row r is the state BEFORE sweep r*thin (row 0 is the pre-existing state, mcmc.js:1021-1027).
 * Output layout: out[row][monitor][chain], fp64, rows = ceil(n/thin).
 *   amwg_sample        : host buffer (pinned memory recommended); D2H copies overlap the sweeps.
 *   amwg_sample_device : device buffer on the handle's device; no host traffic. */
AMWG_API int amwg_sample(amwg_sampler* s, int64_t n, int64_t thin, const int32_t* monitor, int32_t n_monitor, double* host_out);
AMWG_API int amwg_sample_device(amwg_sampler* s, int64_t n, int64_t thin, const int32_t* monitor, int32_t n_monitor, double* dev_out);

/* live state, as sampler.step() returns it (mcmc.js:985-997): out[entry][chain], entries = n_comp + n_derived */
AMWG_API int amwg_get_state(amwg_sampler* s, double* host_out);

/* sampler.log_post() -- the closure the Sampler ctor stores (mcmc.js:958-960): log_post at the chain's current state, out[chain] */
AMWG_API int amwg_get_log_post(amwg_sampler* s, double* host_out);

/* Per-chain starting points (not in the reference, which runs one chain from params[*].init).
 * amwg_set_state: host_in is [n_comp][chain] fp64 -- the first n_comp rows of what amwg_get_state returns. Every chain is placed
 *   there and log_post and its cached terms are evaluated afresh from it; derived quantities follow from the state. Proposal scales,
 *   acceptance counts, visiting orders, stream positions and adaptation counters are untouched and no random number is drawn: chain
 *   g then continues exactly like the reference chain g continued from host_in at the same point of its run. Binary components
 *   must be 0 or 1 (as at amwg_create); otherwise an error is returned and the handle is unchanged.
 * amwg_disperse_state: over-dispersed starting points drawn on the device, for convergence diagnostics that need chains to start
 *   apart (DESIGN.md §2 "Dispersed starting points"). Per chain, attempts a = 0..99 draw every component uniformly within +-radius
 *   of its init on the unconstrained scale (uniform #(2^63 + a*n_comp + c) of the chain's Philox stream, so the draws do not
 *   depend on sharding and never meet Math.random()'s); a chain keeps its first attempt whose components are valid and whose
 *   log_post is finite. The points are then committed as by amwg_set_state. radius must be finite and > 0. If some chains find no
 *   point in 100 attempts, *n_failed (when not null) receives their number, an error is returned and the handle is unchanged.
 * amwg_disperse_state_superchains: the same with superchains of superchain_size consecutive global chains (superchain k holds the
 *   chains [k superchain_size, (k + 1) superchain_size)) that start together, for nested R-hat (DESIGN.md §4.6). Global chain g
 *   draws its attempts from the stream of its superchain's first chain, superchain_size * floor(g / superchain_size), instead of
 *   its own, so every chain of a superchain keeps the same point, whichever handles hold them; superchain_size = 1 is
 *   amwg_disperse_state. The sampling streams stay keyed by g. Errors, before anything on the device changes: superchain_size < 1,
 *   and those of amwg_disperse_state. A handle holds a range of the global chains and does not know how many there are in all:
 *   that superchain_size divides the chain count is the caller's check (the hosts' options.superchain_size). */
AMWG_API int amwg_set_state(amwg_sampler* s, const double* host_in);
AMWG_API int amwg_disperse_state(amwg_sampler* s, double radius, int64_t* n_failed);
AMWG_API int amwg_disperse_state_superchains(amwg_sampler* s, double radius, int64_t superchain_size, int64_t* n_failed);

/* Checkpoints (not in the reference): save the whole run state of a handle and resume it later, bit for bit, in this or another
 * process, on any sharding of the chains (DESIGN.md §2 "Checkpoints" has the image layout and the guarantee).
 * amwg_model_fingerprint: the 64-bit hash of everything in `model` except init (params, options, programs, constants, data, plates
 *   and every table). Needs no device. amwg_create stores it in the handle; an image is only restored into a handle of the same
 *   fingerprint. It detects accidents (another data set, another option, another lowering); it is not a security measure.
 * amwg_checkpoint_size / amwg_checkpoint_save: the image of the handle's chains (state, prop_log_scale, acceptance counts,
 *   substepper orders, stream positions) with the seed, the chain range and the adaptation counters; host_out holds cap bytes.
 * amwg_checkpoint_load: images[k] (sizes[k] bytes) together must cover the handle's chains [first_chain, first_chain + n_chains),
 *   without overlap, from one point of one run of the same model. Everything is checked on the host first; a refused restore
 *   returns an error starting "restore: " and leaves the handle unchanged. With dry_run nothing else happens. Otherwise the
 *   handle's chains, its seed (the images' seed is adopted) and its adaptation counters become the images', and log_post and the
 *   term cache are evaluated afresh from the restored state. */
AMWG_API int amwg_model_fingerprint(const amwg_model* model, uint64_t* out);
AMWG_API int amwg_checkpoint_size(amwg_sampler* s, int64_t* out);
AMWG_API int amwg_checkpoint_save(amwg_sampler* s, uint8_t* host_out, int64_t cap);
AMWG_API int amwg_checkpoint_load(amwg_sampler* s, const uint8_t* const* images, const int64_t* sizes, int32_t n_images, int32_t dry_run);

/* sampler.start_adaptation() / stop_adaptation() -- mcmc.js:1060-1073 */
AMWG_API int amwg_set_adapting(amwg_sampler* s, int32_t flag);

/* stepper info() (mcmc.js:563-571): per component, chain-invariant counters and per-chain arrays.
 * scalars[c*3 + {0,1,2}] = is_adapting, iterations_since_adaption, batch_count  (host, length 3*n_comp)
 * prop_log_scale[c][chain], acceptance_count[c][chain] (host; either may be NULL) */
AMWG_API int amwg_info(amwg_sampler* s, double* scalars, double* prop_log_scale, int32_t* acceptance_count);

/* instrumentation */
AMWG_API int64_t amwg_kernel_launches(const amwg_sampler* s);   /* kernels this handle has launched so far       */
AMWG_API double amwg_last_sweep_kernel_ms(const amwg_sampler* s); /* CUDA-event time of the sweep kernels of the last burn/sample call */
AMWG_API uint64_t amwg_n_chains(const amwg_sampler* s);

AMWG_API const char* amwg_last_error(void);
AMWG_API int amwg_abi_version(void);

/* ld.* evaluated on the device, one value per input row (used by the `ld` host module and by the
 * parity tests): op is an AMWG_OP_LD_* / AMWG_OP_LGAMMA.. opcode, args is [n][arity] row-major. */
AMWG_API int amwg_ld_eval(int32_t op, const double* args, int32_t arity, int64_t n, double* out, int device);

/* Math.log / Math.exp / the Philox uniform stream on the device, for parity tests of the primitives.
 * kind: 0 log, 1 exp, 2 stream uniform (x[i] reinterpreted: out[i] = uniform #i of chain `chain`), 3 rnorm(x[0], x[1]) draws of
 * one chain, 4 Math.round, 5 the Poisson plate's table-driven exp (KS-level path; accuracy test) */
AMWG_API int amwg_primitive_eval(int32_t kind, const double* x, int64_t n, uint64_t seed, uint64_t chain, double* out, int device);

/* ---- post-path reductions on device (SURVEY 8(f).3) ------------------------------------------------------------------
 * The reference returns raw draws only (mcmc.js:1029; README.md:44-52 leaves the summary to the caller). With millions of
 * chains the summary is formed where the draws are. Both calls read a DEVICE-resident sample block in amwg_sample_device's
 * layout, x[row][entry][chain]; neither needs a sampler handle (they are reductions over the block).
 *
 * amwg_summary_moments: host_stats[entry][4] = { chains, mean of the per-chain means, M2 of the per-chain means
 *   (sum_c (m_c - mean)^2), sum over chains of the within-chain M2 (sum_r (x_rc - m_c)^2) }, merged in a fixed order
 *   (deterministic). Pooled mean / sd and the Gelman-Rubin statistic follow from these; shards (multi-GPU) merge exactly.
 *
 * amwg_summary_digit_hist: one pass (0..7, most significant byte first) of an exact radix select over the order-preserving
 *   64-bit key of the draws: dev_counts[entry][prefix][256] += number of values of `entry` whose key's top 8*pass bits equal
 *   dev_prefix[entry][prefix] and whose next byte is the bin (pass 0 ignores the prefixes). Integer counts: exact and
 *   order-independent; the caller sums them over GPUs, picks the byte holding each wanted order statistic and extends the
 *   prefixes. n_prefix <= 32.
 *
 * amwg_summary_autocov: split-chain autocovariances for the effective sample size and split R-hat (Vehtari et al. 2021, §3).
 *   Every chain is split into rows [0, h) and rows [rows-h, rows), h = rows/2 (for odd rows the middle row is in neither half):
 *   M = 2*chains half-chains of h draws. Series: the draws, plus, when host_thresholds[entry][2] is not null, the indicators
 *   1[x <= thresholds[entry][0]] and 1[x <= thresholds[entry][1]] (all formed from one pass over the block). Each half-chain
 *   is centred by its own mean. host_out[entry][series][4 + n_lags] = { M, mean of the half-chain means, M2 of the half-chain
 *   means, sum over half-chains of sum_n d_n^2, then for t = lag0 .. lag0+n_lags-1 the sum over half-chains of
 *   sum_{n<h-t} d_n d_{n+t} (= h * acov(t)) }. The first four merge like amwg_summary_moments' records, the lag sums add;
 *   both are formed in a fixed order (deterministic). Errors: rows < 2, n_lags outside 1..32, lag0 + n_lags > h, null
 *   dev_samples / host_out.
 *
 * Ranks over the pooled half-chain draws (rank-normalised R-hat and bulk ESS, Vehtari et al. 2021, §4). One entry per call; the
 * caller owns every device buffer (keys, indices, rank sums, z-block), so the three calls keep no state between them.
 * amwg_summary_rank_sort: sorts the n = 2*(rows/2)*chains half-chain draws of `entry` (numbered i = r*chains + c, r < 2h: rows
 *   [0, h) then rows [rows-h, rows); the middle row of odd rows is not ranked). Key: the order-preserving 64-bit key of x
 *   (centre NaN: the bulk series) or of |x - centre| (the folded series), with -0 made +0. dev_keys and dev_index hold 2n
 *   values each; on return dev_keys[0, n) is ascending and dev_index[0, n) holds each key's i (ties in ascending i: a stable
 *   LSD radix sort of 8-bit digits, so two calls give the same bits); [n, 2n) is scratch. Digit positions that are the same
 *   for all keys are skipped; *host_passes (when not null) receives the number of passes run (0..8). Errors: rows < 2, entry
 *   outside [0, entries), n >= 2^32, null dev_samples / dev_keys / dev_index.
 * amwg_summary_rank_count: for sorted key arrays Q[nq] (this shard's) and R[nr] (any shard's, or Q itself),
 *   dev_acc[i] += #(R < Q[i]) + #(R <= Q[i]) (merge path). Summed over all shards R, acc + 1 = twice the average rank
 *   (1-based, ties averaged) of Q[i] among all shards' keys. Integers: exact, independent of the order of the shards.
 *   Errors: nq or nr < 1 or >= 2^32, null pointers.
 * amwg_summary_rank_z: dev_z[dev_index[i]] = Phi^-1((r - 3/8) / (total + 1/4)), r = (dev_acc[i] + 1) / 2, for i < n; total is the
 *   number of ranked draws over all shards. Sized [2h][chains], dev_z is a [2h][1][chains] block whose two halves
 *   amwg_summary_autocov splits exactly as they were ranked. Errors: n outside 1..2^32-1, total < n or >= 2^52, null pointers.
 *
 * Posterior histograms (sample_summary(..., histogram=...)): three reductions over the block, integers or exact extremes, so the
 * results do not depend on the order of the atomics and sum (or min / max) across GPUs exactly.
 * amwg_summary_finite_range: dev_range[entry][2] = { smallest, largest finite draw } (+inf / -inf when the entry has none; -0 counts
 *   below +0) and dev_nonfinite[entry][3] = { #-inf, #+inf, #NaN }, both overwritten. Errors: an empty block, null pointers.
 * amwg_summary_histogram: dev_counts[entry][bins + 3] += the counts of the bins over dev_edges[entry][bins + 1] (device memory),
 *   then of the draws below edges[0] (-inf included), above edges[bins] (+inf included) and NaN; the caller zeroes the counts, as
 *   for digit_hist. The edges are numpy.linspace(lo, hi, bins + 1) and a draw lo <= x <= hi gets numpy.histogram's bin (the
 *   operations of its equal-width fast path: csrc/amwg_hist.cuh). Errors: bins outside 1..4096, rows >= 2^32, an empty block,
 *   null pointers.
 * amwg_summary_histogram2d: dev_counts[pair][bins][bins] += the 2-D histogram of entries host_pairs[pair][0] (axis 0) and
 *   host_pairs[pair][1] (axis 1) over their rows of dev_edges[entry][bins + 1], by numpy.histogramdd's rule (per axis
 *   searchsorted(edges, v, "right") - 1, the last edge in the last bin); a draw counts only when both values fall inside (NaN
 *   never does). host_pairs is host memory. Errors: bins outside 1..128, n_pairs outside 1..64, a pair entry outside
 *   [0, entries), rows >= 2^32, an empty block, null pointers.
 *
 * Posterior covariance (sample_summary(..., covariance=...)): the matrix form of amwg_summary_moments' record, for the n_sel
 * entries host_sel[0 .. n_sel) (host memory).
 * amwg_summary_comoments: host_out[1 + n_sel + 2 n_sel^2] = { C (chains), m[n_sel] (mean of the chain means),
 *   B[n_sel][n_sel] = sum_c (xbar_c - m)(xbar_c - m)^T (co-M2 of the chain means), W[n_sel][n_sel] = sum_c sum_r (x_rc - xbar_c)
 *   (x_rc - xbar_c)^T (summed within-chain co-M2) }, row-major and exactly symmetric. xbar_c is a sequential sum over the rows
 *   divided by rows; m sums the chain means in a fixed order. B and W are Gram matrices of the centred values, formed on the fp64
 *   tensor core (mma.sync m8n8k4) by a grid whose size depends on chains only and summed in a fixed order: two calls give the
 *   same bits. A NaN or +-inf draw of an entry makes that entry's rows and columns of B and W NaN. Records of shards merge like
 *   amwg_summary_moments' (Chan, in matrix form). Device scratch, from a per-device pool grown on demand: with T = nb (nb + 1) / 2
 *   tiles, nb = ceil(n_sel / 8), R = 1 when T >= 16 else floor(16 / T) warps per tile and G = min(ceil(chains / 32), 264) CTAs,
 *   8 (n_sel chains + n_sel + 64 T R G + 128 T) bytes, each of the four parts rounded up to 256 bytes. Errors (nothing is touched): an empty block, n_sel outside 1..128, null
 *   pointers, a selected entry outside [0, entries), rows * chains >= 2^53.
 *
 * Nested R-hat (sample_summary(..., nested=M), DESIGN.md §4.6): superchain k is the global chains [k M, (k + 1) M); the block
 * holds the global chains [first_chain, first_chain + chains).
 * amwg_summary_nested: host_out[entry][14]. Per chain, its mean and M2 over the rows (two sequential passes); per superchain the
 *   shard touches, its chains' records (1, mean, 0, M2) merged in chain order into (chains, mean of the chain means, M2 of the chain
 *   means, sum of the within-chain M2). host_out[entry][0..3] = the complete superchains, each as the unit (1, superchain mean, 0,
 *   B~_k + W-_k) with B~_k = M2 of its chain means / (M - 1) (0 when M = 1) and W-_k = its within-chain M2 / (M (rows - 1)) (0 when
 *   rows = 1), Chan-merged in a fixed order; then two cut records { superchain id, chains, mean of the chain means, M2 of the chain
 *   means, sum of the within-chain M2 } for the first and the last superchain when the range cuts them (id -1 and zeros when not).
 *   The grid depends on chains and the number of superchains touched only: two calls give the same bits. Records of shards merge
 *   like amwg_summary_moments' (summary.merge_nested_records). Device scratch, from a per-device pool grown on demand, with S the
 *   superchains touched and G = min(ceil(S / 256), 1184): 16 entries chains + 32 entries G + 32 entries + 64 entries bytes, each
 *   part rounded up to 256 bytes. Errors (nothing is touched): an empty block, null pointers, superchain_size < 1,
 *   first_chain < 0, first_chain + chains > 2^53. */
AMWG_API int amwg_summary_moments(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, double* host_stats);
AMWG_API int amwg_summary_digit_hist(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int32_t pass,
                                     const uint64_t* dev_prefix, int32_t n_prefix, uint64_t* dev_counts);
AMWG_API int amwg_summary_autocov(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                  const double* host_thresholds, int64_t lag0, int32_t n_lags, double* host_out);
AMWG_API int amwg_summary_rank_sort(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int32_t entry,
                                    double centre, uint64_t* dev_keys, uint32_t* dev_index, int32_t* host_passes);
AMWG_API int amwg_summary_rank_count(int device, const uint64_t* dev_q, int64_t nq, const uint64_t* dev_r, int64_t nr, int64_t* dev_acc);
AMWG_API int amwg_summary_rank_z(int device, const int64_t* dev_acc, const uint32_t* dev_index, int64_t n, int64_t total, double* dev_z);
AMWG_API int amwg_summary_finite_range(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                       double* dev_range, int64_t* dev_nonfinite);
AMWG_API int amwg_summary_histogram(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                    const double* dev_edges, int32_t bins, int64_t* dev_counts);
AMWG_API int amwg_summary_histogram2d(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                      const int32_t* host_pairs, int32_t n_pairs, const double* dev_edges, int32_t bins, int64_t* dev_counts);
AMWG_API int amwg_summary_comoments(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                    const int32_t* host_sel, int32_t n_sel, double* host_out);
AMWG_API int amwg_summary_nested(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains, int64_t first_chain,
                                 int64_t superchain_size, double* host_out);

/* ---- PSIS-LOO and WAIC (sample_summary(..., loo=...), DESIGN.md §4.7) ------------------------------------------------------
 * amwg_loo_pointwise: dev_out[row][p][chain] = the pointwise log-likelihood at point p0 + p (p < n_points) of the kept draw (row,
 *   chain) of dev_samples, a block in amwg_sample_device's layout [rows][entries][chains] with chains = the handle's chains. The
 *   program (host_code[n_code], constants host_consts[n_consts]) is an expression program: body_prog leaves the value and ends
 *   with END; COMP and COMP_I address block ENTRIES (the host maps every component the body reads to its entry); DATA_I / COMP_I
 *   read the handle's data columns at the point index. Before the body runs, each fold program host_fold_prog[k] (in order) is
 *   evaluated on the device into constant host_fold_dst[k], as amwg_create folds the model's constants. One thread per (row,
 *   chain) runs the model's interpreter over the points; the output is the sample-block layout with points as entries, so the
 *   amwg_summary_* reductions read it unchanged. Errors (nothing runs): a malformed program, one that is not an expression (sums,
 *   plates, loops, stores, cache words), a constant, entry or fold index out of range, a data read outside its column at some point
 *   of the range, a COMP_I data value that is not an entry, program and constants over 200 KB.
 * amwg_loo_reduce: over a chunk dev_ll[rows][points][chains] and per point the host's llmin, llmax (smallest / largest finite ll)
 *   and cut: host_sums[point][3] = { sum exp(ll - llmax) over all draws, sum exp(lw) and sum exp((lw + ll) - llmin) over the draws
 *   with lw = llmin - ll <= cut }, each formed in a fixed order (deterministic); every draw with lw > cut has its ll appended to
 *   dev_tail[point][tail_cap] at slot dev_count[point]++ (int32, zeroed by the caller; slots past tail_cap are counted, not
 *   written). Errors: an empty block, points > 65535, tail_cap outside 1..2^20, null pointers.
 * amwg_loo_fit: one CTA per point gathers the tails dev_tails[shard][point][tail_cap] (dev_counts[shard][point] values each),
 *   sorts them and fits a generalised Pareto to the ascending exp(lw) - exp(cut), lw = llmin - ll (Zhang & Stephens 2009 with
 *   the prior on k; csrc/amwg_loo.cuh). host_out[point][4] = { k, sum exp(lw), sum exp((lw + ll) - llmin) over the tail with lw
 *   replaced by the smoothed weights when k is finite, the tail draws over all shards }; a tail of <= 4 draws, or one where no
 *   candidate of the fit has a finite profile value, gives k = +inf and raw weights; host_skip[point] != 0 gives NaN. Deterministic. Errors: tail_cap not a power of two in 8..2^20, shards or points
 *   < 1, null pointers.
 * Device scratch of the three calls, from one per-device pool grown on demand: the program (pointwise), 3 x 8 points + 24 points
 *   G (G = min(ceil(chains / 256), 1184)) bytes (reduce), 3 x 8 points + 16 points tail_cap + 32 points bytes (fit). */
AMWG_API int amwg_loo_pointwise(amwg_sampler* s, const int32_t* host_code, int32_t n_code, const double* host_consts, int32_t n_consts,
                                int32_t body_prog, const int32_t* host_fold_prog, const int32_t* host_fold_dst, int32_t n_fold,
                                const double* dev_samples, int64_t rows, int32_t entries, int64_t p0, int32_t n_points, double* dev_out);
AMWG_API int amwg_loo_reduce(int device, const double* dev_ll, int64_t rows, int32_t points, int64_t chains, const double* host_llmin,
                             const double* host_llmax, const double* host_cut, int32_t tail_cap, double* dev_tail, int32_t* dev_count,
                             double* host_sums);
AMWG_API int amwg_loo_fit(int device, const double* dev_tails, const int32_t* dev_counts, int32_t shards, int32_t points, int32_t tail_cap,
                          const double* host_llmin, const double* host_cut, const int32_t* host_skip, double* host_out);

/* ---- posterior predictive checks (sample_summary(..., ppc=...), DESIGN.md §4.8) -----------------------------------------------
 * amwg_ppc_pointwise: dev_out[row][p][chain] = a replicated observation y_rep of point p0 + p (p < n_points, of `points` points in
 *   all) at the kept draw (row, chain) of dev_samples ([rows][entries][chains], chains = the handle's chains), drawn from family
 *   `family` (csrc/amwg_ppc.cuh: 0 norm, 1 lnorm, 2 cauchy, 3 laplace, 4 logis, 5 exp, 6 weibull, 7 pareto, 8 unif, 9 gamma,
 *   10 invgamma, 11 beta, 12 t, 13 bern, 14 pois, 15 binom, 16 nbinom) whose n_args parameters are the values of the expression
 *   programs host_arg_progs[k] at the point (programs, constants and fold programs as amwg_loo_pointwise's, each program leaving
 *   one value). The draw of (row, point i) for global chain g takes the uniforms #(2^62 + (row points + i) 2^16 + k) of chain g's
 *   Math.random() stream, keyed by the handle's seed; one needing k >= 2^16, or parameters outside the family's domain, give NaN.
 *   dev_stats[row][4][chain] carries each draw's running statistics of its replicated dataset over the points in index order
 *   (Welford mean, M2, min, max; min and max propagate NaN): the call with p0 = 0 starts them, and the call whose chunk ends at
 *   `points` replaces M2 by sd = sqrt(M2 / (points - 1)), leaving the sample block (mean, sd, min, max). Errors (nothing runs): as
 *   amwg_loo_pointwise, an unknown family, n_args not the family's parameter count, p0 + n_points > points, rows x points >= 2^46.
 * amwg_summary_threshold_counts: dev_counts[entry][4] (int64, overwritten) = the draws of each entry of a sample block
 *   [rows][entries][chains] that are < host_thresholds[entry], ==, >, and NaN; exact and independent of order. Errors: an empty
 *   block, entries > 65535, null pointers.
 * Device scratch, from the pool of the LOO calls: the programs (pointwise), 8 entries bytes (counts). */
AMWG_API int amwg_ppc_pointwise(amwg_sampler* s, const int32_t* host_code, int32_t n_code, const double* host_consts, int32_t n_consts,
                                int32_t family, const int32_t* host_arg_progs, int32_t n_args, const int32_t* host_fold_prog,
                                const int32_t* host_fold_dst, int32_t n_fold, const double* dev_samples, int64_t rows, int32_t entries,
                                int64_t points, int64_t p0, int32_t n_points, double* dev_out, double* dev_stats);
AMWG_API int amwg_summary_threshold_counts(int device, const double* dev_samples, int64_t rows, int32_t entries, int64_t chains,
                                           const double* host_thresholds, int64_t* dev_counts);

/* ---- run-time specialisation ----------------------------------------------------------------------------------------------
 * For models that run the statistics sweep (stat_prog) amwg_create generates CUDA source from the model's programs, compiles it
 * for sm_90a with NVRTC and steps with that kernel instead of the bytecode interpreter (csrc/amwg_jit.cuh; AMWG_JIT=0 in the
 * environment keeps the interpreter, AMWG_JIT=1 specialises whatever the number of chains). amwg_jit_status: 1 when the handle
 * runs a specialised kernel, with a one-line description (or the reason it does not) in `note`. amwg_jit_compile_check: generate
 * and compile without a GPU (0 compiled, 1 model not eligible, -1 error; message in `log`, generated source in `src`). */
AMWG_API int amwg_jit_status(const amwg_sampler* s, char* note, int64_t cap);
AMWG_API int amwg_jit_compile_check(const amwg_model* model, uint64_t n_chains, char* log, int64_t log_cap, char* src, int64_t src_cap);
/* amwg_plate_sources: where the interpreter kernels (init, sweeps, the log_post re-evaluation) read each plate's column, in plate
 * order, comma-separated: "shared" (resident), "ring" (the TMA tile ring), "L2" (global loads) or "loop" (a bytecode plate).
 * Returns the number of plates. */
AMWG_API int amwg_plate_sources(const amwg_sampler* s, char* out, int64_t cap);
/* amwg_get_term_cache (read-only; for tests of the cached values): copies the term cache, host_out[t][chain] for t < n_terms
 * (amwg_model.n_terms), to the host and returns n_terms; 0 for a handle that keeps no term cache. Slots 0 .. n_sum_terms-1 hold
 * the terms of the sum at the chain's current state; with stat_prog, slots n_sum_terms .. n_terms-1 hold each plate statistic S
 * at the current state. The sweep kernels write the cache back at the end of every launch, so it is current whenever
 * amwg_burn / amwg_sample have returned. An error (with a message) when cap, the number of doubles host_out holds, is too small. */
AMWG_API int amwg_get_term_cache(amwg_sampler* s, double* host_out, int64_t cap);

/* ---- measurement ---------------------------------------------------------------------------------------------------------
 * The binding roof of this path is the non-tensor fp64 pipe (DADD + DFMA per data point), which MEASURED_PEAKS.json does not
 * hold: amwg_peak_fp64 measures it (TFLOP/s, 2 flop per DFMA; best of `reps` launches of a DFMA-chain kernel that fills every SM,
 * CUDA events on the launching stream). bench.py reports roofline fractions against this number, taken in the same process. */
AMWG_API int amwg_peak_fp64(int device, int reps, double* tflops_out, double* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* AMWG_H_ */
