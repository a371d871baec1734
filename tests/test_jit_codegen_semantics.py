"""What the code generator prints, executed -- without a GPU.

tests/test_jit_codegen.py checks that the specialised full-program sweep of a model COMPILES for sm_90a; the GPU tests check that it
draws what the interpreter kernels draw. This file closes the gap on the CPU tier: the generated `jit_logpost()` / `jit_derived()`
(csrc/amwg_jit.cuh) is compiled for the host together with the product's own arithmetic headers and the plate helpers of the kernel
skeleton (csrc/amwg_jit_full_kernel.cuh, taken from the file's text) and evaluated at random states, moved components and proposal
values against tests/prog_eval.py -- the bytecode run with the oracle's arithmetic, which tests/test_tracer.py in turn holds against
the oracle's C models. Bit for bit: the generated code performs the program's operations in the program's order.

Constants that the library folds on the device at create (log(2*pi), lbeta(2,2) ...) are folded here by prog_eval with the oracle's
arithmetic and written into the model descriptor before the generator sees it, exactly what try_jit() reads back from the device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import models
import prog_eval
from conftest import NORM_DATA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bayes.js_b200", "csrc")

HOST_PRELUDE = r'''
#include "cuda_runtime.h"      // tests/host_shim
#include "math_constants.h"
#include <cstdarg>
#include <cstdio>
#define __constant__
static unsigned char* g_smem_base = nullptr;                    // "shared memory": a host buffer, addressed by offset
static unsigned g_smem_limit = 0;                               // its size: every load must lie below it
static char g_fault[2048];                                      // the first breach of the device's rules; the harness reads it after each call
static void hs_fault(const char* fmt, ...) {
  if (g_fault[0]) return;
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_fault, sizeof g_fault, fmt, ap);
  va_end(ap);
}
namespace amwg {
static inline unsigned smem_u32(const void* p) { return (unsigned)((const unsigned char*)p - g_smem_base); }
// an n-byte ld.shared at offset a: aligned to n (a misaligned one faults on the device) and inside the CTA's shared memory
static inline bool lds_ok(unsigned a, unsigned n) {
  if (a % n) { hs_fault("misaligned %u-byte shared-memory load at offset %u", n, a); return false; }
  if ((unsigned long long)a + n > g_smem_limit) { hs_fault("%u-byte shared-memory load at offset %u, past the %u bytes declared", n, a, g_smem_limit); return false; }
  return true;
}
static inline double lds_f64_sa(unsigned a) { double v = 0.0; if (lds_ok(a, 8)) std::memcpy(&v, g_smem_base + a, 8); return v; }
}
#include "amwg_math.cuh"
#include "amwg_ld.cuh"
'''

HOST_EXPORTS = r'''
extern "C" {
void hs_set_smem(unsigned char* p, unsigned n) { g_smem_base = p; g_smem_limit = n; }
const char* hs_fault_msg() { return g_fault; }
int hs_n_res() { return JN_RES; }
unsigned hs_res_off(int k) { return amwg::JRES_OFF[k]; }
int hs_res_col(int k) { return amwg::JRES_COL[k]; }
int hs_n_bern() { return JN_BERN; }
unsigned hs_bern_data(int k) { return amwg::JBERN_DATA[k]; }
int hs_bern_n(int k) { return amwg::JBERN_N[k]; }
unsigned hs_bern_mask(int k) { return amwg::JBERN_MASK[k]; }
double hs_logpost(const double* state, int moved, double val) { return amwg::jit_logpost(g_smem_base, state, 1ull, moved, val); }
void hs_derived(const double* state, double* der) {
#if JN_DERIVED > 0
  amwg::jit_derived(g_smem_base, state, 1ull, der);
#else
  (void)state; (void)der;
#endif
}
}
'''


def _compile(cpp, so):
    """g++ for the host. AMWG_HOST_SANITIZE=address builds with AddressSanitizer (the process must then preload libasan: see
    test_jit_codegen_fuzz.py's ASan run)."""
    extra = ["-fsanitize=address", "-fno-omit-frame-pointer", "-g"] if os.environ.get("AMWG_HOST_SANITIZE") == "address" else []
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", *extra, "-I" + os.path.join(ROOT, "tests", "host_shim"),
                        "-I" + CSRC, str(cpp), "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    lib = C.CDLL(str(so))
    lib.hs_fault_msg.restype = C.c_char_p
    return lib


def _skeleton_helpers():
    """the macros and plate helpers of the kernel skeleton: its text from `#define ST(c)` to the end of the first namespace block"""
    text = open(os.path.join(CSRC, "amwg_jit_full_kernel.cuh")).read()
    a = text.index("#define ST(c)")
    b = text.index("}  // namespace amwg", a)
    return "namespace amwg {\n" + text[a:b] + "}  // namespace amwg\n"


class HostProgram:
    def __init__(self, pkg, orc, tmp_path, params, log_post, data, _opts=None, **opts):
        o = {"chains": 4096, "_model_only": True}
        o.update(opts)
        o.update(_opts or {})                                        # sampler options that may themselves be called `params`
        self.s = s = pkg.mcmc.AmwgSampler(params, log_post, data, o)
        self.prog, self.O = s._program, orc.lib()
        self.consts = prog_eval.fold_constants(self.prog, self.O)
        m = s._model_keepalive[-1]
        for i, v in enumerate(self.consts):                           # what try_jit() reads back from the device after folding
            m.consts[i] = float(v)
        if o.get("_force_full"):                                      # what AMWG_TERM_CACHE=0 does in amwg_create: every step runs the full program
            m.n_terms = 0
        rc, msg, src = s.jit_compile_check()
        assert rc == 0, msg
        assert "#define JFULL 1" in src
        self.src, self.msg = src, msg
        cpp = tmp_path / "gen.cpp"
        # the generated text = the #define prelude (up to the first namespace block), then tables and programs
        cut = src.index("namespace amwg {")
        cpp.write_text(src[:cut] + HOST_PRELUDE + _skeleton_helpers() + src[cut:] + HOST_EXPORTS)
        self.lib = L = _compile(cpp, tmp_path / "gen.so")
        L.hs_logpost.restype, L.hs_logpost.argtypes = C.c_double, [C.POINTER(C.c_double), C.c_int, C.c_double]
        L.hs_derived.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double)]
        for f in ("hs_res_off", "hs_bern_data", "hs_bern_mask"):
            getattr(L, f).restype = C.c_uint
        # stage the data the way the kernel does: resident columns by bulk copy, Bernoulli columns also as bit masks + "bad point" word
        self.smem = np.zeros(1 << 18, dtype=np.uint8)
        for k in range(L.hs_n_res()):
            col = np.asarray(self.prog.columns[L.hs_res_col(k)], dtype=np.float64)
            off = L.hs_res_off(k)
            self.smem[off:off + 8 * col.size] = col.view(np.uint8)
        for k in range(L.hs_n_bern()):
            n, d0, m0 = L.hs_bern_n(k), L.hs_bern_data(k), L.hs_bern_mask(k)
            y = self.smem[d0:d0 + 8 * n].view(np.float64)
            words = np.zeros((n + 31) // 32 + 1, dtype=np.uint32)
            for i in range(n):
                if y[i] == 1.0:
                    words[i >> 5] |= np.uint32(1 << (i & 31))
            words[-1] = 1 if np.any(~((y == 1.0) | (y == 0.0))) else 0
            self.smem[m0:m0 + 4 * words.size] = words.view(np.uint8)
        L.hs_set_smem(self.smem.ctypes.data_as(C.POINTER(C.c_ubyte)), self.smem.size)
        self.D = self.prog.n_comp if hasattr(self.prog, "n_comp") else int(m.n_comp)
        self.types = []                                             # per component: (type, lower, upper)
        for p in range(m.n_params):
            pa = m.params[p]
            self.types += [(pa.type, pa.lower, pa.upper)] * pa.n_comp

    def random_state(self, rng):
        st = np.empty(self.D)
        for c, (t, lo, hi) in enumerate(self.types):
            st[c] = self.random_value(rng, t, lo, hi)
        return st

    @staticmethod
    def random_value(rng, t, lo, hi):
        if t == 2:                                                  # binary
            return float(rng.integers(0, 2))
        a = lo if np.isfinite(lo) else (hi - 20 if np.isfinite(hi) else -10.0)
        b = hi if np.isfinite(hi) else a + 20
        v = rng.uniform(a, b)
        if rng.random() < 0.05:                                     # now and then a value outside the support: -Infinity / NaN paths
            v = a - 1.5 if rng.random() < 0.5 else b + 1.5
        return float(np.floor(v + 0.5)) if t == 1 else float(v)

    def check(self, rng, trials=300):
        n_der = len(self.s._derived_names)
        for _ in range(trials):
            st = self.random_state(rng)
            moved = int(rng.integers(-1, self.D))
            val = self.random_value(rng, *self.types[moved]) if moved >= 0 else 0.0
            got = self.lib.hs_logpost(st.ctypes.data_as(C.POINTER(C.c_double)), moved, val)
            want = prog_eval.logpost(self.prog, self.consts, st, self.O, moved=moved, val=val)
            assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64) or (got != got and want != want), (st, moved, val, got, want)
            if n_der:
                der = np.full(n_der, np.nan)
                self.lib.hs_derived(st.ctypes.data_as(C.POINTER(C.c_double)), der.ctypes.data_as(C.POINTER(C.c_double)))
                ref = [None] * n_der
                pc = self.prog.derived_prog
                if self.prog.variant_comps:
                    v = sum((1 << k) for k, c in enumerate(self.prog.variant_comps) if st[c] != 0)
                    pc = self.prog.variant_derived[v]
                prog_eval.run(self.prog, self.consts, st, pc, self.O, der=ref)
                assert [np.float64(x).view(np.uint64) for x in der] == [np.float64(x).view(np.uint64) for x in ref]
        assert not self.lib.hs_fault_msg(), self.lib.hs_fault_msg().decode()


def _cases(pkg):
    ld, mcmc = pkg.ld, pkg.mcmc
    rng = np.random.default_rng(5)
    y = (rng.random(77) < 0.7).astype(float).tolist()
    nb = [int(v) for v in rng.integers(5, 30, 12)]

    def norm_derived(state, data):
        lp = 0
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], state.mu, state.sigma)
        state.cv = state.sigma / state.mu
        state.var = state.sigma * state.sigma
        return lp
    return {
        "spike_where": (models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y}, {}),
        "spike_literal": (models.PARAMS_SPIKE, models.spike_bern_literal(ld), {"x": y}, {}),
        "spike_bad_point": (models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y[:40] + [2.0] + y[41:]}, {}),
        "complex_literal": (models.PARAMS_COMPLEX, models.complex_model_post_literal(ld), nb, {}),
        "complex_where": (models.PARAMS_COMPLEX, models.complex_model_post(ld, mcmc), nb, {}),
        "norm_faithful_derived": ({"mu": {"type": "real", "init": 180}, "sigma": {"type": "real", "lower": 0, "init": 5}}, norm_derived,
                                  rng.normal(184.5, 4.5, 64).tolist(), {"faithful": True}),
        "multi_bern": ({"x": {"type": "binary", "dim": [2, 2]}}, models.multi_bern_dens(mcmc), None, {}),
        "beta_bern_faithful": (models.PARAMS_THETA, models.beta_bern(ld), {"x": y}, {"faithful": True}),
        # tests/test_data.js:80-91: the Normal model that also writes the derived quantity par.var = sigma^2
        "norm_test_faithful": (models.PARAMS1, models.norm_post_test(ld), NORM_DATA, {"faithful": True}),
    }


@pytest.mark.parametrize("name", ["spike_where", "spike_literal", "spike_bad_point", "complex_literal", "complex_where", "norm_faithful_derived",
                                  "multi_bern", "beta_bern_faithful", "norm_test_faithful"])
def test_generated_log_post_equals_the_program(pkg, orc, tmp_path, name):
    params, f, data, opts = _cases(pkg)[name]
    hp = HostProgram(pkg, orc, tmp_path, params, f, data, **opts)
    hp.check(np.random.default_rng(11))


# ---- the whole specialised kernel on the host: skeleton + generated code, one emulated thread per CTA -----------------------------
KERNEL_SHIM = r'''
#include <cstdlib>
#include <map>
#include <vector>
#define __global__
#define __launch_bounds__(...)
#define __grid_constant__
#define __shared__
#define __align__(n)
struct hs_dim3 { unsigned x = 0, y = 0, z = 0; };
static hs_dim3 threadIdx, blockIdx, blockDim;
static inline void __syncthreads() {}
namespace amwg {
// The CTA's dynamic shared memory (`extern __shared__ ... smem[]` in the kernel): exactly the bytes the launch declares, allocated
// on its own so that AddressSanitizer bounds it too, and filled with 0xff (NaN) before every CTA: the device hands no CTA another
// one's contents. `hs_presets` are what the harness writes in place of code the host cannot run (the ballot loop).
static unsigned char* smem = nullptr;
static unsigned smem_bytes = 0;
static std::vector<std::pair<unsigned, std::vector<unsigned char>>> hs_presets;
// The device allocations a bulk copy may read: the data columns, laid out as amwg_create's dev_upload lays them out.
struct HsAlloc { const unsigned char* p; unsigned long long n; };
static std::vector<HsAlloc> hs_allocs;
// One mbarrier: arrivals still pending in its current phase, transaction bytes announced (expect_tx) and delivered (bulk copies).
struct HsBar { unsigned count, pending, phase; unsigned long long expect, delivered; };
static std::map<const void*, HsBar> hs_bars;

static HsBar* hs_bar(const unsigned long long* bar, const char* what) {
  auto it = hs_bars.find(bar);
  if (it == hs_bars.end()) { hs_fault("%s on an mbarrier that was never initialised", what); return nullptr; }
  return &it->second;
}
static inline void mbar_init(unsigned long long* bar, unsigned count) { hs_bars[bar] = HsBar{count, count, 0u, 0ull, 0ull}; }
static inline void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {        // mbarrier.arrive.expect_tx: one arrival + bytes
  HsBar* b = hs_bar(bar, "mbar_expect_tx");
  if (!b) return;
  if (b->pending == 0) { hs_fault("mbar_expect_tx: an arrival on an mbarrier whose %u arrival(s) of this phase have all happened", b->count); return; }
  b->pending -= 1;
  b->expect += bytes;
  if (b->expect > 0xfffffull) hs_fault("mbar_expect_tx: %llu transaction bytes in one phase, beyond the 2^20 - 1 an mbarrier counts", b->expect);
}
static inline void mbar_wait(unsigned long long* bar, unsigned parity) {
  HsBar* b = hs_bar(bar, "mbar_wait");
  if (!b) return;
  if (parity != b->phase)
    hs_fault("mbar_wait on parity %u while the mbarrier is in phase %u: on the device the wait returns before the data lands", parity, b->phase);
  else if (b->pending != 0 || b->delivered != b->expect)
    hs_fault("mbar_wait would hang on the device: %llu transaction bytes expected, %llu delivered, %u arrival(s) pending",
             b->expect, b->delivered, b->pending);
  b->phase ^= 1u;                                                 // the phase completes: one thread per CTA has nobody to wait for
  b->pending = b->count;
  b->expect = b->delivered = 0;
}
static inline void tma_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {      // cp.async.bulk global -> shared
  const uintptr_t d = (uintptr_t)dst, s = (uintptr_t)src, lo = (uintptr_t)smem;
  const long long doff = (long long)(d - lo);
  HsBar* b = hs_bar(bar, "tma_bulk_g2s");
  if (!b) return;
  if (s % 16 || d % 16) { hs_fault("tma_bulk_g2s: %u bytes from %p to shared offset %lld: source and destination must be 16-byte aligned", bytes, src, doff); return; }
  if (bytes == 0 || bytes % 16) { hs_fault("tma_bulk_g2s: %u bytes to shared offset %lld: the size must be a positive multiple of 16", bytes, doff); return; }
  if (d < lo || d + bytes > lo + smem_bytes) {
    hs_fault("tma_bulk_g2s: %u bytes to shared offset %lld, outside the %u bytes of dynamic shared memory the launch declares", bytes, doff, smem_bytes);
    return;
  }
  const HsAlloc* a = nullptr;
  for (const HsAlloc& x : hs_allocs) if (s >= (uintptr_t)x.p && s < (uintptr_t)x.p + x.n) a = &x;
  if (!a) { hs_fault("tma_bulk_g2s: %u bytes from %p, which lies in no device allocation", bytes, src); return; }
  if (s + bytes > (uintptr_t)a->p + a->n) {
    hs_fault("tma_bulk_g2s: %u bytes from %llu bytes into a %llu-byte device allocation: the copy runs past its end", bytes,
             (unsigned long long)(s - (uintptr_t)a->p), a->n);
    return;
  }
  std::memcpy(dst, src, bytes);
  b->delivered += bytes;
}
}
'''

# What both kernels' exports share: the declared shared memory, the device allocations, the first fault, and the shim's own functions
# (test_the_strict_shim_refuses_* calls them directly).
CONTRACT_EXPORTS = r'''
extern "C" {
void hs_set_dyn_smem(unsigned bytes) {
  std::free(amwg::smem);
  void* p = nullptr;
  if (posix_memalign(&p, 16, bytes ? bytes : 1) != 0) std::abort();
  amwg::smem = (unsigned char*)p;
  amwg::smem_bytes = bytes;
  std::memset(amwg::smem, 0xff, bytes);
  amwg::hs_presets.clear();
  g_smem_base = amwg::smem; g_smem_limit = bytes;
}
unsigned char* hs_kernel_smem() { return amwg::smem; }
void hs_preset(unsigned off, const unsigned char* p, unsigned n) { amwg::hs_presets.emplace_back(off, std::vector<unsigned char>(p, p + n)); }
void hs_clear_allocs() { amwg::hs_allocs.clear(); }
void hs_register_alloc(const void* p, unsigned long long n) { amwg::hs_allocs.push_back(amwg::HsAlloc{(const unsigned char*)p, n}); }
const char* hs_fault_msg() { return g_fault; }
void hs_clear_fault() { g_fault[0] = 0; }
void hs_mbar_init(unsigned long long* bar, unsigned count) { amwg::mbar_init(bar, count); }
void hs_mbar_expect_tx(unsigned long long* bar, unsigned bytes) { amwg::mbar_expect_tx(bar, bytes); }
void hs_mbar_wait(unsigned long long* bar, unsigned parity) { amwg::mbar_wait(bar, parity); }
void hs_tma_bulk_g2s(unsigned long long dst_off, const void* src, unsigned bytes, unsigned long long* bar) {
  amwg::tma_bulk_g2s(amwg::smem + dst_off, src, bytes, bar);
}
}
// a fresh CTA: nothing in its shared memory but what the harness presets
static void hs_cta_begin(unsigned x) {
  std::memset(amwg::smem, 0xff, amwg::smem_bytes);
  for (const auto& pr : amwg::hs_presets) std::memcpy(amwg::smem + pr.first, pr.second.data(), pr.second.size());
  g_smem_base = amwg::smem; g_smem_limit = amwg::smem_bytes;
  blockDim.x = 1; threadIdx.x = 0; blockIdx.x = x;
}
'''

KERNEL_EXPORTS = CONTRACT_EXPORTS + r'''
extern "C" {
double hs_exp_of(double x) { return amwg::js_exp(x); }
void hs_sweep(double* state, double* psd, int* acc, double* curr_lp, unsigned long long* perm, unsigned long long* rng_n,
              unsigned long long C, unsigned long long first_chain, unsigned long long seed, long long n_sweeps, long long sample_i0,
              long long thin, int record, int n_monitor, const int* monitor, double* out, const double** cols, int n_cols,
              const unsigned char* adapting, unsigned char* perm_ext, unsigned short* order_ext) {
  amwg::JitArgs A{};
  A.a.state = state; A.a.psd = psd; A.a.acc = acc; A.a.curr_lp = curr_lp; A.a.perm = perm; A.a.rng_n = rng_n;
  A.a.perm_ext = perm_ext; A.a.order_ext = order_ext;           // > 16 named parameters / dim[0] > 256 (amwg_tma.cuh), else null
  A.a.C = C; A.a.first_chain = first_chain; A.a.seed = seed;
  A.sa.n_sweeps = n_sweeps; A.sa.sample_i0 = sample_i0; A.sa.thin = thin; A.sa.record = record; A.sa.n_monitor = n_monitor;
  A.sa.monitor = monitor; A.sa.out = out;
  for (int k = 0; k < n_cols; ++k) A.col[k] = cols[k];
  A.adapting = adapting;
  for (unsigned long long c = 0; c < C && !g_fault[0]; ++c) { hs_cta_begin((unsigned)c); amwg::amwg_jit_sweep(A); }   // one thread per CTA: chain = blockIdx.x
}
}
'''


def _smem_bytes(msg):
    """the dynamic shared memory a launch of the compiled specialisation declares (amwg_jit_compile_check's message)"""
    m = re.search(r"(\d+) B shared memory", msg)
    assert m, msg
    return int(m.group(1))


def device_columns(columns):
    """the model's data columns as amwg_create uploads them (dev_upload): 16-byte aligned, zero-padded to a multiple of 16 bytes and
    to at least 16"""
    out = []
    for c in columns:
        v = np.asarray(c, dtype=np.float64).ravel()
        n = max(2 * ((v.size + 1) // 2), 2)
        raw = np.zeros(n + 1)
        a = raw[(-raw.ctypes.data % 16) // 8:][:n]
        a[:v.size] = v
        out.append(a)
    return out


class StrictShim:
    """What the kernel harnesses share: the kernel `K` compiled with the strict shim, the dynamic shared memory its launch declares,
    its device columns, and the check after every launch, which fails with the kernel's staging tables when the shim saw a breach."""

    def _shim_setup(self, K, src, msg):
        K.hs_kernel_smem.restype = C.POINTER(C.c_ubyte)
        K.hs_register_alloc.argtypes = [C.c_void_p, C.c_ulonglong]
        K.hs_preset.argtypes = [C.c_uint, C.c_void_p, C.c_uint]
        self.K, self.src, self.smem_bytes = K, src, _smem_bytes(msg)
        K.hs_set_dyn_smem(self.smem_bytes)

    def _upload(self, columns):
        cols = device_columns(columns)
        self.K.hs_clear_allocs()
        for c in cols:
            self.K.hs_register_alloc(c.ctypes.data, c.nbytes)
        colp = (C.POINTER(C.c_double) * max(len(cols), 1))(*[c.ctypes.data_as(C.POINTER(C.c_double)) for c in cols])
        return cols, colp

    def _contract(self, cols):
        msg = self.K.hs_fault_msg()
        if msg:
            tables = [ln for ln in self.src.splitlines()
                      if re.match(r"#define (JN_RES|JRES_TOTAL_BYTES|JSTREAM|JS_COL|JS_BEGIN|JS_TOTAL|JRING_\w+|JWS_\w+|JTHREADS|JN_BERN)\b", ln)
                      or re.search(r"\b(JRES|JBERN)_\w+\[", ln)]
            raise AssertionError(f"{msg.decode()}\n  declared dynamic shared memory: {self.smem_bytes} B; device columns: "
                                 f"{[c.nbytes for c in cols]} B\n  " + "\n  ".join(tables))


def _tma_structs():
    text = open(os.path.join(CSRC, "amwg_tma.cuh")).read()
    a = text.index("struct ChainArrays {")
    b = text.index("// ---- TMA 1-D bulk copy + mbarrier")
    return "namespace amwg {\n" + text[a:b] + "}  // namespace amwg\n"


def _kernel_text(generated):
    """csrc/amwg_jit_full_kernel.cuh as the host compiles it: the generated header spliced in where it is included, the one PTX fence
    dropped (the shim's mbarriers need none), the dynamic shared memory declaration dropped (the shim's `smem` of the declared size
    stands for it), and the Bernoulli bit masks taken as given (the test builds them; the kernel's builder is a
    warp-wide ballot, and the host runs one thread per CTA)."""
    text = open(os.path.join(CSRC, "amwg_jit_full_kernel.cuh")).read()
    lines = []
    n_asm = n_smem = 0
    for ln in text.splitlines():
        if "asm volatile(" in ln:
            assert "fence.mbarrier_init" in ln, ln
            n_asm += 1
            continue
        if "extern __shared__" in ln:
            assert ln.strip() == "extern __shared__ __align__(16) unsigned char smem[];", ln
            n_smem += 1
            continue
        lines.append(ln)
    assert n_asm == 1 and n_smem == 1
    text = "\n".join(lines)
    inc = '#include "amwg_jit_generated.inc"'
    assert text.count(inc) == 1
    return text.replace(inc, generated + "\n#undef JN_BERN\n#define JN_BERN 0\n").replace("#pragma once", "")


class HostKernel(HostProgram, StrictShim):
    def __init__(self, pkg, orc, tmp_path, params, log_post, data, _opts=None, **opts):
        self._tmp = tmp_path
        super().__init__(pkg, orc, tmp_path, params, log_post, data, _opts=_opts, **opts)
        s = self.s
        m = s._model_keepalive[-1]
        src = self.src
        cut = src.index("namespace amwg {")
        cpp = tmp_path / "kernel.cpp"
        cpp.write_text(src[:cut] + HOST_PRELUDE + KERNEL_SHIM + _tma_structs() + _kernel_text(src[cut:]) + KERNEL_EXPORTS)
        K = _compile(cpp, tmp_path / "kernel.so")
        self._shim_setup(K, src, self.msg)
        K.hs_exp_of.restype, K.hs_exp_of.argtypes = C.c_double, [C.c_double]
        # the masks the kernel's ballot loop would build: copied from the evaluation harness's staging buffer
        for k in range(self.lib.hs_n_bern()):
            n, m0 = self.lib.hs_bern_n(k), self.lib.hs_bern_mask(k)
            nb = 4 * ((n + 31) // 32 + 1)
            K.hs_preset(m0, self.smem[m0:m0 + nb].ctypes.data, nb)
        self.init = np.array([m.init[c] for c in range(self.D)], dtype=np.float64)
        self.n_params = int(m.n_params)

    def start(self, chains, first_chain, seed):
        """what amwg_create leaves on the device: every chain at `init`, log_post evaluated once, identity substepper order, stream at 0"""
        D, Cn = self.D, chains
        self.chains, self.first_chain, self.seed = chains, first_chain, seed
        self.state = np.repeat(self.init[:, None], Cn, axis=1).copy()
        self.psd = np.full((D, Cn), self.K.hs_exp_of(0.0))
        self.acc = np.zeros((D, Cn), dtype=np.int32)
        lp0 = self.lib.hs_logpost(self.init.ctypes.data_as(C.POINTER(C.c_double)), -1, 0.0)
        self.curr = np.full(Cn, lp0)
        self.perm = np.full(Cn, sum(p << (4 * p) for p in range(self.n_params)) if self.n_params <= 16 else 0, dtype=np.uint64)
        self.rng_n = np.zeros(Cn, dtype=np.uint64)
        self.cols, self.colp = self._upload(self.prog.columns)
        self.adapting = np.ones(D, dtype=np.uint8)
        m = self.s._model_keepalive[-1]
        max_dim0 = max([m.params[p].dim0 for p in range(self.n_params) if m.params[p].n_comp > 1] + [1])
        self.perm_ext = np.repeat(np.arange(self.n_params, dtype=np.uint8)[:, None], Cn, axis=1).copy() if self.n_params > 16 else None
        self.order_ext = np.zeros((max_dim0, Cn), dtype=np.uint16) if max_dim0 > 256 else None

    def _ext(self):
        pe = self.perm_ext.ctypes.data_as(C.POINTER(C.c_ubyte)) if self.perm_ext is not None else None
        oe = self.order_ext.ctypes.data_as(C.POINTER(C.c_ushort)) if self.order_ext is not None else None
        return pe, oe

    def sweeps(self, n, record=True, thin=1):
        """burn(n) (record=False) or sample(n): -> out[row][entry][chain], row r = the state before sweep r * thin"""
        n_der = len(self.s._derived_names)
        mon = np.arange(self.D + n_der, dtype=np.int32)
        rows = (n + thin - 1) // thin if record else 0
        out = np.full((max(rows, 1), mon.size, self.chains), np.nan)
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
        self.K.hs_sweep(p(self.state, C.c_double), p(self.psd, C.c_double), p(self.acc, C.c_int), p(self.curr, C.c_double), p(self.perm, C.c_uint64),
                        p(self.rng_n, C.c_uint64), C.c_uint64(self.chains), C.c_uint64(self.first_chain), C.c_uint64(self.seed), C.c_longlong(n),
                        C.c_longlong(0), C.c_longlong(thin), 1 if record else 0, int(mon.size), p(mon, C.c_int), p(out, C.c_double), self.colp,
                        len(self.cols), p(self.adapting, C.c_ubyte), *self._ext())
        self._contract(self.cols)
        return out[:rows]

    def run(self, chains, first_chain, seed, sweeps):
        self.start(chains, first_chain, seed)
        out = self.sweeps(sweeps)
        return out, self.state, self.rng_n, self.acc

    # -- the host side of a sweep call, restated: csrc/amwg_kernels.cu run_sweeps() + amwg_adapt_kernel (mcmc.js:536-551). A launch
    #    never crosses a batch boundary; at a boundary the component's prop_log_scale moves by +-delta and its counter is cleared.
    def start_driver(self, first_chain, seed):
        m = self.s._model_keepalive[-1]
        self.opts = [m.comp_options[c] for c in range(self.D)]
        self.start(1, first_chain, seed)
        self.pls = np.array([[o.prop_log_scale] for o in self.opts], dtype=np.float64)
        self.psd[:, 0] = [self.K.hs_exp_of(float(v)) for v in self.pls[:, 0]]
        self.is_adapting = [bool(o.is_adapting) for o in self.opts]
        self.adapting[:] = [1 if f else 0 for f in self.is_adapting]
        self.iter_since = [0.0] * self.D
        self.batch_count = [0.0] * self.D

    def set_adapting(self, flag):
        self.is_adapting = [bool(flag)] * self.D
        self.adapting[:] = 1 if flag else 0

    def advance(self, n, record, thin=1):
        import math
        n_der = len(self.s._derived_names)
        mon = np.arange(self.D + n_der, dtype=np.int32)
        rows = (n + thin - 1) // thin if (record and n > 0) else 0
        out = np.full((max(rows, 1), mon.size, 1), np.nan)
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
        i0 = 0
        while i0 < n:
            L = n - i0
            for c in range(self.D):
                if not self.is_adapting[c]:
                    continue
                need = math.ceil(self.opts[c].batch_size - self.iter_since[c])
                if not need >= 1.0:
                    need = 1.0
                L = min(L, int(need))
            self.K.hs_sweep(p(self.state, C.c_double), p(self.psd, C.c_double), p(self.acc, C.c_int), p(self.curr, C.c_double), p(self.perm, C.c_uint64),
                            p(self.rng_n, C.c_uint64), C.c_uint64(1), C.c_uint64(self.first_chain), C.c_uint64(self.seed), C.c_longlong(L),
                            C.c_longlong(i0), C.c_longlong(thin), 1 if record else 0, int(mon.size), p(mon, C.c_int), p(out, C.c_double), self.colp,
                            len(self.cols), p(self.adapting, C.c_ubyte), *self._ext())
            self._contract(self.cols)
            for c in range(self.D):
                if not self.is_adapting[c]:
                    continue
                self.iter_since[c] += float(L)
                if self.iter_since[c] >= self.opts[c].batch_size:
                    self.batch_count[c] += 1.0
                    adj = self.opts[c].initial_adaptation / math.sqrt(self.batch_count[c])
                    mx = self.opts[c].max_adaptation
                    delta = math.nan if (adj != adj or mx != mx) else min(mx, adj)
                    rate = float(self.acc[c, 0]) / self.opts[c].batch_size if self.opts[c].batch_size != 0 else (math.nan if self.acc[c, 0] == 0 else math.inf)
                    self.pls[c, 0] = self.pls[c, 0] + delta if rate > self.opts[c].target_accept_rate else self.pls[c, 0] - delta
                    self.psd[c, 0] = self.K.hs_exp_of(float(self.pls[c, 0]))
                    self.acc[c, 0] = 0
                    self.iter_since[c] = 0.0
            i0 += L
        return out[:rows]


@pytest.mark.parametrize("name,c_model,data_c", [
    ("spike_where", "spike_bern", lambda d: {"x": np.asarray(d["x"], float)}),
    ("spike_literal", "spike_bern", lambda d: {"x": np.asarray(d["x"], float)}),
    ("complex_literal", "complex", lambda d: {"x": np.asarray(d, float)}),
    ("multi_bern", "multi_bern_dens", lambda d: None),
    ("beta_bern_faithful", "beta_bern", lambda d: {"x": np.asarray(d["x"], float)}),
    ("norm_test_faithful", "norm_test", lambda d: np.asarray(d, float)),
])
def test_the_specialised_kernel_run_on_the_host_draws_what_the_oracle_draws(pkg, orc, tmp_path, name, c_model, data_c):
    """The skeleton (csrc/amwg_jit_full_kernel.cuh) and the generated code, compiled for the host and run one emulated thread per CTA
    -- shuffles, proposals, bounds, Metropolis and binary steps, sample recording -- against the CPU restatement of mcmc.js on the same
    Philox streams: 45 recorded sweeps (inside the first adaptation batch: the batch update is a separate kernel) of 6 chains at a
    global chain offset, bit for bit, and the same number of Math.random() calls consumed."""
    params, f, data, opts = _cases(pkg)[name]
    hk = HostKernel(pkg, orc, tmp_path, params, f, data, **opts)
    chains, first, seed, sweeps = 6, 1000003, 17, 45
    out, state, rng_n, acc = hk.run(chains, first, seed, sweeps)
    ref = orc.run_model(c_model, data_c(data), params, chains=chains, first_chain=first, seed=seed, burn=0, sample=sweeps)
    e = 0
    for pname in hk.s.params:
        n = int(np.prod(hk.s.params[pname]["dim"]))
        got = np.moveaxis(out[:, e:e + n, :], 1, 2).reshape(np.asarray(ref[pname]).shape)     # [rows, chains, *dim]
        assert np.array_equal(got.view(np.uint64), np.asarray(ref[pname], np.float64).view(np.uint64)), pname
        e += n
    for k, dname in enumerate(hk.s._derived_names):               # derived quantities are recorded with the state they belong to
        assert np.array_equal(out[:, e + k, :].view(np.uint64), np.asarray(ref[dname], np.float64).reshape(sweeps, chains).view(np.uint64)), dname
    assert np.all(rng_n >= sweeps) and np.unique(out[-1], axis=1).shape[1] > 1          # every chain drew, and not the same thing


# ---- the production lowering: the specialised statistics sweep (csrc/amwg_jit_kernel.cuh) on the host -------------------------------
STAT_SHIM = KERNEL_SHIM + r'''
static inline int atomicAdd(int* p, int v) { const int o = *p; *p = o + v; return o; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
namespace amwg {
static inline double2 lds_f64x2(unsigned a) { double2 v{0.0, 0.0}; if (lds_ok(a, 16)) std::memcpy(&v, g_smem_base + a, 16); return v; }
}
'''

STAT_EXPORTS = CONTRACT_EXPORTS + r'''
extern "C" {
double hs_exp_of(double x) { return amwg::js_exp(x); }
int hs_nt() { return JNT; }
void hs_sweep(double* state, double* psd, int* acc, double* work /* [2 JNT + 2 JD][C] */, unsigned short* vseq, unsigned long long* perm,
              unsigned long long* rng_n, unsigned long long C, unsigned long long first_chain, unsigned long long seed, long long n_sweeps,
              int n_monitor, const int* monitor, double* out, const double** cols, int n_cols, const unsigned char* adapting,
              unsigned char* perm_ext, unsigned short* order_ext, long long thin) {
  amwg::JitArgs A{};
  A.a.state = state; A.a.psd = psd; A.a.acc = acc; A.a.perm = perm; A.a.rng_n = rng_n; A.a.vseq = vseq;
  A.a.perm_ext = perm_ext; A.a.order_ext = order_ext;
  A.a.tval = work; A.a.tcand = work + (unsigned long long)JNT * C; A.a.bprop = work + 2ull * JNT * C; A.a.bcoin = work + (2ull * JNT + JD) * C;
  A.a.C = C; A.a.first_chain = first_chain; A.a.seed = seed;
  A.sa.n_sweeps = n_sweeps; A.sa.sample_i0 = 0; A.sa.thin = thin; A.sa.record = 1; A.sa.n_monitor = n_monitor; A.sa.monitor = monitor; A.sa.out = out;
  for (int k = 0; k < n_cols; ++k) A.col[k] = cols[k];
  A.adapting = adapting;
  for (unsigned long long c = 0; c < C && !g_fault[0]; ++c) { hs_cta_begin((unsigned)c); amwg::amwg_jit_sweep(A); }
}
}
'''


def _sum_sq_text():
    text = open(os.path.join(CSRC, "amwg_tma.cuh")).read()
    a = text.index("// ---- plates: the O(N) likelihood sums")
    b = text.index("#undef AMWG_ACC8", a)
    return "namespace amwg {\n" + text[a:b] + "#undef AMWG_ACC8\n}  // namespace amwg\n"


def _stat_kernel_text(generated):
    text = open(os.path.join(CSRC, "amwg_jit_kernel.cuh")).read()
    lines, n_asm, n_smem = [], 0, 0
    for ln in text.splitlines():
        if "asm volatile(" in ln:
            assert "fence.mbarrier_init" in ln, ln
            n_asm += 1
            continue
        if "extern __shared__" in ln:
            assert ln.strip() == "extern __shared__ __align__(16) unsigned char smem[];", ln
            n_smem += 1
            continue
        lines.append(ln)
    assert n_asm == 1 and n_smem == 1
    text = "\n".join(lines)
    inc = '#include "amwg_jit_generated.inc"'
    assert text.count(inc) == 1
    return text.replace(inc, generated).replace("#pragma once", "")


class HostStatKernel(StrictShim):
    """`edit`: applied to the kernel's text before it is compiled (the self-checks of tests/stat_check.py plant a defect with it).
    After run(), `work` holds the working set ([tval | tcand | bprop | bcoin][chain]; work[:NT] is the term cache) and `state` the
    chains' components."""

    def __init__(self, pkg, orc, tmp_path, params, log_post, data, chains_hint=4096, edit=None):
        self.s = s = pkg.mcmc.AmwgSampler(params, log_post, data, {"chains": chains_hint, "_model_only": True})
        self.prog, self.O = s._program, orc.lib()
        assert self.prog.stat_prog >= 0
        self.consts = prog_eval.fold_constants(self.prog, self.O)
        m = s._model_keepalive[-1]
        for i, v in enumerate(self.consts):
            m.consts[i] = float(v)
        rc, msg, src = s.jit_compile_check()
        assert rc == 0, msg
        self.src = src
        cut = src.index("namespace amwg {")
        cpp = tmp_path / "stat_kernel.cpp"
        kernel = _stat_kernel_text(src[cut:])
        if edit is not None:
            edited = edit(kernel)
            assert edited != kernel, "the edit did not change the kernel"
            kernel = edited
        cpp.write_text(src[:cut] + HOST_PRELUDE + STAT_SHIM + _tma_structs() + _sum_sq_text() + kernel + STAT_EXPORTS)
        K = _compile(cpp, tmp_path / "stat_kernel.so")
        self._shim_setup(K, src, msg)
        K.hs_exp_of.restype, K.hs_exp_of.argtypes = C.c_double, [C.c_double]
        self.D, self.NT, self.n_params = int(m.n_comp), K.hs_nt(), int(m.n_params)
        assert self.NT == self.prog.n_terms
        self.init = np.array([m.init[c] for c in range(self.D)], dtype=np.float64)

    def run(self, chains, first_chain, seed, sweeps, thin=1, adapting=None):
        """-> out[row][entry][chain] over the D components and the derived quantities, the stream positions; self.acc: acceptance counts"""
        D, NT, Cn = self.D, self.NT, chains
        cache = [0.0] * NT
        prog_eval.run(self.prog, self.consts, self.init, self.prog.logpost_prog, self.O, cache=cache)     # terms and statistics at init (amwg_init_kernel)
        work = np.zeros((2 * NT + 2 * D, Cn))
        work[:NT, :] = np.asarray(cache)[:, None]
        state = np.repeat(self.init[:, None], Cn, axis=1).copy()
        psd = np.full((D, Cn), self.K.hs_exp_of(0.0))
        acc = np.zeros((D, Cn), dtype=np.int32)
        vseq = np.zeros((D, Cn), dtype=np.uint16)
        perm = np.full(Cn, sum(p << (4 * p) for p in range(self.n_params)) if self.n_params <= 16 else 0, dtype=np.uint64)
        perm_ext = np.repeat(np.arange(self.n_params, dtype=np.uint8)[:, None], Cn, axis=1).copy() if self.n_params > 16 else None
        rng_n = np.zeros(Cn, dtype=np.uint64)
        mon = np.arange(D + len(self.s._derived_names), dtype=np.int32)
        out = np.full(((sweeps + thin - 1) // thin, mon.size, Cn), np.nan)
        cols, colp = self._upload(self.prog.columns)
        adapting = np.ones(D, dtype=np.uint8) if adapting is None else np.asarray(adapting, dtype=np.uint8)
        self.acc, self.work, self.state = acc, work, state
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
        self.K.hs_sweep(p(state, C.c_double), p(psd, C.c_double), p(acc, C.c_int), p(work, C.c_double), p(vseq, C.c_ushort), p(perm, C.c_uint64),
                        p(rng_n, C.c_uint64), C.c_uint64(Cn), C.c_uint64(first_chain), C.c_uint64(seed), C.c_longlong(sweeps), int(mon.size), p(mon, C.c_int),
                        p(out, C.c_double), colp, len(cols), p(adapting, C.c_ubyte),
                        perm_ext.ctypes.data_as(C.POINTER(C.c_ubyte)) if perm_ext is not None else None, None, C.c_longlong(thin))
        self._contract(cols)
        return out, rng_n


def _agreement(out, ref, params):
    """fraction of chains whose every recorded row equals the oracle's, and the first row at which any chain differs"""
    same = None
    e = 0
    for pname, pdef in params.items():
        n = int(np.prod(pdef.get("dim", [1])))
        got = np.moveaxis(out[:, e:e + n, :], 1, 2)                # [rows, chains, n]
        want = np.asarray(ref[pname], np.float64).reshape(got.shape)
        eq = (got.view(np.uint64) == want.view(np.uint64)).all(axis=2)
        same = eq if same is None else (same & eq)
        e += n
    return same.all(axis=0).mean(), same


def test_the_statistics_sweep_on_the_host_headline_model(pkg, orc, tmp_path):
    """BASELINE config 2's model and kernel (resident column, working set in shared memory, two component classes): the production
    lowering decides steps on differences of factorised plates, so it equals the reference up to rounding -- a decision can differ
    only when exp(delta) falls within ~1e-13 of the accept uniform. 64 chains x 45 sweeps on the oracle's streams: (nearly) all equal."""
    x = np.random.default_rng(77).normal(184.5, 4.5, 200)
    hk = HostStatKernel(pkg, orc, tmp_path, models.PARAMS_NORM, models.norm_post_readme(pkg.ld), x.tolist())
    assert "#define JWS_SMEM 1" in hk.src and "#define JSTREAM 0" in hk.src
    out, rng_n = hk.run(64, 5000, 3, 45)
    ref = orc.run_model("norm_readme", x, models.PARAMS_NORM, chains=64, first_chain=5000, seed=3, burn=0, sample=45)
    frac, _ = _agreement(out, ref, models.PARAMS_NORM)
    assert frac >= 0.97, frac
    assert np.isfinite(out).all() and np.unique(out[-1, 0]).size > 50


# unequal groups (all >= 8 points, so each is a plate of its own) on a streamed column: boundaries fall mid-tile (tiles of 1024
# points), the 2500-point group spans more than two tiles, the 9-point group lies inside one, and the total (9563) is odd
RAGGED = (9, 2500, 37, 1111, 3001, 14, 777, 1500, 614)


@pytest.mark.parametrize("J,per,stream", [(8, 32, False), (6, 1500, True), (8, 1100, True), (len(RAGGED), RAGGED, True)])
def test_the_statistics_sweep_on_the_host_hierarchical_model(pkg, orc, tmp_path, J, per, stream):
    """BASELINE config 4's shape: a vector of group means (one class, indices from tables, stepped as an index-ordered block between
    the steps the chain visits before and after it) and a shared sd whose plate terms are a loop; with 9000 points the column streams
    through the tile ring (memcpy here). `per` may list unequal group sizes: then a streamed tile is split between plates wherever
    a group ends inside it."""
    sizes = np.broadcast_to(per, (J,))
    rng = np.random.default_rng(4)
    g = np.repeat(np.arange(J), sizes)
    y = rng.normal(100, 5, g.size) + np.repeat(rng.normal(0, 3, J), sizes)
    P = {"mu": {"type": "real", "dim": [J], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    data = {"y": y, "g": g.astype(float)}
    hk = HostStatKernel(pkg, orc, tmp_path, P, models.hier_norm_post(pkg.ld), data)
    assert ("#define JSTREAM 1" in hk.src) == stream
    assert ("#define JBLOCK 0" in hk.src) == (J >= 8)             # the block of group means is stepped in index order from 8 members on
    chains, sweeps = (32, 45) if not stream else (8, 20)
    out, rng_n = hk.run(chains, 77, 9, sweeps)
    ref = orc.run_model("hier_norm", {"y": y, "g": g.astype(float)}, P, chains=chains, first_chain=77, seed=9, burn=0, sample=sweeps)
    frac, _ = _agreement(out, ref, P)
    assert frac >= 0.97, frac                                     # measured: 1.0 on all three shapes
    assert np.isfinite(out).all()


@pytest.mark.parametrize("scenario", ["binary_stepper", "binary_component_stepper"])
def test_the_specialised_kernel_on_the_host_against_the_reference_js_vectors(pkg, orc, tmp_path, scenario):
    """tests/golden/reference_js.json holds what the UNMODIFIED mcmc.js drew (oracle/minijs). Its two all-binary scenarios need no
    adaptation kernel (BinaryStepper does not adapt, mcmc.js:740-767), so the emulated specialised kernel can follow their whole scripts
    -- burn, sample, thinning -- and must reproduce the reference's draws and final state bit for bit, for both recorded chains."""
    import copy
    import golden_util as gu
    cases = [c for c in gu.load()["samplers"] if c["name"] == scenario]
    assert len(cases) == 2
    for case in cases:
        _c, py_model, params, data, _dc = gu.resolve_case(case, pkg)
        opts = copy.deepcopy(case["options"]) or {}
        thin = int(opts.pop("thin", 1))
        assert not opts
        sub = tmp_path / f"chain{case['chain']}"
        sub.mkdir()
        hk = HostKernel(pkg, orc, sub, copy.deepcopy(params), py_model, data)
        hk.start(1, case["chain"], case["seed"])
        results = iter(case["results"])
        for step in case["script"]:
            if step[0] == "burn":
                hk.sweeps(step[1], record=False)
            elif step[0] == "thin":
                thin = int(step[1])
            elif step[0] == "sample":
                want = gu.unhex(next(results)["draws"])
                out = hk.sweeps(step[1], thin=thin)
                e = 0
                for pname in hk.s.params:
                    n = int(np.prod(hk.s.params[pname]["dim"]))
                    got = out[:, e:e + n, 0]
                    assert gu.same(got.reshape(np.asarray(want[pname], dtype=np.float64).shape), want[pname]), (scenario, pname)
                    e += n
            else:
                raise AssertionError(step)
        e = 0
        for pname, want in gu.unhex(case["final_state"]).items():
            n = int(np.prod(hk.s.params[pname]["dim"]))
            assert gu.same(hk.state[e:e + n, 0], np.asarray(want, dtype=np.float64).reshape(-1)), pname
            e += n


def _golden_cases():
    import golden_util as gu
    return [pytest.param(c, id=f"{c['name']}-chain{c['chain']}") for c in gu.load()["samplers"]]


@pytest.mark.parametrize("case", _golden_cases())
def test_the_specialised_kernel_on_the_host_follows_the_golden_scripts(pkg, orc, tmp_path, case):
    """Every sampler scenario of tests/golden/reference_js.json (what the unmodified mcmc.js drew) -- the six whose models step with a
    term cache by default are lowered as with AMWG_TERM_CACHE=0: the emulated full-program
    kernel under the restated host driver (launches that end on batch boundaries, the Roberts-Rosenthal update between them,
    start/stop_adaptation, thinning, monitors) reproduces the reference's draws, final state and stepper info bit for bit."""
    import copy
    import golden_util as gu
    _c, py_model, params, data, _dc = gu.resolve_case(case, pkg)
    opts = copy.deepcopy(case["options"]) or {}
    opts["faithful"] = True
    try:
        hk = HostKernel(pkg, orc, tmp_path, copy.deepcopy(params), py_model, data, _opts=opts)
    except AssertionError as e:
        if "term cache" not in str(e):
            raise
        # by default this model steps with a term cache on the interpreter kernels; lowered as with AMWG_TERM_CACHE=0 (every step
        # runs the full program -- the same bits, term by term) the specialisation takes it
        sub = tmp_path / "full"
        sub.mkdir()
        hk = HostKernel(pkg, orc, sub, copy.deepcopy(params), py_model, data, _opts=dict(opts, _force_full=True))
    hk.start_driver(case["chain"], case["seed"])
    thin = int(opts.get("thin", 1))
    names = list(hk.s.params) + list(hk.s._derived_names)
    width = {k: int(np.prod(hk.s.params[k]["dim"])) for k in hk.s.params}
    width.update({k: 1 for k in hk.s._derived_names})
    monitor = opts.get("monitor", None)
    results = iter(case["results"])
    for step in case["script"]:
        op = step[0]
        if op == "burn": hk.advance(step[1], record=False)
        elif op == "thin": thin = int(step[1])
        elif op == "monitor": monitor = step[1]
        elif op == "stop_adaptation": hk.set_adapting(False)
        elif op == "start_adaptation": hk.set_adapting(True)
        elif op == "sample":
            want = gu.unhex(next(results)["draws"])
            out = hk.advance(step[1], record=True, thin=abs(thin))
            keys = names if monitor is None else [k for k in monitor]
            assert list(want.keys()) == keys
            e = 0
            for k in names:
                if k in want:
                    got = out[:, e:e + width[k], 0]
                    assert gu.same(got.reshape(np.asarray(want[k], dtype=np.float64).shape), want[k]), (case["name"], k)
                e += width[k]
    e = 0
    for k in hk.s.params:
        want = gu.flat_info(case["final_info"].get(k, {}))
        if want:
            sl = slice(e, e + width[k])
            assert gu.same(hk.pls[sl, 0], [w["prop_log_scale"] for w in want]), k
            assert gu.same(hk.acc[sl, 0].astype(float), [w["acceptance_count"] for w in want]), k
            assert gu.same(hk.iter_since[sl], [w["iterations_since_adaption"] for w in want]), k
            assert gu.same(hk.batch_count[sl], [w["batch_count"] for w in want]), k
        e += width[k]
    e = 0
    st = gu.unhex(case["final_state"])
    for k in hk.s.params:
        assert gu.same(hk.state[e:e + width[k], 0], np.asarray(st[k], dtype=np.float64).reshape(-1)), k
        e += width[k]


# ---- the strict shim itself: each rule of the bulk copy and the mbarrier refuses a bad call, with a message that says why -------------
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("shim")
    cpp = d / "shim.cpp"
    cpp.write_text(HOST_PRELUDE + KERNEL_SHIM + CONTRACT_EXPORTS)
    K = _compile(cpp, d / "shim.so")
    K.hs_register_alloc.argtypes = [C.c_void_p, C.c_ulonglong]
    K.hs_kernel_smem.restype = C.POINTER(C.c_ubyte)
    K.hs_tma_bulk_g2s.argtypes = [C.c_ulonglong, C.c_void_p, C.c_uint, C.c_void_p]
    K.hs_mbar_init.argtypes = K.hs_mbar_expect_tx.argtypes = K.hs_mbar_wait.argtypes = [C.c_void_p, C.c_uint]
    return K


def _stage(K, col, dst_off, bytes_, expect=None, parity=0, smem=1024, register=None):
    """one staging as the kernels do it: init, expect_tx, one bulk copy of `bytes_` from `col`, wait -> the shim's first fault"""
    K.hs_clear_fault()
    K.hs_set_dyn_smem(smem)
    K.hs_clear_allocs()
    base, n = register if register is not None else (col.ctypes.data, col.nbytes)
    K.hs_register_alloc(base, n)
    bar = np.zeros(1, dtype=np.uint64)
    K.hs_mbar_init(bar.ctypes.data, 1)
    K.hs_mbar_expect_tx(bar.ctypes.data, bytes_ if expect is None else expect)
    K.hs_tma_bulk_g2s(dst_off, col.ctypes.data, bytes_, bar.ctypes.data)
    K.hs_mbar_wait(bar.ctypes.data, parity)
    return K.hs_fault_msg().decode()


def test_the_strict_shim_accepts_a_staging_that_follows_the_rules(shim):
    (col,) = device_columns([np.arange(71.0)])                   # 568 bytes of data, 576 on the device
    assert col.nbytes == 576 and col.ctypes.data % 16 == 0 and col[71] == 0.0
    assert _stage(shim, col, 64, 576) == ""
    got = np.ctypeslib.as_array(shim.hs_kernel_smem(), shape=(1024,))[64:64 + 576].copy().view(np.float64)
    assert np.array_equal(got, col)


def test_the_strict_shim_refuses_a_misaligned_source(shim):
    (col,) = device_columns([np.arange(72.0)])
    raw = np.ctypeslib.as_array((C.c_double * 72).from_address(col.ctypes.data + 8), shape=(71,))
    msg = _stage(shim, raw, 0, 560, register=(col.ctypes.data, col.nbytes))
    assert "16-byte aligned" in msg, msg


def test_the_strict_shim_refuses_the_unpadded_column_copies(shim):
    col = np.arange(71.0)                                         # a 568-byte column as numpy holds it
    msg = _stage(shim, col, 0, 568, register=(col.ctypes.data, 568))
    assert "positive multiple of 16" in msg, msg
    msg = _stage(shim, col, 0, 576, register=(col.ctypes.data, 568))           # the padded size from an unpadded allocation
    assert "runs past its end" in msg, msg


def test_the_strict_shim_refuses_a_copy_past_the_declared_shared_memory(shim):
    (col,) = device_columns([np.arange(71.0)])
    msg = _stage(shim, col, 512, 576, smem=1024)
    assert "outside the 1024 bytes of dynamic shared memory" in msg, msg


def test_the_strict_shim_reports_an_expect_tx_that_differs_as_a_hang(shim):
    (col,) = device_columns([np.arange(71.0)])
    for expect in (576 + 16, 576 - 16):
        msg = _stage(shim, col, 0, 576, expect=expect)
        assert "would hang on the device" in msg and f"{expect} transaction bytes expected, 576 delivered" in msg, msg


def test_the_strict_shim_refuses_a_wait_on_the_wrong_phase(shim):
    (col,) = device_columns([np.arange(71.0)])
    msg = _stage(shim, col, 0, 576, parity=1)
    assert "parity 1 while the mbarrier is in phase 0" in msg, msg
