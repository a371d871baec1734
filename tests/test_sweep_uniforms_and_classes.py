"""The Philox uniforms formed without integer-to-double conversions, and a statistics sweep whose component classes differ in shape.

csrc/amwg_math.cuh u53 forms (double)v of a 32-bit word as (2^52 + v) - 2^52 from its bit pattern; it is held here against the
conversion form bit for bit. The second part runs a model of three component classes -- one of them with two members, so its code
reads its indices from tables -- that take different numbers of logarithms and divisions through the emulated specialised
statistics sweep (and, with -m gpu, the device) against the oracle, draw for draw."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import prog_eval

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bayes.js_b200", "csrc")

U53_HOST = r'''
#include "amwg_math.cuh"
extern "C" {
void hs_u53(const uint32_t* a, const uint32_t* b, long long n, double* fast, double* conv) {
  for (long long i = 0; i < n; ++i) {
    fast[i] = amwg::u53(a[i], b[i]);
    conv[i] = ((double)(a[i] >> 5) * 67108864.0 + (double)(b[i] >> 6)) * (1.0 / 9007199254740992.0);
  }
}
void hs_u32(const uint32_t* v, long long n, double* out) { for (long long i = 0; i < n; ++i) out[i] = amwg::u32_to_double(v[i]); }
}
'''


def test_uniforms_without_conversions_equal_the_conversion_form(tmp_path):
    cpp, so = tmp_path / "u53.cpp", tmp_path / "u53.so"
    cpp.write_text(U53_HOST)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
                        "-I" + CSRC, str(cpp), "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(so))
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    special = np.array([0, 0xffffffff] + [1 << k for k in range(32)] + [(1 << k) - 1 for k in range(1, 32)], dtype=np.uint32)
    out = np.empty(special.size)
    lib.hs_u32(p(special, C.c_uint32), C.c_longlong(special.size), p(out, C.c_double))
    assert np.array_equal(out, special.astype(np.float64)) and not np.signbit(out).any()
    rng = np.random.default_rng(53)
    a = np.concatenate([np.repeat(special, special.size), rng.integers(0, 1 << 32, 10 ** 6, dtype=np.uint32)]).astype(np.uint32)
    b = np.concatenate([np.tile(special, special.size), rng.integers(0, 1 << 32, 10 ** 6, dtype=np.uint32)]).astype(np.uint32)
    fast, conv = np.empty(a.size), np.empty(a.size)
    lib.hs_u53(p(a, C.c_uint32), p(b, C.c_uint32), C.c_longlong(a.size), p(fast, C.c_double), p(conv, C.c_double))
    assert np.array_equal(fast.view(np.uint64), conv.view(np.uint64))
    want = ((a >> 5).astype(np.float64) * 67108864.0 + (b >> 6).astype(np.float64)) * 2.0 ** -53
    assert np.array_equal(conv.view(np.uint64), want.view(np.uint64))
    assert fast.min() == 0.0 and fast.max() < 1.0


def _jit_step(src):
    a = src.index("bool jit_step(")
    return src[a:src.index("\n}\n", a)]


# ---- three classes with different numbers of logarithms and divisions ------------------------------------------------------------
# mu: its prior and two plate terms (2 logarithms, 3 divisions); {s1, s2}: one class of two members, a bound prior and one plate term
# each (1, 1); p: a bounded scalar with a Normal prior (0, 1).
P3 = {"mu": {"type": "real", "init": 5.0}, "s1": {"type": "real", "lower": 0, "init": 2.0}, "s2": {"type": "real", "lower": 0, "init": 1.0},
      "p": {"type": "real", "lower": 0, "upper": 1, "init": 0.5}}


def three_class_model(ld):
    rng = np.random.default_rng(33)
    data = {"y1": rng.normal(5.0, 2.0, 150).tolist(), "y2": rng.normal(5.5, 1.0, 90).tolist()}

    def log_post(state, d):
        lp = 0
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.s1, 0, 100)
        lp += ld.unif(state.s2, 0, 100)
        lp += ld.norm(state.p, 0.5, 0.3)
        for i in range(len(d.y1)):
            lp += ld.norm(d.y1[i], state.mu, state.s1)
        for i in range(len(d.y2)):
            lp += ld.norm(d.y2[i], state.mu, state.s2)
        return lp
    return log_post, data


def _check_classes(src):
    """three cases, one of them indexed by member, and one Metropolis test after the switch for all of them"""
    step = _jit_step(src)
    assert "  case 2: {" in step and "case 3:" not in step and "const int m = JMEM[c];" in step
    assert step.count("js_exp(") == 1


def _oracle(pkg, orc, log_post, data):
    """the reference's log_post: the bit-faithful lowering's bytecode with the oracle's arithmetic"""
    s = pkg.mcmc.AmwgSampler(P3, log_post, data, {"chains": 4096, "_model_only": True, "faithful": True})
    O = orc.lib()
    prog = s._program
    consts = prog_eval.fold_constants(prog, O)
    return lambda st: prog_eval.logpost(prog, consts, st, O)


def test_three_classes_on_the_host_equal_the_oracle(pkg, orc, tmp_path):
    from test_jit_codegen_semantics import HostStatKernel
    log_post, data = three_class_model(pkg.ld)
    hk = HostStatKernel(pkg, orc, tmp_path, P3, log_post, data)
    _check_classes(hk.src)
    chains, first, seed, sweeps = 12, 3000, 17, 30
    out, rng_n = hk.run(chains, first, seed, sweeps)
    ref_lp = _oracle(pkg, orc, log_post, data)
    for c in range(chains):
        o = orc.OracleSampler(ref_lp, None, P3, seed=seed, chain=first + c)
        ref = o.sample(sweeps)
        want = np.stack([np.asarray(ref[n], np.float64) for n in P3], axis=1)
        assert np.array_equal(out[:, :len(P3), c].view(np.uint64), want.view(np.uint64)), c
        assert int(rng_n[c]) == o.rng_position()
    assert all(np.unique(out[-1, e]).size > 6 for e in range(len(P3)))


@pytest.mark.gpu
def test_three_classes_on_the_gpu_equal_the_oracle(gpu_pkg, orc, monkeypatch):
    """The device kernel at 1061 chains (a ragged last CTA), forced onto the specialised sweep below its chain threshold: 40 chains,
    the first and the last among them, against the oracle draw for draw; a chain that differs must be a rounding tie
    (tests/stat_check.py audit_divergence)."""
    import plate_ref as pr
    import stat_check as sc
    pr.require_extended()
    pkg = gpu_pkg
    log_post, data = three_class_model(pkg.ld)
    C_, first, seed, burn, sample = 1061, 2 ** 32 + 9, 29, 20, 20
    monkeypatch.setenv("AMWG_JIT", "1")
    s = pkg.mcmc.AmwgSampler(P3, log_post, data, {"chains": C_, "seed": seed, "first_chain": first})
    monkeypatch.delenv("AMWG_JIT")
    assert s.jit_status()[0], s.jit_status()
    rc, msg, src = s.jit_compile_check(C_)
    assert rc == 0, msg
    _check_classes(src)
    s.burn(burn)
    d = s.sample(sample)
    got = np.stack([np.asarray(d[n], np.float64) for n in P3], axis=2)         # [rows, chains, D]
    consts = prog_eval.fold_constants(s._program, orc.lib())
    ref_lp = _oracle(pkg, orc, log_post, data)
    y1, y2 = np.asarray(data["y1"]), np.asarray(data["y2"])
    pts = np.concatenate([y1, y2])

    def err(st):
        sd = np.concatenate([np.full(y1.size, st[1]), np.full(y2.size, st[2])])
        priors = [pr.norm_term([st[0]], 0.0, 100.0), pr.unif_term([st[1]], 0, 100), pr.unif_term([st[2]], 0, 100), pr.norm_term([st[3]], 0.5, 0.3)]
        return pr.oracle_norm_error(pts, st[0], sd, priors)
    D = len(P3)
    picks = sorted(set([0, 1, C_ - 1] + np.random.default_rng(5).choice(C_, 37, replace=False).tolist()))
    audited = 0
    for c in picks:
        o = orc.OracleSampler(ref_lp, None, P3, seed=seed, chain=first + c)
        o.trace((burn + sample) * D)
        o.burn(burn)
        ref = o.sample(sample)
        want = np.stack([np.asarray(ref[n], np.float64) for n in P3], axis=1)
        g = got[:, c]
        if np.array_equal(g.view(np.uint64), want.view(np.uint64)):
            continue
        r = int(np.flatnonzero((g.view(np.uint64) != want.view(np.uint64)).any(axis=1))[0])
        assert r > 0, f"chain {c} differs already in its first recorded row"
        tr = o.trace_rows()
        sweep = burn + r - 1
        sc.audit_divergence(s._program, consts, tr[sweep * D:(sweep + 1) * D], g[r - 1], g[r], want[r], pr.JRING_TILE, err)
        audited += 1
    print(f"{len(picks)} chains compared, {audited} audited as rounding ties")
