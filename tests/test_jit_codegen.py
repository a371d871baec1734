"""Run-time specialisation (csrc/amwg_jit.cuh), CPU side: the generated CUDA source of eligible models compiles for sm_90a
with NVRTC (no GPU needed), ineligible models say why, and malformed programs are refused by amwg_create's validation."""
import ctypes as C

import numpy as np
import pytest

import models


def _model_only(pkg, params, log_post, data, chains=1 << 16, **opts):
    o = {"chains": chains, "_model_only": True}
    o.update(opts)
    return pkg.mcmc.AmwgSampler(params, log_post, data, o)


def test_headline_model_specialises_and_compiles(pkg):
    from conftest import config2_data
    s = _model_only(pkg, models.PARAMS_NORM, models.norm_post_readme(pkg.ld), config2_data().tolist(), chains=1 << 20)
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "ok: cubin" in msg and "0 bytes spill stores" in msg
    # two component classes (mu: prior + plate at the candidate statistic; sigma: prior + plate at the committed one), no interpreter
    assert "switch (JCLS[c])" in src and "case 1:" in src and "js_exp(dl) > coin" in src
    assert "#define JWS_SMEM 1" in src and "#define JN_RSTAT 1" in src and "#define JSTREAM 0" in src


def test_hierarchical_model_classes_loops_and_streaming(pkg):
    J, per = 64, 1024
    g = np.repeat(np.arange(J), per)
    y = np.random.default_rng(0).normal(100, 5, J * per)
    P = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    s = _model_only(pkg, P, models.hier_norm_post(pkg.ld), {"y": y, "g": g.astype(float)})
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "0 bytes spill stores" in msg
    # the 64 group means are ONE class (indices from tables), sigma's 64 plate terms are a loop, y (512 KB) streams through the ring
    assert "const int m = JMEM[c];" in src and "for (int j = 0; j < 63; ++j)" in src
    assert "#define JSTREAM 1" in src and "#define JN_SSTAT 64" in src and "#define JS_TOTAL 65536" in src
    # 2^16 chains: 512 CTAs of 128 threads, four per SM (the default CTA size; no other size balances the SMs markedly better)
    assert "#define JTHREADS 128" in src and "#define JMINB 4" in src


def test_expression_means_and_derived_quantities(pkg):
    ld = pkg.ld

    def lp(state, d):
        out = 0
        out += ld.norm(state.a, 0, 10)
        out += ld.gamma(state.s, 2, 0.5)
        for i in range(len(d)):
            out += ld.norm(d[i], state.a * 2 + 1, state.s)
        state.prec = 1 / (state.s * state.s)
        return out
    P = {"a": {"type": "real"}, "s": {"type": "real", "lower": 0}}
    s = _model_only(pkg, P, lp, list(np.random.default_rng(1).normal(3, 1, 200)))
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "jit_derived" in src and "ld_gamma(" in src and "sum_sq_dev(" in src.split("jit_stat_extra")[1]


def test_full_program_models_specialise_too(pkg):
    """models that evaluate all of log_post at every step (binary parameters, `faithful` lowerings): the program itself, per
    configuration of the binary components, printed as straight-line code (amwg_jit_full_kernel.cuh)"""
    y = (np.random.default_rng(2).random(64) < 0.5).astype(float)
    s = _model_only(pkg, models.PARAMS_SPIKE, models.spike_bern(pkg.ld, pkg.mcmc), {"x": y.tolist()})
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "0 bytes spill stores" in msg and "#define JFULL 1" in src
    assert "jit_plate_bern_mask<64>(" in src and "#define JN_BERN 1" in src and "jit_prog_0" in src and "jit_prog_1" not in src
    # the reference's literal `if (m === 0)`: one program per configuration of m, chosen by the value the evaluation sees
    s = _model_only(pkg, models.PARAMS_SPIKE, models.spike_bern_literal(pkg.ld), {"x": y.tolist()})
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "jit_prog_1" in src and "switch (0 | ((CM(1) != 0.0) ? 1 : 0))" in src
    # int + binary + real parameters, negative-binomial likelihood in a loop (tests/test_data.js:154-171)
    x = [int(v) for v in np.random.default_rng(3).integers(5, 30, 12)]
    s = _model_only(pkg, models.PARAMS_COMPLEX, models.complex_model_post_literal(pkg.ld), x)
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "ld_nbinom(" in src and "js_round" not in src.split("jit_logpost")[0]      # rounding of int proposals is the skeleton's
    # the bit-faithful lowering of the headline model: the N-point sum as a loop over the resident column, in data order
    from conftest import config2_data
    s = _model_only(pkg, models.PARAMS_NORM, models.norm_post_readme(pkg.ld), config2_data().tolist(), faithful=True)
    rc, msg, src = s.jit_compile_check()
    assert rc == 0, msg
    assert "for (int i_" in src or "LD(" in src


def test_models_with_a_term_cache_keep_the_interpreter(pkg):
    s = _model_only(pkg, models.PARAMS_HIER_BINOM, models.hierarchical_binomial_post(pkg.ld, pkg.mcmc), models.BINOM_DATA)
    rc, msg, _ = s.jit_compile_check()
    assert rc == 1 and "term cache" in msg


def test_deeply_nested_expressions_are_refused_not_corrupted(pkg):
    """ADVICE r1: the interpreter's operand stack is fixed; a program that needs more must be rejected by validation."""
    ld, mcmc = pkg.ld, pkg.mcmc

    def deep(state, d):
        e = state.x
        for k in range(40):
            e = 1.0 / (1.0 + (0.5 + (0.25 * (2.0 - e))))          # right-nested: every level keeps operands waiting
        t = state.x
        for k in range(60):
            t = (k + 1.0) - (t * 0.5)
        acc = 1.0
        for k in range(45):
            acc = state.x + (state.x * (state.x - acc))
        return ld.norm(state.x, 0, 1) + e + acc
    s = _model_only(pkg, {"x": {"type": "real"}}, deep, None)
    log = C.create_string_buffer(4096)
    rc = pkg._ffi.lib().amwg_jit_compile_check(C.byref(s._model_keepalive[-1]), 1, log, len(log), None, 0)
    # either the lowering keeps it shallow (fine) or validation names the limit; never silently accepted beyond the stack
    if rc == -1:
        assert "operand stack" in log.value.decode()


def test_parameter_array_indexed_out_of_bounds_is_refused(pkg):
    """ADVICE r1: mu[data.g[i]] with 1-based group ids reads past the parameter; JS yields undefined -> NaN, here it must not
    silently alias the next parameter."""
    ld = pkg.ld
    J = 3
    g = np.repeat(np.arange(1, J + 1), 20).astype(float)           # 1..3: out of bounds for a length-3 array
    y = np.random.default_rng(3).normal(0, 1, g.size)

    def hier(state, d):
        lp = ld.unif(state.sigma, 0, 10)
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 10)
        for i in pkg.mcmc.points(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        return lp
    P = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    with pytest.raises(pkg.JsThrow, match="outside its bounds"):
        _model_only(pkg, P, hier, {"y": y, "g": g})
    _model_only(pkg, P, hier, {"y": y, "g": g - 1})                 # 0-based ids are fine


def test_every_golden_model_is_specialised_or_says_why(pkg):
    """Code generation over the reference's own fixtures (the 32 sampler scenarios of tests/golden/reference_js.json, `faithful`
    lowering as the golden tests run them): each model either compiles for sm_90a or is turned down for a stated reason -- the
    generator never fails on a valid program. (With AMWG_JIT=1 the GPU golden tests run these kernels against the vectors.)"""
    import copy
    import golden_util as gu
    seen, compiled, declined = set(), 0, {}
    for case in gu.load()["samplers"]:
        key = (case["log_post"], str(case["params"]), str(case["options"]))
        if key in seen:
            continue
        seen.add(key)
        _c, py_model, params, data, _dc = gu.resolve_case(case, pkg)
        opts = copy.deepcopy(case["options"]) or {}
        opts.update({"chains": 4096, "faithful": True, "_model_only": True})
        s = pkg.mcmc.AmwgSampler(copy.deepcopy(params), py_model, data, opts)
        rc, msg, src = s.jit_compile_check()
        assert rc in (0, 1), (case["name"], msg)
        if rc == 0:
            compiled += 1
            assert "jit_logpost" in src and "ok: cubin" in msg, case["name"]
        else:
            declined[msg.splitlines()[0]] = declined.get(msg.splitlines()[0], 0) + 1
    assert compiled >= 5, (compiled, declined)
    assert set(declined) <= {"the model steps with a term cache"}, declined
