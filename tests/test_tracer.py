"""Host logic (no GPU): the log_post tracer/lowering against the oracle's C models, evaluated with tests/prog_eval.py."""
import numpy as np
import pytest

import models
import prog_eval
from conftest import NORM_DATA, PRESIDENTS, config2_data, config3_data


def _trace(pkg, log_post, params, data):
    mcmc = pkg.mcmc
    cp = mcmc.complete_params(params)
    offsets, n = {}, 0
    for name, p in cp.items():
        offsets[name] = n
        n += int(np.prod(p["dim"]))
    prog, derived = pkg.tracer.trace(log_post, cp, offsets, n, data)
    return prog, derived, n


def _oracle_logpost(orc, model, data, params, state):
    s = orc.OracleSampler(model, data, params)
    import ctypes
    L = orc.lib()
    st = np.array(list(state) + [0.0] * 4, dtype=np.float64)
    fn = getattr(L, "orc_model_" + model)
    fn.restype = ctypes.c_double
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    dptr = ctypes.cast(ctypes.pointer(s._keep[-1]), ctypes.c_void_p) if s._keep[-1] is not None else None
    return fn(st.ctypes.data, dptr, None), st


def test_normal_model_becomes_two_terms_and_a_plate(pkg, orc):
    prog, derived, n = _trace(pkg, models.norm_post_test(pkg.ld), models.PARAMS1, config2_data().tolist())
    assert prog.summary[:3] == ["term LD_NORM", "term LD_UNIF", "plate NORM_IID n=1024"]
    assert prog.summary[3].startswith("pre-evaluated statistics: 1 plate(s), 1024 points") and prog.stat_prog >= 0
    assert derived == ["var"] and n == 2
    assert len(prog.fold_prog) >= 3                    # log(2pi)-log(100), 2*100*100, log(1/(100-0)) are computed once
    consts = prog_eval.fold_constants(prog, orc.lib())
    rng = np.random.default_rng(0)
    for _ in range(20):
        st = [rng.normal(184, 3), rng.uniform(0.5, 20)]
        ref, full = _oracle_logpost(orc, "norm_test", config2_data(), models.PARAMS1, st)
        got = prog_eval.logpost(prog, consts, st, orc.lib())
        assert abs(got - ref) <= 1e-12 * abs(ref)     # factorised plate: equal up to rounding
        der = [None]
        prog_eval.run(prog, consts, st, prog.derived_prog, orc.lib(), der=der)
        assert der[0] == full[2] == st[1] * st[1]
    # outside the support of the uniform prior: -Infinity, like ld.unif (distributions.js:221-223)
    assert prog_eval.logpost(prog, consts, [184.0, 150.0], orc.lib()) == -np.inf


def test_bernoulli_models_are_bit_faithful(pkg, orc):
    y = config3_data()
    prog, _, _ = _trace(pkg, models.spike_bern(pkg.ld, pkg.mcmc), models.PARAMS_SPIKE, {"x": y.tolist()})
    assert prog.summary[-1] == "plate BERN_IID n=256"
    consts = prog_eval.fold_constants(prog, orc.lib())
    rng = np.random.default_rng(1)
    for _ in range(20):
        st = [rng.uniform(-0.1, 1.1), float(rng.integers(0, 2))]
        ref, _ = _oracle_logpost(orc, "spike_bern", {"x": y}, models.PARAMS_SPIKE, st)
        got = prog_eval.logpost(prog, consts, st, orc.lib())
        assert got == ref or (np.isnan(got) and np.isnan(ref)), (st, got, ref)
        # evaluating "state with component c replaced" == evaluating the replaced state
        assert prog_eval.logpost(prog, consts, [0.3, st[1]], orc.lib(), moved=0, val=st[0]) == got or np.isnan(got)


def test_short_loops_stay_unrolled_and_generic_bodies_loop(pkg, orc):
    ld = pkg.ld

    def short(state, data):                         # 5 points: below the plate threshold
        lp = 0
        for i in range(len(data)):
            lp += ld.norm(data[i], state.mu, state.sigma)
        return lp
    prog, _, _ = _trace(pkg, short, models.PARAMS_NORM, PRESIDENTS[:5])
    assert prog.summary == ["term LD_NORM"] * 5

    def cauchy_lik(state, data):                    # no specialised kernel for cauchy: bytecode loop
        lp = ld.norm(state.mu, 0, 100) + ld.unif(state.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.cauchy(data[i], state.mu, state.sigma)
        return lp
    prog, _, _ = _trace(pkg, cauchy_lik, models.PARAMS_NORM, NORM_DATA)
    assert prog.summary[-1] == "plate GENERIC n=10 body=LD_CAUCHY"
    consts = prog_eval.fold_constants(prog, orc.lib())
    O = orc.lib()
    st = [100.0, 30.0]
    ref = O.orc_ld_norm(st[0], 0, 100) + O.orc_ld_unif(st[1], 0, 100)
    for v in NORM_DATA:
        ref = ref + O.orc_ld_cauchy(v, st[0], st[1])
    assert prog_eval.logpost(prog, consts, st, O) == ref


def test_symbolic_index_gives_the_same_program_as_the_concrete_loop(pkg):
    ld, mcmc = pkg.ld, pkg.mcmc
    data = config2_data().tolist()

    def sym(state, d):
        lp = ld.norm(state.mu, 0, 100) + ld.unif(state.sigma, 0, 100)
        for i in mcmc.points(len(d)):
            lp += ld.norm(d[i], state.mu, state.sigma)
        return lp

    def conc(state, d):
        lp = ld.norm(state.mu, 0, 100) + ld.unif(state.sigma, 0, 100)
        for i in range(len(d)):
            lp += ld.norm(d[i], state.mu, state.sigma)
        return lp
    a, _, _ = _trace(pkg, sym, models.PARAMS_NORM, data)
    b, _, _ = _trace(pkg, conc, models.PARAMS_NORM, data)
    assert a.code == b.code and a.plates == b.plates and a.summary == b.summary


def test_hierarchical_and_regression_plates(pkg, orc):
    ld, mcmc = pkg.ld, pkg.mcmc
    rng = np.random.default_rng(2)
    J, per = 4, 8                                  # 32 plate points: below tracer.MIN_STAT_POINTS, so the plates stay single terms
    g = np.repeat(np.arange(J), per)
    y = rng.normal(100, 20, J)[g] + rng.normal(0, 5, J * per)

    def hier(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        return lp
    params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    prog, _, n = _trace(pkg, hier, params, {"y": y.tolist(), "g": g.tolist()})
    assert n == J + 1
    plates = [x for x in prog.summary if x.startswith("plate")]
    assert plates == [f"plate NORM_IID n={per}"] * J                    # one plate per group: mu_j only touches its own
    consts = prog_eval.fold_constants(prog, orc.lib())
    st = list(rng.normal(100, 20, J)) + [4.0]
    ref, _ = _oracle_logpost(orc, "hier_norm", {"y": y, "g": g}, params, st)
    assert abs(prog_eval.logpost(prog, consts, st, orc.lib()) - ref) <= 1e-12 * abs(ref)
    # dependency-aware evaluation: a step on mu_j recomputes its prior and its group's plate only; the other terms come from the
    # chain's term cache, in their original positions -> the same sum, bit for bit, as the full program
    assert prog.n_terms == 2 * J + 1 and len(prog.comp_prog) == J + 1
    assert [prog.touch_off[c + 1] - prog.touch_off[c] for c in range(J + 1)] == [2] * J + [J + 1]
    O = orc.lib()
    cache = [None] * prog.n_terms
    full0 = prog_eval.run(prog, consts, st, prog.logpost_prog, O, cache=cache)            # initial full evaluation fills the cache
    assert None not in cache and full0 == prog_eval.logpost(prog, consts, st, O)
    for step in range(60):
        c = int(rng.integers(0, J + 1))
        v = st[c] + rng.normal(0, 0.5) if c < J else abs(st[c] + rng.normal(0, 0.3))
        cand = list(cache)
        fast = prog_eval.run(prog, consts, st, prog.comp_prog[c], O, moved=c, val=v, cache=cache, cand=cand)
        slow = prog_eval.logpost(prog, consts, st, O, moved=c, val=v)
        assert fast == slow, (step, c)
        if rng.random() < 0.5:                                           # accept: commit the touched terms
            st[c] = v
            for k in range(prog.touch_off[c], prog.touch_off[c + 1]):
                cache[prog.touch_terms[k]] = cand[prog.touch_terms[k]]

    K, n_pts = 3, 40
    X = np.column_stack([np.ones(n_pts), rng.normal(0, 0.5, (n_pts, K - 1))])
    beta_true = rng.normal(0, 0.3, K)
    yy = rng.poisson(np.exp(X @ beta_true)).astype(float)

    def poisreg(state, d):
        lp = 0
        for k in range(K):
            lp += ld.norm(state.beta[k], 0, 10)
        for i in mcmc.points(len(d.y)):
            eta = 0
            for k in range(K):
                eta += d.X[i][k] * state.beta[k]
            lp += ld.pois(d.y[i], mcmc.Math.exp(eta))
        return lp
    params = {"beta": {"type": "real", "dim": [K]}}
    prog, _, _ = _trace(pkg, poisreg, params, {"y": yy.tolist(), "X": X.tolist()})
    assert prog.summary[-1] == f"plate POIS_LOGLIN n={n_pts} K={K}"
    consts = prog_eval.fold_constants(prog, orc.lib())
    st = list(rng.normal(0, 0.3, K))
    ref, _ = _oracle_logpost(orc, "pois_reg", {"y": yy, "X": X}, params, st)
    assert abs(prog_eval.logpost(prog, consts, st, orc.lib()) - ref) <= 1e-11 * abs(ref)


def test_poisson_plate_with_a_negative_count_is_minus_infinity(pkg, orc):
    """ld.pois of a negative count is -Infinity (distributions.js:282-284). The factorised plate would carry lfactorial(-1) = NaN in
    its constant, so such data keeps the term-by-term loop: log_post is -Infinity, as the oracle's, at every state."""
    ld, mcmc = pkg.ld, pkg.mcmc
    rng = np.random.default_rng(6)
    K, n_pts = 2, 30
    X = np.column_stack([np.ones(n_pts), rng.normal(0, 0.5, n_pts)])
    yy = rng.poisson(1.5, n_pts).astype(float)
    yy[11] = -1.0

    def poisreg(state, d):
        lp = 0
        for k in range(K):
            lp += ld.norm(state.beta[k], 0, 10)
        for i in mcmc.points(len(d.y)):
            lp += ld.pois(d.y[i], mcmc.Math.exp(d.X[i][0] * state.beta[0] + d.X[i][1] * state.beta[1]))
        return lp
    params = {"beta": {"type": "real", "dim": [K]}}
    prog, _, _ = _trace(pkg, poisreg, params, {"y": yy.tolist(), "X": X.tolist()})
    assert prog.summary[-1] == f"plate GENERIC n={n_pts} body=LD_POIS"
    consts = prog_eval.fold_constants(prog, orc.lib())
    for _ in range(5):
        st = list(rng.normal(0, 0.3, K))
        ref, _ = _oracle_logpost(orc, "pois_reg", {"y": yy, "X": X}, params, st)
        assert ref == -np.inf and prog_eval.logpost(prog, consts, st, orc.lib()) == -np.inf


def test_pre_evaluated_statistics_programs(pkg, orc, monkeypatch):
    """amwg.h stat_prog: NORM_IID plates whose mean reads one component are split into S (one data pass per sweep, at every
    component's proposal) and f(S, sd); the per-component programs then hold no O(N) work and still give the full program's value."""
    ld = pkg.ld
    rng = np.random.default_rng(3)
    J, per = 4, 16
    g = np.repeat(np.arange(J), per)
    y = rng.normal(100, 20, J)[g] + rng.normal(0, 5, J * per)

    def hier(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]] * 1.0, state.sigma * 1.0)     # operands that are expressions, not bare components
        return lp
    params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    prog, _, D = _trace(pkg, hier, params, {"y": y.tolist(), "g": g.tolist()})
    assert prog.summary[-1].startswith("pre-evaluated statistics: 4 plate(s), 64 points")
    assert prog.stat_prog >= 0 and prog.n_sum_terms == 2 * J + 1 and prog.n_terms == 3 * J + 1 and not prog.block_params
    assert [prog.touch_off[c + 1] - prog.touch_off[c] for c in range(D)] == [3] * J + [J + 1]
    O = orc.lib()
    consts = prog_eval.fold_constants(prog, O)
    st = list(rng.normal(100, 20, J)) + [4.0]
    ref, _ = _oracle_logpost(orc, "hier_norm", {"y": y, "g": g}, params, st)
    cache = [None] * prog.n_terms
    full0 = prog_eval.run(prog, consts, st, prog.logpost_prog, O, cache=cache)            # fills terms AND statistics
    assert None not in cache and abs(full0 - ref) <= 1e-12 * abs(ref)
    for sweep in range(25):
        props = [st[c] + rng.normal(0, 0.5) if c < J else abs(st[c] + rng.normal(0, 0.3)) for c in range(D)]
        cand = list(cache)
        prog_eval.run(prog, consts, st, prog.stat_prog, O, cache=cache, cand=cand, props=props)       # (b) one data pass
        for c in rng.permutation(D):                                                                   # (c) the steps, in any order
            c = int(c)
            fast = prog_eval.run(prog, consts, st, prog.comp_prog[c], O, moved=c, val=props[c], cache=cache, cand=cand)
            slow = prog_eval.run(prog, consts, st, prog.logpost_prog, O, moved=c, val=props[c])
            assert fast == slow, (sweep, c)
            if rng.random() < 0.5:
                st[c] = props[c]
                for k in range(prog.touch_off[c], prog.touch_off[c + 1]):
                    cache[prog.touch_terms[k]] = cand[prog.touch_terms[k]]
    # config-2 shape: both parameters scalar, the plate's mean is mu: lowered the same way (the run-time specialised sweep makes
    # one data pass per sweep pay for two-component models too); AMWG_STAT_LOWERING=0 keeps the full program
    monkeypatch.setenv("AMWG_STAT_LOWERING", "0")
    prog, _, _ = _trace(pkg, models.norm_post_readme(ld), models.PARAMS1, config2_data().tolist())
    assert prog.stat_prog == -1 and prog.n_terms == 0
    monkeypatch.delenv("AMWG_STAT_LOWERING")
    prog, _, _ = _trace(pkg, models.norm_post_readme(ld), models.PARAMS1, config2_data().tolist())
    assert prog.stat_prog >= 0 and prog.n_sum_terms == 3 and prog.n_terms == 4
    assert list(prog.touch_terms[prog.touch_off[0]:prog.touch_off[1]]) == [0, 3, 2] and list(prog.touch_terms[prog.touch_off[1]:prog.touch_off[2]]) == [1, 2]
    # a mean that reads two components cannot be pre-evaluated; neither can a model with a binary parameter; `faithful` keeps the JS loop
    two = lambda s, d: sum((ld.norm(d[i], s.a + s.b, 1.0) for i in range(len(d))), 0)
    prog, _, _ = _trace(pkg, two, {"a": {"type": "real"}, "b": {"type": "real"}}, list(range(100)))
    assert prog.stat_prog == -1
    prog, _, _ = _trace(pkg, models.spike_bern(ld, pkg.mcmc), {"theta": {"type": "real", "lower": 0, "upper": 1}, "m": {"type": "binary"}},
                        {"x": [1.0, 0.0] * 64})
    assert prog.stat_prog == -1


def test_control_flow_on_binary_parameters_is_recorded_per_configuration(pkg, orc):
    """`if (m === 0) ... else ...` (tests/test_data.js:163-168) written as a plain Python `if`: one program per value of m,
    each bit-faithful to the oracle's C model."""
    y = config3_data()
    prog, _, _ = _trace(pkg, models.spike_bern_literal(pkg.ld), models.PARAMS_SPIKE, {"x": y.tolist()})
    assert prog.variant_comps == [1] and len(prog.variant_logpost) == 2
    consts = prog_eval.fold_constants(prog, orc.lib())
    rng = np.random.default_rng(4)
    for _ in range(20):
        st = [rng.uniform(0.01, 0.99), float(rng.integers(0, 2))]
        ref, _ = _oracle_logpost(orc, "spike_bern", {"x": y}, models.PARAMS_SPIKE, st)
        assert prog_eval.logpost(prog, consts, st, orc.lib()) == ref
        other = 1.0 - st[1]                       # the binary stepper evaluates the other value of m as the "moved" component
        ref2, _ = _oracle_logpost(orc, "spike_bern", {"x": y}, models.PARAMS_SPIKE, [st[0], other])
        assert prog_eval.logpost(prog, consts, st, orc.lib(), moved=1, val=other) == ref2
    x = [float(v) for v in np.random.default_rng(7).negative_binomial(21, 0.5, 12)]
    prog, _, _ = _trace(pkg, models.complex_model_post_literal(pkg.ld), models.PARAMS_COMPLEX, x)
    assert prog.variant_comps == [2]
    consts = prog_eval.fold_constants(prog, orc.lib())
    for m in (0.0, 1.0):
        st = [0.37, 4.0, m]
        ref, _ = _oracle_logpost(orc, "complex", {"x": np.array(x)}, models.PARAMS_COMPLEX, st)
        assert prog_eval.logpost(prog, consts, st, orc.lib()) == ref


def test_untraceable_closures_throw(pkg):
    ld, mcmc = pkg.ld, pkg.mcmc

    def branches(state, data):
        if state.theta > 0.5:                        # control flow on a REAL parameter cannot be recorded
            return ld.bern(1, 0.5)
        return ld.bern(1, state.theta)
    with pytest.raises(pkg.JsThrow, match="use mcmc.where"):
        _trace(pkg, branches, models.PARAMS_SPIKE, None)
    with pytest.raises(pkg.JsThrow, match="returned undefined"):
        _trace(pkg, lambda s, d: None, models.PARAMS_NORM, None)
