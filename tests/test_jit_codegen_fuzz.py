"""Randomly composed models through the code generator, executed on the host (tests/test_jit_codegen_semantics.py's harness).

Each seed builds a log_post out of the operations a user can write -- arithmetic, Math.log/exp/sqrt/abs/pow/min/max, comparisons and
mcmc.where, every scalar ld.*, loops over data columns with data-indexed parameters, a Bernoulli column, derived quantities, real / int /
binary / vector parameters -- lowers it with the product's tracer, specialises it (csrc/amwg_jit.cuh), compiles the generated code for
the host and compares jit_logpost() / jit_derived() with the bytecode run on the oracle's arithmetic at random states, bit for bit.
Half of the models are lowered as with AMWG_TERM_CACHE=0 (every step runs the full program); of the others, those the generator
turns down (they step with a term cache) are counted, not failed."""
import os

import numpy as np
import pytest

from test_jit_codegen_semantics import HostProgram


def _build(pkg, seed):
    ld, mcmc = pkg.ld, pkg.mcmc
    M = mcmc.Math
    rng = np.random.default_rng(seed)
    params = {"theta": {"type": "real", "lower": 0, "upper": 1}, "mu": {"type": "real"}, "s": {"type": "real", "lower": 0, "init": 2},
              "n": {"type": "int", "lower": 1, "init": 3}, "m": {"type": "binary"}, "v": {"type": "real", "dim": [3]}}
    n_pts = int(rng.integers(5, 40))
    data = {"y": rng.normal(1, 2, n_pts).tolist(), "g": rng.integers(0, 3, n_pts).astype(float).tolist(),
            "x": (rng.random(n_pts) < 0.6).astype(float).tolist(), "k": rng.poisson(3, n_pts).astype(float).tolist()}
    plan = {"terms": [int(v) for v in rng.integers(0, 1 << 30, int(rng.integers(2, 7)))], "loops": [int(v) for v in rng.integers(0, 4, int(rng.integers(0, 3)))],
            "derived": int(rng.integers(0, 3)), "seed": seed}

    def log_post(state, d):
        r = np.random.default_rng(plan["seed"] + 1)               # the same choices every time the closure is traced

        def leaf():
            k = int(r.integers(0, 9))
            if k == 0: return state.theta
            if k == 1: return state.mu
            if k == 2: return state.s
            if k == 3: return state.n
            if k == 4: return state.m
            if k == 5: return state.v[int(r.integers(0, 3))]
            return float(np.round(r.normal(0, 2), 3))

        def expr(depth):
            if depth <= 0 or r.random() < 0.25:
                return leaf()
            k = int(r.integers(0, 14))
            a = expr(depth - 1)
            if k == 0: return a + expr(depth - 1)
            if k == 1: return a - expr(depth - 1)
            if k == 2: return a * expr(depth - 1)
            if k == 3: return a / (M.abs(expr(depth - 1)) + 0.5)
            if k == 4: return M.log(M.abs(a) + 0.1)
            if k == 5: return M.exp(a * 0.1)
            if k == 6: return M.sqrt(M.abs(a))
            if k == 7: return M.pow(M.abs(a) + 0.1, float(r.choice([2.0, 0.5, 3.0, 1.7])))
            if k == 8: return M.max(a, expr(depth - 1))
            if k == 9: return M.min(a, expr(depth - 1))
            if k == 10: return mcmc.where(a > expr(depth - 1), expr(depth - 1), a)
            if k == 11: return mcmc.where(state.m == 0, a, expr(depth - 1))
            if k == 12: return mcmc.where((a <= 0.3) | (state.n >= 4), 1.5, a) if hasattr(a, "__or__") and not isinstance(a, float) else a
            return -a

        pos = lambda e: M.abs(e) + 0.2
        prob = lambda e: 1 / (1 + M.exp(-e))
        lp = 0
        for t in plan["terms"]:
            k = t % 22
            e1, e2 = expr(2), expr(2)
            if k == 0: lp += ld.norm(e1, e2, pos(expr(1)))
            elif k == 1: lp += ld.beta(state.theta, pos(e1), pos(e2))
            elif k == 2: lp += ld.pois(state.n, pos(e1))
            elif k == 3: lp += ld.bern(state.m, prob(e1))
            elif k == 4: lp += ld.binom(state.n, state.n + 4, prob(e1))
            elif k == 5: lp += ld.gamma(state.s, pos(e1), pos(e2))
            elif k == 6: lp += ld.unif(state.theta, -0.5, pos(e1))
            elif k == 7: lp += ld.exp(state.s, pos(e1))
            elif k == 8: lp += ld.cauchy(e1, e2, pos(expr(1)))
            elif k == 9: lp += ld.laplace(e1, e2, pos(expr(1)))
            elif k == 10: lp += ld.logis(e1, e2, pos(expr(1)))
            elif k == 11: lp += ld.lnorm(state.s, e1, pos(e2))
            elif k == 12: lp += ld.nbinom(state.n, pos(e1), prob(e2))
            elif k == 13: lp += ld.t(e1, e2, pos(expr(1)), pos(expr(1)))
            elif k == 14: lp += ld.weibull(state.s, pos(e1), pos(e2))
            elif k == 15: lp += ld.pareto(state.s + 1, pos(e1) * 0.1, pos(e2))
            elif k == 16: lp += ld.invgamma(state.s, pos(e1), pos(e2))
            elif k == 17: lp += ld.hyper(state.n, state.n + 6, 9, 5)
            elif k == 18: lp += ld.lgamma(pos(e1)) - ld.lfactorial(state.n) + ld.lchoose(state.n + 3, 2) - ld.lbeta(pos(e2), 1.5)
            elif k == 19: lp += e1 * 0.01
            elif k == 20: lp += ld.norm(state.v[0], state.v[1] * state.m, pos(state.v[2]))
            else: lp += ld.beta(prob(e1), 2, 3)
        for kind in plan["loops"]:
            for i in range(len(d.y)):
                if kind == 0: lp += ld.norm(d.y[i], state.mu + state.v[d.g[i]], state.s)
                elif kind == 1: lp += ld.bern(d.x[i], mcmc.where(state.m == 0, 0.5, state.theta))
                elif kind == 2: lp += ld.pois(d.k[i], M.exp(state.mu * 0.1 + state.v[d.g[i]] * 0.05) + 0.1)
                else: lp += ld.laplace(d.y[i], state.v[d.g[i]] * d.x[i], state.s + 0.5)
        if plan["derived"] >= 1: state.z1 = expr(2)
        if plan["derived"] >= 2: state.z2 = state.s * state.s + state.n
        return lp
    return params, log_post, data


@pytest.mark.parametrize("block", range(4))
def test_random_models_generated_code_equals_the_program(pkg, orc, tmp_path, block):
    compiled = declined = 0
    for seed in range(100 * block, 100 * block + 8):
        params, log_post, data = _build(pkg, seed)
        sub = tmp_path / f"m{seed}"
        sub.mkdir()
        try:
            hp = HostProgram(pkg, orc, sub, params, log_post, data, faithful=bool(seed & 1), _force_full=bool(seed & 2))
        except AssertionError as e:
            if "term cache" in str(e):
                declined += 1
                continue
            raise
        hp.check(np.random.default_rng(seed), trials=120)
        compiled += 1
    assert compiled >= 4, (compiled, declined)


# ---- the production lowering: random Normal-plate models, statistics sweep vs full-program sweep (both emulated) ----------------------
def _build_stat(pkg, seed):
    ld, mcmc = pkg.ld, pkg.mcmc
    M = mcmc.Math
    rng = np.random.default_rng(1000 + seed)
    J = int(rng.choice([1, 3, 8, 12]))
    per = int(rng.integers(40, 100))
    hyper = bool(rng.integers(0, 2)) and J > 1
    two = bool(rng.integers(0, 2))
    derived = bool(rng.integers(0, 2))
    lin = (float(np.round(rng.uniform(0.5, 2.0), 2)), float(np.round(rng.normal(0, 1), 2)))
    pri = [int(v) for v in rng.integers(0, 5, 4)]
    centre = float(rng.normal(10, 3))
    g = np.repeat(np.arange(J), per)
    y = rng.normal(centre, 2.0, J * per) + (np.repeat(rng.normal(0, 1.5, J), per) if J > 1 else 0.0)
    data = {"y": y.tolist(), "g": g.astype(float).tolist(), "y2": rng.normal(-3, 1.0, 60).tolist()}
    params = {"sigma": {"type": "real", "lower": 0, "init": 2.0}}
    if J > 1: params["mu"] = {"type": "real", "dim": [J], "init": centre}
    else: params["a"] = {"type": "real", "init": centre}
    if hyper: params.update({"m0": {"type": "real", "init": centre}, "tau": {"type": "real", "lower": 0, "init": 2.0}})
    if two: params.update({"b": {"type": "real", "init": -3.0}, "s2": {"type": "real", "lower": 0, "init": 1.0}})

    def prior(kind, x, loc, scale):
        if kind == 0: return ld.norm(x, loc, scale * 20)
        if kind == 1: return ld.cauchy(x, loc, scale * 5)
        if kind == 2: return ld.laplace(x, loc, scale * 10)
        if kind == 3: return ld.logis(x, loc, scale * 8)
        return ld.unif(x, loc - 100, loc + 100)

    def log_post(state, d):
        lp = 0
        if J > 1:
            for j in range(J):
                lp += ld.norm(state.mu[j], state.m0, state.tau) if hyper else prior(pri[0], state.mu[j], centre, 1.0)
        else:
            lp += prior(pri[0], state.a, centre, 1.0)
        if hyper:
            lp += prior(pri[1], state.m0, centre, 2.0)
            lp += ld.gamma(state.tau, 2, 0.5)
        lp += ld.gamma(state.sigma, 2, 0.5) if pri[2] < 2 else ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]] if J > 1 else state.a * lin[0] + lin[1], state.sigma)
        if two:
            lp += prior(pri[3], state.b, -3.0, 1.0)
            lp += ld.lnorm(state.s2, 0, 1)
            for i in range(len(d.y2)):
                lp += ld.norm(d.y2[i], state.b, state.s2)
        if derived:
            state.prec = 1 / (state.sigma * state.sigma)
        return lp
    return params, log_post, data


@pytest.mark.parametrize("block", range(3))
def test_random_normal_plate_models_statistics_sweep_equals_full_program_sweep(pkg, orc, tmp_path, block):
    """The two specialised kernels on the same random model and Philox streams: the statistics sweep (production lowering: one data pass
    per sweep, steps decided on term differences, component classes / term loops / index-ordered blocks) against the full-program sweep
    of the bit-faithful lowering. They may differ where exp(delta) falls within rounding of an accept uniform -- in 16 chains x 40 sweeps
    per model that did not happen once when this was written; the test allows one chain in sixteen."""
    from test_jit_codegen_semantics import HostKernel, HostStatKernel
    ran = 0
    for seed in range(10 * block, 10 * block + 5):
        params, log_post, data = _build_stat(pkg, seed)
        sub = tmp_path / f"s{seed}"
        sub.mkdir()
        probe = pkg.mcmc.AmwgSampler(params, log_post, data, {"chains": 4096, "_model_only": True})
        if probe._program.stat_prog < 0:
            continue                                              # the tracer did not choose the statistics lowering for this one
        hs = HostStatKernel(pkg, orc, sub, params, log_post, data)
        (sub / "full").mkdir()
        hf = HostKernel(pkg, orc, sub / "full", params, log_post, data, faithful=True, _force_full=True)
        chains, sweeps = 16, 40
        out_s, _ = hs.run(chains, 31 + seed, 5 + seed, sweeps)
        out_f, _st, _n, _a = hf.run(chains, 31 + seed, 5 + seed, sweeps)
        D = hs.D
        same = (out_s[:, :D, :].view(np.uint64) == out_f[:, :D, :].view(np.uint64)).all(axis=(0, 1))
        assert same.mean() >= 15 / 16, (seed, same.mean())
        assert np.isfinite(out_s).all() and np.unique(out_s[-1, 0]).size > 8
        ran += 1
    assert ran >= 3, ran


def test_a_one_row_matrix_of_group_means_is_stepped_component_by_component(pkg, orc, tmp_path):
    """dim [1, n] (tests/test_data.js:176 declares p that way): one top-level entry, n components. The specialised skeletons compile their
    multi-component stepping in on JMAX_DIM0 > 1 -- which has to hold for such a parameter too (it did not: every round stepped
    component 0; found by running the hierarchical-binomial golden script through the emulated kernel). Both kernels, same draws."""
    from test_jit_codegen_semantics import HostKernel, HostStatKernel
    ld = pkg.ld
    J, per = 6, 50
    rng = np.random.default_rng(3)
    g = np.repeat(np.arange(J), per)
    y = rng.normal(10, 2, J * per) + np.repeat(rng.normal(0, 1.5, J), per)
    P = {"mu": {"type": "real", "dim": [1, J], "init": 10.0}, "sigma": {"type": "real", "lower": 0, "init": 2.0}}

    def log_post(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[0][j], 10, 20)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[0][d.g[i]], state.sigma)
        return lp
    data = {"y": y.tolist(), "g": g.astype(float).tolist()}
    hs = HostStatKernel(pkg, orc, tmp_path, P, log_post, data)
    assert "#define JMAX_DIM0 2" in hs.src
    (tmp_path / "full").mkdir()
    hf = HostKernel(pkg, orc, tmp_path / "full", P, log_post, data, faithful=True, _force_full=True)
    out_s, _ = hs.run(16, 9, 4, 40)
    out_f, _st, _n, _a = hf.run(16, 9, 4, 40)
    assert (out_s[:, :J + 1, :].view(np.uint64) == out_f[:, :J + 1, :].view(np.uint64)).all(axis=(0, 1)).mean() >= 15 / 16
    assert all(np.unique(out_s[-1, c]).size > 8 for c in range(J + 1))          # every component moved


# ---- stepping logic over random parameter shapes: the emulated full-program kernel against the oracle's restatement of mcmc.js --------
def _build_shapes(pkg, seed):
    ld, mcmc = pkg.ld, pkg.mcmc
    rng = np.random.default_rng(5000 + seed)
    n_named = int(rng.choice([1, 2, 3, 5, 18, 21]))
    params, comps = {}, []                                          # comps: (name, index tuple, type)
    for k in range(n_named):
        t = str(rng.choice(["real", "real", "int", "binary"]))
        shape = rng.choice(["scalar", "vec", "mat", "row"], p=[0.55, 0.2, 0.15, 0.1]) if n_named < 10 else "scalar"
        dim = {"scalar": None, "vec": [int(rng.integers(2, 6))], "mat": [int(rng.integers(2, 4)), int(rng.integers(2, 4))], "row": [1, int(rng.integers(2, 6))]}[str(shape)]
        d = {"type": t}
        if dim: d["dim"] = dim
        if t == "real" and rng.random() < 0.4: d.update({"lower": -2.0, "upper": 6.0})
        if t == "int": d.update({"lower": int(rng.integers(-6, 0)), "upper": int(rng.integers(3, 9))})
        name = "q%d" % k
        params[name] = d
        for ix in (np.ndindex(*dim) if dim else [()]):
            comps.append((name, tuple(int(v) for v in ix), t))
    locs = rng.normal(1, 1.5, len(comps)).round(2).tolist()
    couple = [(int(a), int(b)) for a, b in rng.integers(0, len(comps), (min(3, len(comps)), 2))]

    def ref(state, name, ix):
        v = state[name]
        for i in ix:
            v = v[i]
        return v

    def log_post(state, d=None):
        lp = 0
        vals = [ref(state, n, ix) for n, ix, _t in comps]
        for (n, ix, t), v, loc in zip(comps, vals, locs):
            lp += ld.bern(v, 0.3 + 0.05 * (len(ix) + 1)) if t == "binary" else ld.norm(v, loc, 1.5)
        for a, b in couple:                                           # a few couplings: the log_post is not a product of independent factors
            lp += ld.norm(vals[a] - vals[b], 0.0, 2.0)
        return lp
    return params, log_post


@pytest.mark.parametrize("seed", range(8))
def test_random_parameter_shapes_stepping_equals_the_oracle(pkg, orc, tmp_path, seed):
    """Scalars, vectors, matrices, one-row matrices, real / bounded real / int / binary, up to 21 named parameters (more than 16: the
    substepper order lives in a per-chain byte array): the emulated specialised kernel's shuffles, visiting orders, proposals, bounds
    checks and accept decisions against the oracle (mcmc.js restated in C) stepping the same log_post -- the model's bytecode evaluated
    with the oracle's arithmetic -- on the same Philox streams. Bit for bit, 30 sweeps inside the first adaptation batch."""
    import prog_eval
    from test_jit_codegen_semantics import HostKernel
    params, log_post = _build_shapes(pkg, seed)
    hk = HostKernel(pkg, orc, tmp_path, params, log_post, None, _force_full=True)
    sweeps, first, sd = 30, 123 + seed, 77 + seed
    hk.start(2, first, sd)
    out = hk.sweeps(sweeps)
    prog, consts, O = hk.prog, hk.consts, hk.O
    for c in range(2):
        o = orc.OracleSampler(lambda st: prog_eval.logpost(prog, consts, st, O), None, params, seed=sd, chain=first + c)
        refd = o.sample(sweeps)
        e = 0
        for name in hk.s.params:
            n = int(np.prod(hk.s.params[name]["dim"]))
            want = np.asarray(refd[name], np.float64).reshape(sweeps, n)
            assert np.array_equal(out[:, e:e + n, c].view(np.uint64), want.view(np.uint64)), (seed, name)
            e += n
        assert int(hk.rng_n[c]) == o.rng_position()


def test_a_vector_longer_than_256_keeps_its_visiting_order_in_global_memory(pkg, orc, tmp_path):
    """dim[0] = 260 > 256: the per-sweep visiting order of the parameter is 16-bit rows of a per-chain global array (amwg_tma.cuh
    ord_get / ord_set) instead of a local byte array. Emulated specialised kernel against the oracle, as above."""
    import prog_eval
    from test_jit_codegen_semantics import HostKernel
    ld = pkg.ld
    J = 260
    params = {"x": {"type": "real", "dim": [J]}, "s": {"type": "real", "lower": 0}}

    def lp_wide(state, d=None):
        lp = ld.gamma(state.s, 2, 1)
        for j in range(J):
            lp += ld.norm(state.x[j], 0.01 * j, state.s)
        return lp
    hk = HostKernel(pkg, orc, tmp_path, params, lp_wide, None, _force_full=True)
    assert "#define JMAX_DIM0 260" in hk.s.jit_compile_check()[2]
    sweeps = 6
    hk.start(1, 3, 43)
    assert hk.order_ext is not None
    out = hk.sweeps(sweeps)
    prog, consts, O = hk.prog, hk.consts, hk.O
    o = orc.OracleSampler(lambda st: prog_eval.logpost(prog, consts, st, O), None, params, seed=43, chain=3)
    ref = o.sample(sweeps)
    assert np.array_equal(out[:, :J, 0].view(np.uint64), np.asarray(ref["x"], np.float64).reshape(sweeps, J).view(np.uint64))
    assert np.array_equal(out[:, J, 0].view(np.uint64), np.asarray(ref["s"], np.float64).reshape(sweeps).view(np.uint64))
    assert int(hk.rng_n[0]) == o.rng_position()


def _build_stat_shapes(pkg, seed):
    """Normal plates whose means are a scalar, a vector, a one-row matrix or a matrix indexed by two data columns, beside parameters
    that only have priors: bounded reals and ints (their proposals can fall out of bounds: no accept uniform is drawn then)."""
    ld = pkg.ld
    rng = np.random.default_rng(9000 + seed)
    kind = str(rng.choice(["scalar", "vec", "row", "mat"]))
    n_extra = int(rng.choice([0, 2, 4, 16]))
    n = int(rng.integers(60, 140))
    R, Cc = 3, 4
    g = rng.integers(0, {"scalar": 1, "vec": 5, "row": 5, "mat": R}[kind], n)
    h = rng.integers(0, Cc, n) if kind == "mat" else np.zeros(n, dtype=np.int64)
    order = np.lexsort((h, g))                                      # points grouped by the component their mean reads (contiguous plates)
    g, h = g[order], h[order]
    y = rng.normal(5, 2, n) + 0.7 * g
    data = {"y": y.tolist(), "g": g.astype(float).tolist(), "h": h.astype(float).tolist()}
    params = {"sigma": {"type": "real", "lower": 0, "init": 2.0}}
    params["mu"] = {"scalar": {"type": "real", "init": 5.0}, "vec": {"type": "real", "dim": [5], "init": 5.0},
                    "row": {"type": "real", "dim": [1, 5], "init": 5.0}, "mat": {"type": "real", "dim": [R, Cc], "init": 5.0}}[kind]
    extras = []
    for k in range(n_extra):
        t = "int" if k % 3 == 0 else "real"
        d = {"type": t, "lower": -3 if t == "int" else -1.5, "upper": 4 if t == "int" else 2.5, "init": 0}
        params["e%d" % k] = d
        extras.append(("e%d" % k, float(rng.normal(0.5, 1))))

    def log_post(state, d):
        lp = ld.gamma(state.sigma, 2, 0.5)
        mu = state.mu
        if kind == "scalar": lp += ld.norm(mu, 5, 10)
        elif kind == "vec":
            for j in range(5): lp += ld.norm(mu[j], 5, 10)
        elif kind == "row":
            for j in range(5): lp += ld.cauchy(mu[0][j], 5, 4)
        else:
            for r in range(R):
                for c in range(Cc): lp += ld.norm(mu[r][c], 5, 10)
        for name, loc in extras:
            lp += ld.norm(state[name], loc, 1.2)
        for i in range(len(d.y)):
            m = mu if kind == "scalar" else (mu[d.g[i]] if kind == "vec" else (mu[0][d.g[i]] if kind == "row" else mu[d.g[i]][d.h[i]]))
            lp += ld.norm(d.y[i], m, state.sigma)
        return lp
    return params, log_post, data


@pytest.mark.parametrize("seed", range(8))
def test_random_shapes_statistics_sweep_equals_full_program_sweep(pkg, orc, tmp_path, seed):
    from test_jit_codegen_semantics import HostKernel, HostStatKernel
    params, log_post, data = _build_stat_shapes(pkg, seed)
    probe = pkg.mcmc.AmwgSampler(params, log_post, data, {"chains": 4096, "_model_only": True})
    if probe._program.stat_prog < 0:
        pytest.skip("the tracer did not choose the statistics lowering for this model")
    hs = HostStatKernel(pkg, orc, tmp_path, params, log_post, data)
    (tmp_path / "full").mkdir()
    hf = HostKernel(pkg, orc, tmp_path / "full", params, log_post, data, faithful=True, _force_full=True)
    chains, sweeps = 12, 35
    out_s, rng_s = hs.run(chains, 400 + seed, 60 + seed, sweeps)
    out_f, _st, rng_f, _a = hf.run(chains, 400 + seed, 60 + seed, sweeps)
    D = hs.D
    same = (out_s[:, :D, :].view(np.uint64) == out_f[:, :D, :].view(np.uint64)).all(axis=(0, 1))
    assert same.mean() >= 11 / 12, (seed, same.mean())
    assert np.array_equal(rng_s[same], rng_f[same])               # and the same number of Math.random() calls


def test_statistics_sweep_bounded_block_derived_thinning_and_acceptance_counts(pkg, orc, tmp_path):
    """A block of eight group means with TIGHT bounds (proposals fall outside: no accept uniform, no evaluation, mcmc.js:520-522 -- the
    index-ordered block path that cannot pre-draw its uniforms), derived quantities recorded with their state, thinning by 3, and
    adaptation switched off for half of the components (acceptance counts are only kept where it is on): statistics sweep against
    full-program sweep, both emulated -- draws, derived values, stream positions and acceptance counters."""
    from test_jit_codegen_semantics import HostKernel, HostStatKernel
    ld = pkg.ld
    J, per = 8, 40
    rng = np.random.default_rng(12)
    g = np.repeat(np.arange(J), per)
    y = rng.normal(10, 2, J * per) + np.repeat(rng.normal(0, 1.5, J), per)
    P = {"mu": {"type": "real", "dim": [J], "init": 10.0, "lower": 8.5, "upper": 11.5}, "sigma": {"type": "real", "lower": 0, "init": 2.0}}

    def log_post(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 10, 20)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        state.prec = 1 / (state.sigma * state.sigma)
        state.spread = state.mu[0] - state.mu[J - 1]
        return lp
    data = {"y": y.tolist(), "g": g.astype(float).tolist()}
    hs = HostStatKernel(pkg, orc, tmp_path, P, log_post, data)
    assert "#define JBLOCK 0" in hs.src and "#define JBLOCK_FREE 0" in hs.src and "#define JN_DERIVED 2" in hs.src
    (tmp_path / "full").mkdir()
    hf = HostKernel(pkg, orc, tmp_path / "full", P, log_post, data, faithful=True, _force_full=True)
    chains, sweeps, thin = 16, 45, 3
    adapting = [c % 2 for c in range(J + 1)]
    out_s, rng_s = hs.run(chains, 21, 8, sweeps, thin=thin, adapting=adapting)
    hf.start(chains, 21, 8)
    hf.adapting[:] = adapting
    out_f = hf.sweeps(sweeps, thin=thin)
    assert out_s.shape == out_f.shape == (15, J + 3, chains)
    same = (out_s.view(np.uint64) == out_f.view(np.uint64)).all(axis=(0, 1))
    assert same.mean() >= 15 / 16, same.mean()
    assert np.array_equal(rng_s[same], hf.rng_n[same])
    assert np.array_equal(hs.acc[:, same], hf.acc[:, same]) and hs.acc[1::2].sum() > 0 and hs.acc[0::2].sum() == 0
    # the bounds bind: some proposals were refused without a uniform, so the chains consumed different numbers of Math.random() calls
    assert np.unique(rng_s).size > 4 and out_s[:, :J, :].min() >= 8.5 and out_s[:, :J, :].max() <= 11.5


# ---- the seeds tests/test_gpu_fuzz.py runs on the device: each one is cleared here first, on the emulated kernels it reaches there, under
#      the strict shim (bulk copies, mbarrier accounting, declared shared memory, device-shaped columns) and, in a subprocess, ASan -------
GPU_SEEDS = (("generic", 3), ("generic", 7), ("stat", 4), ("stat", 51), ("shapes", 2), ("shapes", 7))


def gpu_model(pkg, kind, seed):
    """(params, log_post, data) of one of the builders above"""
    if kind == "generic":
        return _build(pkg, seed)
    if kind == "stat":
        return _build_stat(pkg, seed)
    params, log_post = _build_shapes(pkg, seed)
    return params, log_post, None


@pytest.mark.parametrize("kind,seed", GPU_SEEDS)
def test_gpu_fuzz_seeds_on_the_emulated_kernels(pkg, orc, tmp_path, kind, seed):
    """The full-program sweep of the faithful lowering (what AMWG_JIT=1 runs for a faithful handle, with AMWG_TERM_CACHE=0 where that
    lowering keeps a term cache) against the oracle stepping the same program, bit for bit, with the stream positions; for a model the
    tracer gives the statistics lowering, also the statistics sweep against that full-program sweep (one chain in sixteen may differ)."""
    import prog_eval
    from test_jit_codegen_semantics import HostKernel, HostStatKernel
    params, log_post, data = gpu_model(pkg, kind, seed)
    (tmp_path / "full").mkdir()
    hk = HostKernel(pkg, orc, tmp_path / "full", params, log_post, data, faithful=True, _force_full=True)
    chains, first, sd, sweeps = 4, 30 + seed, 11 + seed, 25
    hk.start(chains, first, sd)
    out = hk.sweeps(sweeps)
    prog, consts, O = hk.prog, hk.consts, hk.O
    for c in range(chains):
        o = orc.OracleSampler(lambda st: prog_eval.logpost(prog, consts, st, O), None, params, seed=sd, chain=first + c)
        refd = o.sample(sweeps)
        e = 0
        for name in hk.s.params:
            n = int(np.prod(hk.s.params[name]["dim"]))
            want = np.asarray(refd[name], np.float64).reshape(sweeps, n)
            assert np.array_equal(out[:, e:e + n, c].view(np.uint64), want.view(np.uint64)), (kind, seed, name, c)
            e += n
        assert int(hk.rng_n[c]) == o.rng_position()
    if kind == "stat":
        probe = pkg.mcmc.AmwgSampler(params, log_post, data, {"chains": 4096, "_model_only": True})
        assert probe._program.stat_prog >= 0
        hs = HostStatKernel(pkg, orc, tmp_path, params, log_post, data)
        out_s, rng_s = hs.run(16, first, sd, sweeps, thin=2)
        hk.start(16, first, sd)
        out_f = hk.sweeps(sweeps, thin=2)
        same = (out_s.view(np.uint64) == out_f.view(np.uint64)).all(axis=(0, 1))
        assert same.mean() >= 15 / 16, same.mean()
        assert np.array_equal(rng_s[same], hk.rng_n[same])


def test_gpu_fuzz_seeds_under_address_sanitizer(tmp_path):
    """The cleared seeds again, every emulated kernel built with -fsanitize=address, in a pytest subprocess with g++'s libasan preloaded
    (the test process itself cannot load an instrumented library). Any heap overflow, use after free or misaligned access ends that
    run with a report under `log_path`."""
    import subprocess
    import sys
    lib = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(lib) or not os.path.exists(lib):
        pytest.skip("g++ has no libasan.so here")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = tmp_path / "asan"
    env = dict(os.environ, LD_PRELOAD=lib, ASAN_OPTIONS=f"detect_leaks=0:log_path={log}", AMWG_HOST_SANITIZE="address",
               PYTHONDONTWRITEBYTECODE="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", "-q", "-p", "no:cacheprovider", f"--basetemp={tmp_path / 'run'}",
        os.path.join(root, "tests", "test_jit_codegen_fuzz.py"), "-k", "test_gpu_fuzz_seeds_on_the_emulated_kernels"]
    r = subprocess.run(cmd, cwd=root, env=env, capture_output=True, text=True, timeout=1800)
    reports = sorted(tmp_path.glob("asan*"))
    text = "".join(p.read_text(errors="replace")[:6000] for p in reports)
    assert not reports, text
    assert r.returncode == 0, (r.stdout[-4000:], r.stderr[-4000:])
    assert f"{len(GPU_SEEDS)} passed" in r.stdout, r.stdout[-2000:]
