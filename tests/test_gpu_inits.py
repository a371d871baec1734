"""Per-chain starting points on the GPU: sampler.set_state (amwg_set_state) and options.init_radius (amwg_disperse_state).

set_state must leave every kernel path exactly where construction from the same point would (draws, state, log_post and info bit for
bit), must be a no-op when given the current state mid-run, and must make chain g the reference chain g started there. The dispersal
must be what DESIGN.md §2 defines (tests/init_ref.py restates it over the oracle), independent of sharding, and it must expose the
multimodal posterior that identical starting points hide."""
import ctypes as C
import os
from contextlib import contextmanager

import numpy as np
import pytest

import init_ref
import models
from conftest import PRESIDENTS, config2_data, config3_data

pytestmark = pytest.mark.gpu


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _bits_equal(a, b, what=""):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a.keys()) == list(b.keys()), what
        for k in a:
            _bits_equal(a[k], b[k], what + "/" + str(k))
    elif isinstance(a, (list, tuple)) and not (len(a) and isinstance(a[0], (int, float))):
        assert len(a) == len(b), what
        for k, (x, y) in enumerate(zip(a, b)):
            _bits_equal(x, y, what + "[%d]" % k)
    elif a is None or isinstance(a, (str, bool)):
        assert a == b, what
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.shape == y.shape and x.dtype == y.dtype, what
        if x.dtype == np.float64:
            x, y = x.view(np.uint64), y.view(np.uint64)
        assert np.array_equal(x, y), what


def _run(s):
    s.burn(120)                                   # crosses two adaptation batches
    d = s.sample(60)
    return {"draws": d, "state": s.state, "log_post": s.log_post(), "info": s.info()}


def _with_init(params, values):
    """params with every parameter's init set to one chain's values"""
    out = {k: dict(v) for k, v in params.items()}
    for k, v in values.items():
        out[k]["init"] = float(v) if np.ndim(v) == 0 else np.asarray(v).tolist()
    return out


def _poisreg(ld, mcmc, K):
    def f(state, d):
        lp = 0
        for k in range(K):
            lp += ld.norm(state.beta[k], 0, 10)
        for i in mcmc.points(len(d.y)):
            eta = 0
            for k in range(K):
                eta += d.X[i][k] * state.beta[k]
            lp += ld.pois(d.y[i], mcmc.Math.exp(eta))
        return lp
    return f


def _hier_norm(ld, J):
    def f(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        return lp
    return f


def _case(pkg, name):
    """(params, log_post, data, options, envs, check(sampler)) of one kernel path"""
    ld, mcmc = pkg.ld, pkg.mcmc
    big = 4096 + 37                                # a ragged last CTA: shadow threads take part
    if name in ("stat_specialised", "stat_interpreter"):
        jit = name == "stat_specialised"
        return (models.PARAMS_NORM, models.norm_post_readme(ld), config2_data().tolist(), {"chains": big, "seed": 3},
                {} if jit else {"AMWG_JIT": "0"}, lambda s: s.jit_status()[0] == jit and "plate NORM_IID n=1024" in s.program_summary())
    if name == "full_specialised":
        y = config3_data().tolist()
        return (models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y}, {"chains": big, "seed": 4}, {"AMWG_JIT": "1"},
                lambda s: s.jit_status()[0] and "full-program" in s.jit_status()[1])
    if name == "faithful":
        return (models.PARAMS_NORM, models.norm_post_readme(ld), PRESIDENTS, {"chains": 1000, "seed": 5, "faithful": True}, {},
                lambda s: not s.jit_status()[0])
    if name == "term_cache":
        return (models.PARAMS_HIER_BINOM, models.hierarchical_binomial_post(ld, mcmc), models.BINOM_DATA, {"chains": 300, "seed": 6}, {},
                lambda s: not s.jit_status()[0] and "term cache" in s.jit_status()[1])
    if name == "ring":
        J, per = 8, 4096                           # 256 KB of data: more than a CTA stages
        rng = np.random.default_rng(66)
        g = np.repeat(np.arange(J), per)
        y = rng.normal(100, 20, J)[g] + rng.normal(0, 5, J * per)
        params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
        return (params, _hier_norm(ld, J), {"y": y.tolist(), "g": g.tolist()}, {"chains": 256 + 37, "seed": 7}, {},
                lambda s: "ring" in s.plate_sources())
    if name == "pois":
        K, n = 3, 300
        rng = np.random.default_rng(8)
        X = rng.normal(0, 0.3, (n, K))
        y = rng.poisson(np.exp(X @ np.array([0.5, -0.3, 0.2]))).astype(float)
        return ({"beta": {"type": "real", "dim": [K]}}, _poisreg(ld, mcmc, K), {"y": y.tolist(), "X": X.tolist()}, {"chains": 200, "seed": 9}, {},
                lambda s: any("POIS_LOGLIN" in line for line in s.program_summary()))
    raise KeyError(name)


PATHS = ["stat_specialised", "stat_interpreter", "full_specialised", "faithful", "term_cache", "ring", "pois"]


@pytest.mark.parametrize("name", PATHS)
def test_set_state_equals_construction_at_that_state_on_every_kernel_path(gpu_pkg, name):
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, check = _case(gpu_pkg, name)
    with env(AMWG_JIT="0"):                          # per-chain points inside the support: a short run from the default init
        probe = mcmc.AmwgSampler(params, lp, data, dict(opts, seed=opts["seed"] + 100))
        probe.burn(30)
        per_chain = {k: v for k, v in probe.state.items() if k in params}
        probe.close()
    same = {k: np.asarray(v)[0] for k, v in per_chain.items()}      # chain 0's point, for every chain
    with env(**envs):
        h1 = mcmc.AmwgSampler(_with_init(params, same), lp, data, dict(opts))
        h2 = mcmc.AmwgSampler(params, lp, data, dict(opts))
        h2.set_state(same)
        h3 = mcmc.AmwgSampler(params, lp, data, dict(opts))
        h4 = mcmc.AmwgSampler(_with_init(params, same), lp, data, dict(opts))
        for h in (h3, h4):
            h.set_state(per_chain)
    for h in (h1, h2, h3, h4):
        assert check(h), (name, h.jit_status(), h.plate_sources())
    _bits_equal(h3.state, {**per_chain, **{k: v for k, v in h3.state.items() if k not in params}}, "set_state")
    r1, r2, r3, r4 = (_run(h) for h in (h1, h2, h3, h4))
    _bits_equal(r1, r2, name + " (a)")
    _bits_equal(r3, r4, name + " (b)")
    assert np.all(np.isfinite(np.asarray(r3["log_post"])))


@pytest.mark.parametrize("name", ["stat_specialised", "term_cache", "full_specialised"])
def test_set_state_to_the_current_state_mid_run_changes_nothing(gpu_pkg, name):
    """burn(75) ends in the middle of an adaptation batch: proposal scales, acceptance counts, visiting orders and stream positions
    must carry on as if set_state had not been called."""
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, check = _case(gpu_pkg, name)
    with env(**envs):
        a = mcmc.AmwgSampler(params, lp, data, dict(opts))
        b = mcmc.AmwgSampler(params, lp, data, dict(opts))
    out = []
    for s, touch in ((a, False), (b, True)):
        s.burn(75)
        if touch:
            s.set_state({k: v for k, v in s.state.items() if k in params})
        out.append({"lp0": s.log_post(), "draws": s.sample(50), "state": s.state, "info": s.info()})
    _bits_equal(out[0], out[1], name)


def test_set_state_chains_are_the_reference_chains_started_there(gpu_pkg, orc):
    """The reference's "complex" model (real + int + binary, tests/test_data.js:138-171): after set_state right after construction,
    chains {0, 1, 1234, C-1} are the oracle's chains g started from their own points, draw for draw."""
    Cn, seed = 1300, 21
    x = [float(v) for v in np.random.default_rng(7).negative_binomial(21, 0.5, 12)]
    s = gpu_pkg.mcmc.AmwgSampler(models.PARAMS_COMPLEX, models.complex_model_post(gpu_pkg.ld, gpu_pkg.mcmc), x,
                                 {"chains": Cn, "seed": seed, "faithful": True})
    rng = np.random.default_rng(22)
    pts = {"p1": rng.uniform(0.05, 0.95, Cn), "n1": rng.integers(1, 40, Cn).astype(float), "m": (rng.random(Cn) < 0.5).astype(float)}
    s.set_state(pts)
    s.burn(60)
    got = s.sample(40)
    for g in (0, 1, 1234, Cn - 1):
        params = _with_init(models.PARAMS_COMPLEX, {k: v[g] for k, v in pts.items()})
        q = orc.OracleSampler("complex", {"x": np.array(x)}, params, seed=seed, chain=g)
        q.burn(60)
        ref = q.sample(40)
        for k in ("p1", "n1", "m"):
            _bits_equal(np.asarray(got[k])[:, g], np.asarray(ref[k], np.float64).reshape(-1), "chain %d %s" % (g, k))


def _mixed(ld):
    def f(state, data):
        lp = 0
        lp += ld.norm(state.a, 0, 10)
        lp += ld.norm(state.b, 1, 5)
        lp += ld.norm(state.c, 0, 5)
        lp += ld.unif(state.d, -1, 4)
        lp += ld.pois(state.k, 4)
        lp += ld.bern(state.m, 0.3)
        return lp
    params = {"a": {"type": "real", "init": 1.5}, "b": {"type": "real", "lower": 0, "init": 2}, "c": {"type": "real", "upper": 3, "init": 1},
              "d": {"type": "real", "lower": -1, "upper": 4, "init": 0.5}, "k": {"type": "int", "lower": 0, "upper": 20, "init": 5},
              "m": {"type": "binary"}}
    return params, f


def _expected(O, s, seed, first, count, radius, finite=lambda xs: True):
    comps = init_ref.comps_of(s)
    rows, tries = [], []
    for g in range(first, first + count):
        xs, a = init_ref.disperse_chain(O, seed, g, comps, radius, finite)
        rows.append(xs)
        tries.append(a)
    return np.asarray(rows), np.asarray(tries)


def _flat_state(s):
    st = s.state
    return np.concatenate([np.asarray(st[k], np.float64).reshape(s.local_chains, -1) for k in s.param_names], axis=1)


def test_dispersal_is_the_definition_and_independent_of_sharding(gpu_pkg, orc):
    O = orc.lib()
    params, f = _mixed(gpu_pkg.ld)
    seed, Cn, radius = 5, 1000, 2.0
    a = gpu_pkg.mcmc.AmwgSampler(params, f, None, {"chains": Cn, "seed": seed, "init_radius": radius})
    b = gpu_pkg.mcmc.AmwgSampler(params, f, None, {"chains": Cn, "seed": seed, "init_radius": radius, "first_chain": 600})
    xa, xb = _flat_state(a), _flat_state(b)
    want, tries = _expected(O, a, seed, 0, Cn, radius)
    assert np.all(tries == 0)
    _bits_equal(xa, want, "first_chain 0")
    _bits_equal(xb[:400], xa[600:], "overlapping global chains")
    _bits_equal(xb, _expected(O, b, seed, 600, Cn, radius)[0], "first_chain 600")
    assert np.all(np.isfinite(a.log_post())) and len(np.unique(xa[:, 0])) == Cn and set(np.unique(xa[:, 5])) == {0.0, 1.0}
    for r in (1e-3, 50.0):                        # small and large radii through the device
        s = gpu_pkg.mcmc.AmwgSampler(params, f, None, {"chains": 64, "seed": 9, "init_radius": r})
        w, t = _expected(O, s, 9, 0, 64, r, lambda xs: xs[3] >= -1 and xs[3] <= 4)
        _bits_equal(_flat_state(s), w, "radius %g" % r)


def test_dispersal_retries_chains_whose_log_post_is_not_finite(gpu_pkg, orc):
    """sigma >= 0 with a U(0, 1) prior and radius 2 around init 0.5: about a third of the first attempts land above 1."""
    O = orc.lib()
    ld = gpu_pkg.ld
    seed, Cn = 11, 4096

    def f(state, data):
        lp = 0
        lp += ld.unif(state.sigma, 0, 1)
        return lp
    s = gpu_pkg.mcmc.AmwgSampler({"sigma": {"type": "real", "lower": 0}}, f, None, {"chains": Cn, "seed": seed, "init_radius": 2})
    got = _flat_state(s)
    want, tries = _expected(O, s, seed, 0, Cn, 2.0, lambda xs: 0 <= xs[0] <= 1)
    assert 0.25 < np.mean(tries > 0) < 0.42 and tries.max() >= 2, (np.mean(tries > 0), tries.max())
    _bits_equal(got, want, "with retries")
    assert np.all(np.isfinite(s.log_post())) and np.all(got <= 1)


def test_dispersal_without_a_finite_point_raises_and_leaves_the_handle_unchanged(gpu_pkg):
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc

    def f(state, data):                            # finite only within 1e-300 of 0: no attempt gets there
        lp = 0
        lp += ld.unif(state.x, -1e-300, 1e-300)
        return lp
    params = {"x": {"type": "real", "init": 0}}
    with pytest.raises(mcmc.JsThrow) as e:
        mcmc.AmwgSampler(params, f, None, {"chains": 64, "seed": 1, "init_radius": 2})
    assert str(e.value) == "options.init_radius: 64 of 64 chains found no starting point with a finite log_post in 100 attempts"
    s = mcmc.AmwgSampler(params, f, None, {"chains": 64, "seed": 1})
    s.burn(3)
    st, lp, info = s.state, s.log_post(), s.info()
    L = gpu_pkg._ffi.lib()
    n = C.c_int64(-1)
    assert L.amwg_disperse_state(s._handle, 2.0, C.byref(n)) != 0 and n.value == 64
    assert "64 of 64 chains" in L.amwg_last_error().decode()
    assert L.amwg_disperse_state(s._handle, float("inf"), C.byref(n)) != 0 and n.value == 0
    _bits_equal({"state": s.state, "lp": s.log_post(), "info": s.info()}, {"state": st, "lp": lp, "info": info})
    with pytest.raises(mcmc.JsThrow) as e:                                  # set_state checks binary values like amwg_create
        b = mcmc.AmwgSampler({"m": {"type": "binary"}}, lambda st_, d: ld.bern(st_.m, 0.5), None, {"chains": 4, "seed": 1})
        b.set_state({"m": [0, 1, 0.5, 1]})
    assert str(e.value) == "amwg_set_state: binary parameters must start at 0 or 1"
    assert b.state["m"].tolist() == [1.0, 1.0, 1.0, 1.0]


def test_dispersal_exposes_a_mode_identical_starts_hide(gpu_pkg):
    """Two well-separated modes at -10 and +10. From one init (almost) every chain stays at +10 and rank R-hat reports convergence
    (1.02 with this seed); from points spread uniformly over (-10, 30) about a quarter of the chains sit in the other mode and R-hat
    says so (1.50: ranks bound how far apart two modes can look, so it stays well below the ratio of the raw variances)."""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc

    def f(state, data):
        return mcmc.Math.log(0.5 * mcmc.Math.exp(ld.norm(state.x, -10, 1)) + 0.5 * mcmc.Math.exp(ld.norm(state.x, 10, 1)))
    params = {"x": {"type": "real", "init": 10}}
    res = {}
    for key, extra in (("same", {}), ("dispersed", {"init_radius": 20})):
        s = mcmc.AmwgSampler(params, f, None, dict({"chains": 1 << 14, "seed": 2}, **extra))
        s.burn(500)
        below = float(np.mean(np.asarray(s.state["x"]) < 0))
        res[key] = (s.sample_summary(200, diagnostics="rank")["x"]["rhat_rank"], below)
        s.close()
    assert res["same"][0] < 1.05 and res["same"][1] < 0.01, res
    assert res["dispersed"][0] > 1.3 and 0.2 < res["dispersed"][1] < 0.3, res


JS_NORM = r"""
var readme_norm_post = function(state, data) {
  var log_post = 0;
  log_post += ld.norm(state.mu, 0, 100);
  log_post += ld.unif(state.sigma, 0, 100);
  for(var i = 0; i < data.length; i++) {
    log_post += ld.norm(data[i], state.mu, state.sigma);
  }
  return log_post;
};
"""


def test_javascript_host_gives_the_python_hosts_bits(gpu_pkg):
    from js_host import JsHost, to_py
    from js_native_inits import InitsDeviceNative
    from oracle.minijs.minijs import to_js
    h = JsHost(native=InitsDeviceNative(gpu_pkg))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.it.set_global("ld", h.load("distributions"))
    h.run(JS_NORM)
    x = config2_data()
    Cn, seed = 512, 4
    mu = 184 + np.random.default_rng(3).normal(0, 2, Cn)
    it = h.it
    it.set_global("the_data", to_js(it, [float(v) for v in x]))
    it.set_global("the_mu", to_js(it, [float(v) for v in mu]))
    with env(AMWG_JIT="1"):
        h.run("""
          var S = new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, readme_norm_post, the_data, {chains: 512, seed: 4});
          S.set_state({mu: the_mu, sigma: 4.5});
          S.burn(60);
          var d1 = S.sample(20);
          S.close();
          var T = new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, readme_norm_post, the_data, {chains: 512, seed: 4, init_radius: 2});
          var t0 = T.state();
          T.burn(60);
          var d2 = T.sample(20);
          T.close();
        """)
        S = gpu_pkg.mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(gpu_pkg.ld), x.tolist(), {"chains": Cn, "seed": seed})
        S.set_state({"mu": mu, "sigma": 4.5})
        S.burn(60)
        p1 = S.sample(20)
        T = gpu_pkg.mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(gpu_pkg.ld), x.tolist(), {"chains": Cn, "seed": seed, "init_radius": 2})
        p0 = T.state
        T.burn(60)
        p2 = T.sample(20)
    for js, py in ((to_py(h.get("d1")), p1), (to_py(h.get("t0")), p0), (to_py(h.get("d2")), p2)):
        for k in ("mu", "sigma"):
            _bits_equal(np.asarray(js[k], np.float64), np.asarray(py[k], np.float64), k)
