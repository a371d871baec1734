"""The run-time specialised sweep (csrc/amwg_jit.cuh) on the GPU, against the interpreter kernels of the same library and against
exact posteriors. The specialised step forms log_post(proposal) - log_post(current) from per-term differences, so a decision can
differ from the interpreter's only when exp(delta) falls within rounding of the accept uniform: with the same Philox streams the
two paths must agree on (nearly) every chain bit for bit, and on every statistic."""
import numpy as np
import pytest

import models
from conftest import PRESIDENTS, config2_data

pytestmark = pytest.mark.gpu


def _pair(pkg, monkeypatch, params, log_post, data, chains, seed=11, **opts):
    """the same model on the interpreter kernels and on the specialised kernel"""
    o = {"chains": chains, "seed": seed}
    o.update(opts)
    monkeypatch.setenv("AMWG_JIT", "0")
    a = pkg.mcmc.AmwgSampler(params, log_post, data, dict(o))
    monkeypatch.setenv("AMWG_JIT", "1")
    b = pkg.mcmc.AmwgSampler(params, log_post, data, dict(o))
    monkeypatch.delenv("AMWG_JIT")
    assert not a.jit_status()[0]
    on, note = b.jit_status()
    assert on, note
    return a, b


def _agreement(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    same = x.view(np.uint64) == y.view(np.uint64)
    return same.reshape(same.shape[0], same.shape[1], -1).all(axis=2).all(axis=0).mean()      # fraction of chains equal in every row / component


def test_headline_model_matches_the_interpreter_and_the_exact_posterior(gpu_pkg, monkeypatch):
    pkg = gpu_pkg
    C = 8192
    x = np.random.default_rng(77).normal(184.5, 4.5, 200)
    a, b = _pair(pkg, monkeypatch, models.PARAMS_NORM, models.norm_post_readme(pkg.ld), x.tolist(), C)
    for s in (a, b):
        s.burn(130)                                  # crosses two adaptation batches
    da, db = a.sample(40), b.sample(40)
    assert _agreement(da["mu"][:, :, None], db["mu"][:, :, None]) > 0.995
    assert _agreement(da["sigma"][:, :, None], db["sigma"][:, :, None]) > 0.995
    # log_post() is evaluated afresh for specialised handles: equal to the interpreter's carried value up to rounding
    la, lb = a.log_post(), b.log_post()
    ok = np.asarray(da["mu"][-1]) == np.asarray(db["mu"][-1])
    assert np.allclose(la[ok], lb[ok], rtol=1e-12, atol=1e-9)
    ia, ib = a.info()["steppers"][0], b.info()["steppers"][0]
    assert np.mean(ia["mu"]["prop_log_scale"] == ib["mu"]["prop_log_scale"]) > 0.99
    assert ia["mu"]["batch_count"] == ib["mu"]["batch_count"]
    # the posterior itself: flat-ish priors, so mu | y ~ t around ybar with scale s/sqrt(n), sigma^2 | y ~ scaled inverse chi-square
    b.burn(800)
    d = b.sample(50)
    n, ybar, s2 = x.size, x.mean(), x.var(ddof=1)
    assert abs(d["mu"].mean() - ybar) < 0.02 and abs(d["mu"].std() - np.sqrt(s2 / n) * np.sqrt((n - 1) / (n - 4))) < 0.02
    # sigma has a flat prior on sigma: sigma^2 | y ~ Inv-chi2(n - 2, .): E[sigma] ~ s * sqrt((n-1)/2) * Gamma((n-3)/2) / Gamma((n-2)/2)
    from math import lgamma, exp, sqrt
    e_sigma = sqrt(s2) * sqrt((n - 1) / 2.0) * exp(lgamma((n - 3) / 2.0) - lgamma((n - 2) / 2.0))
    assert abs(d["sigma"].mean() - e_sigma) < 0.03


def test_config2_size_data_thin_monitor_and_stop_adaptation(gpu_pkg, monkeypatch):
    pkg = gpu_pkg
    a, b = _pair(pkg, monkeypatch, models.PARAMS1, models.norm_post_test(pkg.ld), config2_data().tolist(), 4096, seed=3)
    for s in (a, b):
        s.burn(60)
        s.stop_adaptation()
        s.thin(3)
        s.monitor(["var", "mu"])
    da, db = a.sample(31), b.sample(31)
    assert list(db.keys()) == ["var", "mu"] and db["mu"].shape == (11, 4096)
    assert _agreement(da["mu"][:, :, None], db["mu"][:, :, None]) > 0.995
    assert _agreement(da["var"][:, :, None], db["var"][:, :, None]) > 0.995      # derived quantity: generated code too
    for s in (a, b):
        s.start_adaptation()
        s.thin(1)
        s.monitor(None)
        s.burn(50)
    sa, sb = a.state, b.state
    assert np.mean(sa["sigma"] == sb["sigma"]) > 0.99 and np.allclose(sb["var"], sb["sigma"] ** 2, rtol=0, atol=0)


def _hier_data(J, per, seed=5):
    g = np.repeat(np.arange(J), per)
    mu_true = np.random.default_rng(seed).normal(100, 20, J)
    y = mu_true[g] + np.random.default_rng(seed + 1).normal(0, 5, g.size)
    return {"y": y, "g": g.astype(float)}, mu_true


# unequal groups of >= 8 points on a streamed column (tiles of 1024 points): boundaries mid-tile, a 2500-point group spanning more
# than two tiles, a 9-point group inside one, an odd total (9563)
RAGGED = (9, 2500, 37, 1111, 3001, 14, 777, 1500, 614)


@pytest.mark.parametrize("J,per,chains", [(6, 40, 4096), (12, 1024, 2200), (len(RAGGED), RAGGED, 2200)])
def test_hierarchical_model_resident_and_streamed(gpu_pkg, monkeypatch, J, per, chains):
    """(6 x 40): every column resident in shared memory; (12 x 1024 = 96 KB): the column streams through the TMA tile ring, with a
    chain count that is not a multiple of the CTA size (shadow threads take part in the ring); unequal groups: the sweep splits a
    streamed tile between plates wherever a group ends inside it."""
    pkg = gpu_pkg
    sizes = np.broadcast_to(per, (J,))
    data, mu_true = _hier_data(J, sizes)
    g = data["g"].astype(np.int64)
    P = {"mu": {"type": "real", "dim": [J], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    a, b = _pair(pkg, monkeypatch, P, models.hier_norm_post(pkg.ld), data, chains, seed=21)
    assert ("streamed column" in b.jit_status()[1]) == (g.size * 8 > 64 * 1024)
    for s in (a, b):
        s.burn(55)
    da, db = a.sample(6), b.sample(6)
    # streamed partial sums associate differently from the interpreter's: decisions agree except within rounding of the coin
    assert _agreement(da["mu"], db["mu"]) > 0.98
    assert _agreement(da["sigma"][:, :, None], db["sigma"][:, :, None]) > 0.98
    b.burn(2500)
    d = b.sample(20)
    ybar = np.bincount(g, weights=data["y"]) / sizes
    assert np.allclose(d["mu"].mean(axis=(0, 1)), ybar, atol=6 * 5 / np.sqrt(sizes) / np.sqrt(chains * 20 / 50) + 0.05)
    assert abs(d["sigma"].mean() - np.sqrt(((data["y"] - ybar[g]) ** 2).sum() / (g.size - J))) < 0.05 + 2.0 / np.sqrt(g.size)


def test_expression_means_int_parameter_and_bounds(gpu_pkg, monkeypatch):
    pkg = gpu_pkg
    ld = pkg.ld
    x = np.random.default_rng(9).normal(7.0, 2.0, 300)

    def lp(state, d):
        out = 0
        out += ld.norm(state.a, 0, 10)
        out += ld.unif(state.k, -20, 20)
        out += ld.gamma(state.s, 2, 0.5)
        for i in range(len(d)):
            out += ld.norm(d[i], state.a * 2 + 1, state.s)
        for i in range(100):
            out += ld.norm(d[i], state.k, 3.0)
        state.prec = 1 / (state.s * state.s)
        return out
    P = {"a": {"type": "real"}, "k": {"type": "int", "lower": -20, "upper": 20}, "s": {"type": "real", "lower": 0, "upper": 50}}
    a, b = _pair(pkg, monkeypatch, P, lp, x.tolist(), 4096, seed=2)
    for s in (a, b):
        s.burn(120)
    da, db = a.sample(10), b.sample(10)
    for name in ("a", "k", "s", "prec"):
        assert _agreement(da[name][:, :, None], db[name][:, :, None]) > 0.99, name
    assert np.all(db["k"] == np.round(db["k"])) and np.all(np.abs(db["k"]) <= 20)


# ---- the full-program form (amwg_jit_full_kernel.cuh): the same operations in the same order as the interpreter -> the same bits ----
def _bit_equal(da, db):
    for k in da:
        x, y = np.asarray(da[k], np.float64), np.asarray(db[k], np.float64)
        assert x.shape == y.shape and (x.view(np.uint64) == y.view(np.uint64)).all(), k


@pytest.mark.parametrize("name", ["spike_where", "spike_literal", "complex_literal", "complex_where", "norm_faithful", "norm_faithful_derived",
                                  "multi_bern", "spike_ragged", "spike_bad_point"])
def test_full_program_specialisation_is_bit_identical_to_the_interpreter(gpu_pkg, monkeypatch, name):
    pkg = gpu_pkg
    ld, mcmc = pkg.ld, pkg.mcmc
    rng = np.random.default_rng(5)
    y = (rng.random(100) < 0.7).astype(float).tolist()
    nb = [int(v) for v in rng.integers(5, 30, 12)]
    opts = {}
    if name == "spike_where":
        P, f, d = models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y}
    elif name == "spike_ragged":                     # 77 points: two full mask words and a 13-bit tail
        P, f, d = models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y[:77]}
    elif name == "spike_bad_point":                  # a point that is neither 0 nor 1: ld.bern gives -Infinity, the sum stays sequential
        P, f, d = models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": y[:40] + [2.0] + y[41:]}
    elif name == "spike_literal":
        P, f, d = models.PARAMS_SPIKE, models.spike_bern_literal(ld), {"x": y}
    elif name == "complex_literal":
        P, f, d = models.PARAMS_COMPLEX, models.complex_model_post_literal(ld), nb
    elif name == "complex_where":
        P, f, d = models.PARAMS_COMPLEX, models.complex_model_post(ld, mcmc), nb
    elif name == "norm_faithful":
        P, f, d, opts = models.PARAMS_NORM, models.norm_post_readme(ld), rng.normal(184.5, 4.5, 64).tolist(), {"faithful": True}
    elif name == "norm_faithful_derived":
        def f(state, data):
            lp = 0
            lp += ld.norm(state.mu, 0, 100)
            lp += ld.unif(state.sigma, 0, 100)
            for i in range(len(data)):
                lp += ld.norm(data[i], state.mu, state.sigma)
            state.cv = state.sigma / state.mu
            return lp
        P, d, opts = {"mu": {"type": "real", "init": 180}, "sigma": {"type": "real", "lower": 0, "init": 5}}, rng.normal(184.5, 4.5, 64).tolist(), {"faithful": True}
    else:
        P = {"x": {"type": "binary", "dim": [2, 2]}}
        f, d = models.multi_bern_dens(mcmc), None
    a, b = _pair(pkg, monkeypatch, P, f, d, 4096 + 37, **opts)          # a ragged last CTA
    assert "full-program" in b.jit_status()[1]
    for s in (a, b):
        s.burn(120)                                   # crosses two adaptation batches
    _bit_equal(a.sample(25), b.sample(25))
    _bit_equal({"lp": a.log_post()}, {"lp": b.log_post()})
    for s in (a, b):
        s.burn(7)
    _bit_equal(a.sample(6), b.sample(6))
    ia, ib = a.info()["steppers"][0], b.info()["steppers"][0]
    for k in ia:
        if isinstance(ia[k], dict) and "prop_log_scale" in ia[k]:
            assert np.array_equal(np.asarray(ia[k]["prop_log_scale"]), np.asarray(ib[k]["prop_log_scale"])), k
