"""PSIS-LOO and WAIC in sample_summary(..., loo=...) on the GPU: the device's pointwise log-likelihood against the oracle's ld.* at
every kept draw, bit for bit; the config-2 model's "loo" against the numpy restatement (tests/loo_ref.py) on the ll of an identically
seeded twin's sample() draws; every other key and the chains' state unchanged by the option; and a conjugate Normal model against
its closed-form leave-one-out predictive density."""
import math

import numpy as np
import pytest
import torch

import loo_ref
import models
from conftest import config2_data

pytestmark = pytest.mark.gpu


def _pointwise(s, log_lik, points, n):
    """-> (block [rows, entries, chains] of every parameter's draws, ll [rows, points, chains]) of the next n sweeps, formed by the
    library's pointwise kernel on the sampled block (entries = the components in order)."""
    import ctypes as C
    from bayes_js_b200 import _ffi
    from bayes_js_b200.summary import CudaPointwise
    from bayes_js_b200.tracer import trace_log_lik
    entries = list(range(s.n_comp))
    block = torch.empty((n, len(entries), s.local_chains), dtype=torch.float64, device="cuda:%d" % s.device)
    mon = np.asarray(entries, dtype=np.int32)
    torch.cuda.synchronize()
    _ffi.check(_ffi.lib().amwg_sample_device(s._handle, n, 1, mon.ctypes.data_as(C.POINTER(C.c_int32)), len(entries), block.data_ptr()))
    lik = trace_log_lik(log_lik, s.params, s._offsets, s.data, points)
    prog = lik.lower({name: s._offsets[name] for name in lik.reads})
    ll = CudaPointwise(s._handle, prog, block, s.device).chunk(0, points)
    return block.cpu().numpy(), ll.cpu().numpy()


def test_device_ll_equals_the_oracle_bit_for_bit(gpu_pkg, orc):
    mcmc, ld, Math = gpu_pkg.mcmc, gpu_pkg.ld, gpu_pkg.mcmc.Math
    O = orc.lib()
    rng = np.random.default_rng(23)
    N, J = 10, 3
    d = {"y": rng.normal(1, 2, N).round(3).tolist(), "b": rng.integers(0, 2, N).astype(float).tolist(),
         "c": rng.poisson(3, N).astype(float).tolist(), "g": np.sort(rng.integers(0, J, N)).astype(float).tolist(),
         "X": rng.normal(0, 0.5, (N, 2)).round(3).tolist(), "s": [1.7, 2.3]}
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0, "init": 1}, "p": {"type": "real", "lower": 0, "upper": 1, "init": 0.5},
              "a": {"type": "real", "dim": [J]}, "beta": {"type": "real", "dim": [2]}}

    def log_post(st, dd):
        lp = ld.norm(st.mu, 0, 10) + ld.unif(st.sigma, 0, 10) + ld.beta(st.p, 2, 2)
        for j in range(J):
            lp += ld.norm(st.a[j], 0, 5)
        lp += ld.norm(st.beta[0], 0, 1) + ld.norm(st.beta[1], 0, 1)
        for i in range(N):
            lp += ld.norm(dd.y[i], st.a[dd.g[i]], st.sigma) + ld.bern(dd.b[i], st.p)
            lp += ld.pois(dd.c[i], Math.exp(dd.X[i][0] * st.beta[0] + dd.X[i][1] * st.beta[1]))
        return lp
    s = mcmc.AmwgSampler(params, log_post, d, {"chains": 200, "seed": 5})
    s.burn(300)
    cases = {
        "norm": (lambda st, dd, i: ld.norm(dd.y[i], st.mu, st.sigma), lambda x, i: O.orc_ld_norm(d["y"][i], x[0], x[1])),
        "bern": (lambda st, dd, i: ld.bern(dd.b[i], st.p), lambda x, i: O.orc_ld_bern(d["b"][i], x[2])),
        "grouped": (lambda st, dd, i: ld.norm(dd.y[i], st.a[dd.g[i]], st.sigma), lambda x, i: O.orc_ld_norm(d["y"][i], x[3 + int(d["g"][i])], x[1])),
        "poisson": (lambda st, dd, i: ld.pois(dd.c[i], Math.exp(dd.X[i][0] * st.beta[0] + dd.X[i][1] * st.beta[1])),
                    lambda x, i: O.orc_ld_pois(d["c"][i], O.orc_exp(d["X"][i][0] * x[6] + d["X"][i][1] * x[7]))),
        "composed": (lambda st, dd, i: ld.norm(dd.y[i], st.mu, st.sigma) + ld.bern(dd.b[i], st.p) - Math.log(st.sigma * 2),
                     lambda x, i: (O.orc_ld_norm(d["y"][i], x[0], x[1]) + O.orc_ld_bern(d["b"][i], x[2])) - O.orc_log(x[1] * 2)),
        # a data element at a fixed index: the folded constants read it (the fold programs hold DATA)
        "fixed_index": (lambda st, dd, i: ld.norm(dd.y[i], st.mu, dd.s[0]), lambda x, i: O.orc_ld_norm(d["y"][i], x[0], d["s"][0])),
    }
    for name, (f, want) in cases.items():
        block, ll = _pointwise(s, f, N, 3)
        rows, _, chains = block.shape
        ref = np.array([[[want(block[r, :, c], i) for c in range(chains)] for i in range(N)] for r in range(rows)])
        assert np.array_equal(ll.view(np.int64), ref.view(np.int64)), name


def _norm_ll_oracle(O, y, mu, sd):
    """ld.norm(y_i, mu, sd) in the operations distributions.js uses (the body's expansion), with the oracle's log: ll [S, N]."""
    k1 = np.array([(-0.5 * O.orc_log(2 * math.pi)) - O.orc_log(float(v)) for v in sd])
    k2 = (2 * sd) * sd
    dy = np.asarray(y, dtype=np.float64)[None, :] - mu[:, None]
    return k1[:, None] - (dy * dy) / k2[:, None]


def test_config2_loo_equals_the_restatement(gpu_pkg, orc):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    O = orc.lib()
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    a = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 31})
    b = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 31})
    a.burn(1500); b.burn(1500)
    raw = a.sample(8)
    out = b.sample_summary(8, loo={"log_lik": lambda st, d, i: ld.norm(d[i], st.mu, st.sigma), "points": len(data)})["loo"]
    ll = _norm_ll_oracle(O, data, raw["mu"].reshape(-1), raw["sigma"].reshape(-1))
    ref = loo_ref.loo(ll)
    for key, want in ref["pointwise"].items():
        got = out["pointwise"][key]
        fin = np.isfinite(want)
        assert np.array_equal(fin, np.isfinite(got)), key
        assert np.all(np.abs(got[fin] - want[fin]) <= 1e-10 * np.maximum(1.0, np.abs(ref["pointwise"]["lppd"][fin]))), key
    for key in ("elpd_loo", "se_elpd_loo", "p_loo", "looic", "elpd_waic", "se_elpd_waic", "p_waic", "waic"):
        assert abs(out[key] - ref[key]) <= 1e-10 * max(1.0, abs(ref[key])), key
    assert out["n_high_k"] == ref["n_high_k"] and out["n_draws"] == 8 * 4096 and out["points"] == 1024


def _same(x, y):
    """the same keys and, for numbers, the same bytes"""
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    a, b = np.asarray(x), np.asarray(y)
    if a.dtype.kind in "fiub":
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


@pytest.mark.parametrize("monitor", [None, ["sigma"]])
def test_other_keys_and_the_chains_keep_their_bits(gpu_pkg, monitor):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()[:200].tolist()
    opts = {"chains": 1000, "seed": 9}
    if monitor:
        opts["monitor"] = monitor                                 # mu is read by log_lik but not monitored: sampled alongside
    a = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, dict(opts))
    b = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, dict(opts))
    a.burn(500); b.burn(500)
    kw = dict(diagnostics=True, histogram=16, covariance=True)
    plain = a.sample_summary(20, **kw)
    with_loo = b.sample_summary(20, loo={"log_lik": lambda st, d, i: ld.norm(d[i], st.mu, st.sigma), "points": 200}, **kw)
    assert set(with_loo) == set(plain) | {"loo"}
    for key in plain:
        assert _same(plain[key], with_loo[key]), key
    assert _same(a.state, b.state) and _same(a.log_post(), b.log_post())
    assert np.isfinite(with_loo["loo"]["elpd_loo"])


def test_loo_does_not_depend_on_where_the_block_holds_the_parameters(gpu_pkg):
    """monitor None (block [mu, sigma]), ["sigma"] (mu appended: [sigma, mu]) and ["sigma", "mu"]: the body reads its parameters
    from wherever the block holds them, so the ll bits, the summation order and the whole "loo" dict are the same"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()[:300].tolist()
    loo = {"log_lik": lambda st, d, i: ld.norm(d[i], st.mu, st.sigma), "points": 300}
    outs = []
    for monitor in (None, ["sigma"], ["sigma", "mu"]):
        opts = {"chains": 2000, "seed": 13}
        if monitor:
            opts["monitor"] = monitor
        s = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, opts)
        s.burn(400)
        outs.append(s.sample_summary(6, loo=loo)["loo"])
    assert np.isfinite(outs[0]["elpd_loo"])
    for other in outs[1:]:
        assert _same(outs[0], other)


def test_conjugate_normal_against_the_exact_leave_one_out_density(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    y = np.random.default_rng(41).normal(2.0, 1.0, 20)
    tau0 = 10.0

    def log_post(st, d):
        lp = ld.norm(st.mu, 0, tau0)
        for i in range(len(d)):
            lp += ld.norm(d[i], st.mu, 1.0)
        return lp
    s = mcmc.AmwgSampler({"mu": {"type": "real"}}, log_post, y.tolist(), {"chains": 16384, "seed": 3})
    twin = mcmc.AmwgSampler({"mu": {"type": "real"}}, log_post, y.tolist(), {"chains": 16384, "seed": 3})
    s.burn(2000); twin.burn(2000)
    out = s.sample_summary(1, loo={"log_lik": lambda st, d, i: ld.norm(d[i], st.mu, 1.0), "points": len(y)})["loo"]
    mu = twin.sample(1)["mu"].reshape(-1)                        # the same draws: one per chain, the chains independent
    exact = np.empty(len(y))
    for i in range(len(y)):
        rest = np.delete(y, i)
        prec = 1 / tau0 ** 2 + len(rest)
        m = rest.sum() / prec
        v = 1.0 + 1 / prec
        exact[i] = -0.5 * np.log(2 * np.pi * v) - (y[i] - m) ** 2 / (2 * v)
    # Monte Carlo standard error of each point's estimate -log mean_s r_s, r_s = 1 / p(y_i | mu_s) the importance ratios, by the
    # delta method: sd(r) / (mean(r) sqrt(S)); the points share the draws, so the total's bound adds them
    r = np.exp(0.5 * np.log(2 * np.pi) + (y[None, :] - mu[:, None]) ** 2 / 2)
    se = r.std(axis=0) / (r.mean(axis=0) * np.sqrt(len(mu)))
    err = out["pointwise"]["elpd_loo"] - exact
    assert np.all(np.abs(err) < 5 * se), (err, se)
    assert abs(out["elpd_loo"] - exact.sum()) < 5 * se.sum()
    assert np.all(out["pointwise"]["pareto_k"] < out["pareto_k_threshold"]) and out["n_high_k"] == 0
