"""Posterior predictive checks in sample_summary(..., ppc=...) on the GPU: the device's replicated data against the independent
restatement of tests/ppc_ref.py at every kept draw, bit for bit, for every family; the config-2 model's whole "ppc" dict against the
restatement on an identically seeded twin's draws; every other key and the chains' state unchanged by the option, alone and with
loo=; the dict independent of where the block holds the parameters; calibration on a conjugate Normal model; a misfit detected;
10^6 device draws per sampler regime against scipy.stats and 2000 of them bit for bit; an out-of-domain body, NaN throughout; the
dict byte-equal over chunks of points; and the threshold counts on an adversarial block against numpy."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import stats as st

import models
import ppc_ref
from conftest import config2_data
from test_summary_ppc_host import REGIMES, distribution_p

pytestmark = pytest.mark.gpu


def _sample_block(s, n):
    """-> the device block [n, entries, chains] of every component's draws over the next n sweeps (entries = the components in order)"""
    from bayes_js_b200 import _ffi
    entries = list(range(s.n_comp))
    block = torch.empty((n, len(entries), s.local_chains), dtype=torch.float64, device="cuda:%d" % s.device)
    mon = np.asarray(entries, dtype=np.int32)
    torch.cuda.synchronize()
    _ffi.check(_ffi.lib().amwg_sample_device(s._handle, n, 1, mon.ctypes.data_as(C.POINTER(C.c_int32)), len(entries), block.data_ptr()))
    return block


def _ppc_source(s, log_lik, points, block):
    """-> (family, observed y, a function giving a fresh CudaPpc over `block`): the library's replicated data of the traced body"""
    from bayes_js_b200.summary import PPC_FAMILIES, CudaPpc
    from bayes_js_b200.tracer import trace_log_lik
    lik = trace_log_lik(log_lik, s.params, s._offsets, s.data, points, what="ppc")
    fam, y, args = lik.observed_call(points)
    prog, offs = lik.lower_exprs(args, {name: s._offsets[name] for name in lik.reads})
    return fam, y, lambda: CudaPpc(s._handle, prog, offs, PPC_FAMILIES.index(fam), block, points)


def _replicated(s, log_lik, points, n):
    """-> (block [rows, entries, chains] of every component's draws, y_rep [rows, points, chains], T [rows, 4, chains]) of the next
    n sweeps, formed by the library's kernel on the sampled block (entries = the components in order)."""
    block = _sample_block(s, n)
    src = _ppc_source(s, log_lik, points, block)[2]()
    yrep = src.chunk(0, points).cpu().numpy()
    return block.cpu().numpy(), yrep, src.stats().cpu().numpy()


def test_device_draws_equal_the_restatement_for_every_family(gpu_pkg, orc):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    O = orc.lib()
    N = 5
    d = {"y": [0.5, 1.0, 2.0, 3.0, 4.0], "n": [3.0, 40.0, 200.0, 1000.0, 7.0]}
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0, "init": 1}, "p": {"type": "real", "lower": 0, "upper": 1, "init": 0.5}}

    def log_post(s, dd):
        return ld.norm(s.mu, 0, 1) + ld.gamma(s.sigma, 3, 3) + ld.beta(s.p, 2, 2)
    s = mcmc.AmwgSampler(params, log_post, d, {"chains": 256, "seed": 31, "first_chain": 1000})
    s.burn(200)
    # (body, the parameters of point i from (mu, sigma, p) in the same fp64 operations)
    cases = {
        "norm": (lambda t, dd, i: ld.norm(dd.y[i], t.mu, t.sigma), lambda m, sg, p, i: (m, sg)),
        "lnorm": (lambda t, dd, i: ld.lnorm(dd.y[i], t.mu, t.sigma), lambda m, sg, p, i: (m, sg)),
        "cauchy": (lambda t, dd, i: ld.cauchy(dd.y[i], t.mu, t.sigma), lambda m, sg, p, i: (m, sg)),
        "laplace": (lambda t, dd, i: ld.dexp(dd.y[i], t.mu, t.sigma), lambda m, sg, p, i: (m, sg)),
        "logis": (lambda t, dd, i: ld.logis(dd.y[i], t.mu, t.sigma), lambda m, sg, p, i: (m, sg)),
        "exp": (lambda t, dd, i: ld.exp(dd.y[i], t.sigma), lambda m, sg, p, i: (sg,)),
        "weibull": (lambda t, dd, i: ld.weibull(dd.y[i], t.sigma + 0.3, t.sigma), lambda m, sg, p, i: (sg + 0.3, sg)),
        "pareto": (lambda t, dd, i: ld.pareto(dd.y[i], t.sigma, t.sigma + 1), lambda m, sg, p, i: (sg, sg + 1.0)),
        "unif": (lambda t, dd, i: ld.unif(dd.y[i], t.mu, t.mu + t.sigma), lambda m, sg, p, i: (m, m + sg)),
        "gamma": (lambda t, dd, i: ld.gamma(dd.y[i], t.sigma, t.p), lambda m, sg, p, i: (sg, p)),
        "invgamma": (lambda t, dd, i: ld.invgamma(dd.y[i], t.sigma + 2, t.sigma), lambda m, sg, p, i: (sg + 2.0, sg)),
        "beta": (lambda t, dd, i: ld.beta(dd.y[i], t.sigma, t.p * 3), lambda m, sg, p, i: (sg, p * 3.0)),
        "t": (lambda t, dd, i: ld.t(dd.y[i], t.mu, t.sigma, t.sigma * 5), lambda m, sg, p, i: (m, sg, sg * 5.0)),
        "bern": (lambda t, dd, i: ld.bern(dd.y[i], t.p), lambda m, sg, p, i: (p,)),
        "pois": (lambda t, dd, i: ld.pois(dd.y[i], t.sigma * dd.n[i]), lambda m, sg, p, i: (sg * d["n"][i],)),
        "binom": (lambda t, dd, i: ld.binom(dd.y[i], dd.n[i], t.p), lambda m, sg, p, i: (d["n"][i], p)),
        "nbinom": (lambda t, dd, i: ld.nbinom(dd.y[i], t.sigma * 3, t.p), lambda m, sg, p, i: (sg * 3.0, p)),
    }
    rows = 4
    for fam, (f, args) in cases.items():
        block, yrep, T = _replicated(s, f, N, rows)
        for r in range(rows):
            for c in range(0, 256, 5):
                m, sg, p = block[r, :, c]
                for i in range(N):
                    want, _ = ppc_ref.draw_at(O, fam, args(m, sg, p, i), 31, 1000 + c, r, N, i)
                    assert np.float64(yrep[r, i, c]).tobytes() == np.float64(want).tobytes(), (fam, r, c, i, yrep[r, i, c], want)
        assert np.all(np.isfinite(yrep)), fam
        flat = np.moveaxis(yrep, 1, 2).reshape(-1, N)
        assert np.array_equal(np.moveaxis(T, 1, 2).reshape(-1, 4), ppc_ref.dataset_stats_many(flat), equal_nan=True), fam


def _same(x, y):
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    a, b = np.asarray(x), np.asarray(y)
    if a.dtype.kind in "fiub":
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


def test_config2_dict_equals_the_restatement(gpu_pkg, orc):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    O = orc.lib()
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()
    probs = (0.05, 0.5, 0.95)
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    a = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data.tolist(), {"chains": 4096, "seed": 17})
    b = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data.tolist(), {"chains": 4096, "seed": 17})
    a.burn(300); b.burn(300)
    out = a.sample_summary(8, probs=probs, ppc={"log_lik": f, "points": 1024})["ppc"]
    block, yrep, T = _replicated(b, f, 1024, 8)
    rng = np.random.default_rng(5)
    for _ in range(3000):                                          # the device draws against the restatement
        r, c, i = int(rng.integers(8)), int(rng.integers(4096)), int(rng.integers(1024))
        want, _ = ppc_ref.draw_at(O, "norm", (block[r, 0, c], block[r, 1, c]), 17, c, r, 1024, i)
        assert np.float64(yrep[r, i, c]).tobytes() == np.float64(want).tobytes()
    flat = np.moveaxis(yrep, 1, 2).reshape(-1, 1024)
    ref = ppc_ref.ppc(flat, data, probs)
    assert np.array_equal(np.moveaxis(T, 1, 2).reshape(-1, 4), ppc_ref.dataset_stats_many(flat), equal_nan=True)
    assert out["family"] == "norm" and out["points"] == 1024 and out["n_draws"] == 8 * 4096
    for key in ("n_below", "n_equal", "n_nan", "pit"):
        assert np.array_equal(out["pointwise"][key], ref["pointwise"][key]), key
    for key in ("mean", "sd"):
        assert np.allclose(out["pointwise"][key], ref["pointwise"][key], rtol=1e-12), key
    for name in ppc_ref.STATS:
        got, want = out["stats"][name], ref["stats"][name]
        assert got["observed"] == want["observed"], name
        for key in ("n_greater", "n_equal", "n_nan", "p_value"):
            assert got[key] == want[key], (name, key)
        assert np.isclose(got["mean"], want["mean"], rtol=1e-12) and np.isclose(got["sd"], want["sd"], rtol=1e-10), name
        assert np.array_equal(got["quantiles"], want["quantiles"]), name


def test_other_keys_and_the_chains_keep_their_bits(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()[:200].tolist()
    f = lambda st_, d, i: ld.norm(d[i], st_.mu, st_.sigma)
    samplers = [mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 1000, "seed": 9}) for _ in range(4)]
    for s in samplers:
        s.burn(500)
    kw = dict(diagnostics=True, histogram=16, covariance=True)
    plain = samplers[0].sample_summary(20, **kw)
    with_ppc = samplers[1].sample_summary(20, ppc={"log_lik": f, "points": 200}, **kw)
    with_loo = samplers[2].sample_summary(20, loo={"log_lik": f, "points": 200}, **kw)
    both = samplers[3].sample_summary(20, loo={"log_lik": f, "points": 200}, ppc={"log_lik": f, "points": 200}, **kw)
    assert set(with_ppc) == set(plain) | {"ppc"} and set(both) == set(plain) | {"ppc", "loo"}
    for key in plain:
        assert _same(plain[key], with_ppc[key]) and _same(plain[key], both[key]), key
    assert _same(with_loo["loo"], both["loo"]) and _same(with_ppc["ppc"], both["ppc"])
    for s in samplers[1:]:
        assert _same(samplers[0].state, s.state) and _same(samplers[0].log_post(), s.log_post())
    outs = []
    for monitor in (None, ["sigma"], ["sigma", "mu"]):
        opts = {"chains": 1000, "seed": 13}
        if monitor:
            opts["monitor"] = monitor
        s = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, opts)
        s.burn(300)
        outs.append(s.sample_summary(3, ppc={"log_lik": f, "points": 200})["ppc"])
    for other in outs[1:]:
        assert _same(outs[0], other)


def test_conjugate_normal_calibration(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    sigma, tau0, m0 = 1.5, 10.0, 0.0
    y = np.random.default_rng(43).normal(2.0, sigma, 300)

    def log_post(t, d):
        lp = ld.norm(t.mu, m0, tau0)
        for i in range(len(d)):
            lp += ld.norm(d[i], t.mu, sigma)
        return lp
    s = mcmc.AmwgSampler({"mu": {"type": "real"}}, log_post, y.tolist(), {"chains": 65536, "seed": 4})
    s.burn(1500)
    out = s.sample_summary(1, ppc={"log_lik": lambda t, d, i: ld.norm(d[i], t.mu, sigma), "points": len(y)})["ppc"]
    prec = 1 / tau0 ** 2 + len(y) / sigma ** 2
    mun, taun2 = (m0 / tau0 ** 2 + y.sum() / sigma ** 2) / prec, 1 / prec
    sd = np.sqrt(sigma ** 2 + taun2)
    S = out["n_draws"]
    assert np.all(np.abs(out["pointwise"]["mean"] - mun) < 5 * sd / np.sqrt(S)), out["pointwise"]["mean"] - mun
    assert np.all(np.abs(out["pointwise"]["sd"] - sd) < 5 * sd / np.sqrt(2 * S)), out["pointwise"]["sd"] - sd
    assert st.kstest(out["pointwise"]["pit"], "uniform").pvalue > 1e-3
    assert np.all(out["pointwise"]["n_nan"] == 0) and all(0.001 < out["stats"][k]["p_value"] < 0.999 for k in ("mean", "sd"))


def test_a_normal_fitted_to_heavy_tailed_data_fails_the_max_check(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    y = np.random.default_rng(47).standard_t(1.5, 500)
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    s = mcmc.AmwgSampler(params, models.norm_post_readme(ld), y.tolist(), {"chains": 4096, "seed": 8})
    s.burn(1500)
    out = s.sample_summary(2, ppc={"log_lik": lambda t, d, i: ld.norm(d[i], t.mu, t.sigma), "points": len(y)})["ppc"]
    assert out["stats"]["max"]["p_value"] < 0.01, out["stats"]["max"]


def test_device_draws_follow_the_distribution(gpu_pkg, orc):
    """10^6 device draws per regime against scipy, and 2000 of them bit for bit against the restatement"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    O = orc.lib()
    N = 1000
    s = mcmc.AmwgSampler({"mu": {"type": "real"}}, lambda t, d: ld.norm(t.mu, 0, 1), {"y": [0.0] * N}, {"chains": 1000, "seed": 2})
    s.burn(10)
    fn = {"dexp": "laplace"}
    rng = np.random.default_rng(3)
    for fam, p in REGIMES:
        call = getattr(ld, fam)
        f = (lambda call, p: lambda t, d, i: call(d.y[i], *p))(call, p)
        _, yrep, _ = _replicated(s, f, N, 1)
        for _ in range(2000):
            c, i = int(rng.integers(1000)), int(rng.integers(N))
            want, _ = ppc_ref.draw_at(O, fn.get(fam, fam), tuple(float(v) for v in p), 2, c, 0, N, i)
            assert np.float64(yrep[0, i, c]).tobytes() == np.float64(want).tobytes(), (fam, p, c, i, yrep[0, i, c], want)
        x = yrep.ravel()
        assert x.size == 10 ** 6 and np.all(np.isfinite(x)), fam
        assert distribution_p(x, fn.get(fam, fam), p) > 1e-3, (fam, p)


def test_out_of_domain_parameters_give_nan_everywhere(gpu_pkg):
    """ld.norm with sd = -1: every y_rep is NaN, so no draw is below, equal to or above y_i (pit 0), every dataset statistic of a
    draw is NaN, no draw counts as >= T(y) (p-values 0) and the summaries of T(y_rep) are NaN"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    y = [0.5, -1.0, 2.0, 3.25, 0.0]
    mk = lambda: mcmc.AmwgSampler({"mu": {"type": "real"}}, lambda t, d: ld.norm(t.mu, 0, 1), {"y": y}, {"chains": 300, "seed": 6})
    a, b = mk(), mk()
    a.burn(20); b.burn(20)
    f = lambda t, d, i: ld.norm(d.y[i], 0, -1)
    out = a.sample_summary(4, probs=(0.1, 0.5), ppc={"log_lik": f, "points": len(y)})["ppc"]
    _, yrep, T = _replicated(b, f, len(y), 4)
    assert np.all(np.isnan(yrep)) and np.all(np.isnan(T))
    S = 4 * 300
    pw = out["pointwise"]
    assert out["n_draws"] == S and np.all(pw["n_nan"] == S) and np.all(pw["n_below"] == 0) and np.all(pw["n_equal"] == 0)
    assert np.all(pw["pit"] == 0) and np.all(np.isnan(pw["mean"])) and np.all(np.isnan(pw["sd"]))
    obs = ppc_ref.dataset_stats(y)
    for k, name in enumerate(ppc_ref.STATS):
        st_ = out["stats"][name]
        assert st_["observed"] == obs[k] and st_["n_nan"] == S and st_["n_greater"] == 0 and st_["n_equal"] == 0, name
        assert st_["p_value"] == 0 and np.isnan(st_["mean"]) and np.isnan(st_["sd"]) and np.all(np.isnan(st_["quantiles"])), name


def test_chunks_of_points_give_the_same_bytes(gpu_pkg):
    """ppc_block over chunks of 1, 7 and all N points: the draws' Welford records carry across chunks on the device, so the whole
    dict keeps its bytes"""
    from bayes_js_b200.summary import CudaBlockReducer, ppc_block
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()[:60]
    s = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data.tolist(), {"chains": 3000, "seed": 19})
    s.burn(300)
    rows, N = 5, len(data)
    block = _sample_block(s, rows)
    fam, y, fresh = _ppc_source(s, lambda t, d, i: ld.norm(d[i], t.mu, t.sigma), N, block)
    outs = [ppc_block(CudaBlockReducer(0), fresh(), rows, 3000, N, fam, y, (0.05, 0.5, 0.95), chunk, False) for chunk in (N, 1, 7)]
    assert np.isfinite(outs[0]["stats"]["sd"]["mean"])
    for other in outs[1:]:
        assert _same(outs[0], other)


def test_threshold_counts_on_an_adversarial_block(gpu_pkg):
    """amwg_summary_threshold_counts over draws and thresholds from both zeros, subnormals, infinities and NaN of both signs, at
    (rows, chains) of (1, 1), (7, 255) and (3, 1184 x 256 + 77), and at 65535 entries: numpy's <, ==, > and isnan, count for count"""
    from bayes_js_b200.summary import CudaBlockReducer
    from test_gpu_summary_hist import _pool
    red = CudaBlockReducer(0)
    rng = np.random.default_rng(73)
    pool = np.concatenate([_pool(-1.0, 1.0, (7, 64), rng), [-np.nan, np.copysign(np.nan, -1.0)]])
    assert np.signbit(pool[np.isnan(pool)]).any() and not np.signbit(pool[np.isnan(pool)]).all()

    def check(x, thr):
        got = red.threshold_counts(torch.from_numpy(x).to("cuda:0"), thr).cpu().numpy()
        t = thr[None, :, None]
        want = np.stack([(x < t).sum(axis=(0, 2)), (x == t).sum(axis=(0, 2)), (x > t).sum(axis=(0, 2)), np.isnan(x).sum(axis=(0, 2))], axis=1)
        assert got.dtype == np.int64 and np.array_equal(got, want), (x.shape, np.flatnonzero((got != want).any(axis=1))[:5])

    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 5e-324, -1e-310])
    for rows, chains in ((1, 1), (7, 255), (3, 1184 * 256 + 77)):
        thr = np.concatenate([special, rng.choice(pool, 9)])
        check(rng.choice(pool, size=(rows, len(thr), chains)), thr)
    thr = rng.choice(np.concatenate([pool, special]), 65535)
    check(rng.choice(pool, size=(1, 65535, 3)), thr)
