"""Tempered ladders on the GPU (options.temperatures, DESIGN.md §2 "Tempered ladders").

The device is held to tests/temper_ref.py (the oracle's steppers with the rung's beta, and the swap round) chain for chain on the
interpreter sweeps; its results must not depend on how the chains are split over handles; and the ladder must sample a bimodal
posterior that a single chain per start cannot: the cold chains follow the exact mixture, every rung its tempered law."""
import ctypes as C
import math
import os
from contextlib import contextmanager

import numpy as np
import pytest
from scipy import stats

import temper_ref
from conftest import config2_data

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


def _bits(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    return a.view(np.uint64)


# ---- a model with a real, an int, a vector and a binary parameter and a derived quantity ------------------------------------------
PARAMS_MIX = {"mu": {"type": "real"}, "s": {"type": "real", "lower": 0, "init": 1.5}, "k": {"type": "int", "lower": -20, "upper": 20},
              "v": {"type": "real", "dim": [3]}, "m": {"type": "binary"}}
Y = [0.3, 1.7, -0.4, 2.2, 0.9]


def _lp_mix(ld):
    def lp(st, d):
        l = 0
        l += ld.norm(st.mu, 0, 5)
        l += ld.gamma(st.s, 2, 1)
        l += ld.norm(st.k, 2, 3)
        l += ld.bern(st.m, 0.3)
        for j in range(3):
            l += ld.norm(st.v[j], st.mu, st.s)
        for i in range(len(d)):
            l += ld.norm(d[i], st.mu + 0.5 * st.m, st.s)
        st.var = st.s * st.s
        return l
    return lp


def _f_mix(O):
    def f(x):
        mu, s, k, v, m = x[0], x[1], x[2], x[3:6], x[6]
        lp = 0.0
        lp += O.orc_ld_norm(mu, 0, 5)
        lp += O.orc_ld_gamma(s, 2, 1)
        lp += O.orc_ld_norm(k, 2, 3)
        lp += O.orc_ld_bern(m, 0.3)
        for j in range(3):
            lp += O.orc_ld_norm(v[j], mu, s)
        for yi in Y:
            lp += O.orc_ld_norm(yi, mu + 0.5 * m, s)
        x[7] = s * s
        return lp
    return f


TEMPS = [1.0, 1.7, 3.1, 6.5]


@pytest.mark.parametrize("path", ["full_program", "term_cache"])
def test_tempered_sweeps_equal_the_reference_chain_for_chain(gpu_pkg, orc, path):
    """K = 4, 6 ladders, first_chain 8: every chain's state, prop_log_scale, acceptance counts, the cold draws (thin 3, monitor with
    the derived quantity), the rounds and the per-pair swap counts equal the reference ladder's, bit for bit."""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    ladders, K, seed, first = 6, len(TEMPS), 91, 8
    envs = {"AMWG_TERM_CACHE": "0"} if path == "full_program" else {}
    with env(**envs):
        s = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": ladders * K, "seed": seed, "first_chain": first, "faithful": True,
                                                          "temperatures": TEMPS, "params": {"mu": {"batch_size": 7}}})
        s.burn(23)
        s.thin(3)
        s.monitor(["mu", "v", "var", "k", "m"])
        got = s.sample(31)
        info = s.info()
        state = s.state
    assert s.jit_status() == (False, "tempered ladder (options.temperatures): interpreter kernels")
    if path == "term_cache":
        assert s._program.n_terms > 0
    ref = temper_ref.RefLadder(orc, _f_mix(orc.lib()), PARAMS_MIX, seed, [1.0 / t for t in TEMPS], ladders, first_chain=first, n_derived=1,
                               comp_options={"mu": {"batch_size": 7}})
    ref.burn(23)
    draws = ref.sample(31, [0, 3, 4, 5, 7, 2, 6], thin=3)                 # [rows, entries, ladders]
    assert got["mu"].shape == (11, ladders) and got["v"].shape == (11, ladders, 3)
    assert np.array_equal(_bits(got["mu"]), _bits(draws[:, 0]))
    assert np.array_equal(_bits(got["v"]), _bits(np.moveaxis(draws[:, 1:4], 1, 2)))
    assert np.array_equal(_bits(got["var"]), _bits(draws[:, 4]))
    assert np.array_equal(_bits(got["k"]), _bits(draws[:, 5])) and np.array_equal(_bits(got["m"]), _bits(draws[:, 6]))
    X = ref.states()                                                          # [chains, D + 1]
    for j, name in enumerate(["mu", "s", "k"]):
        assert np.array_equal(_bits(state[name]), _bits(X[:, j])), name
    assert np.array_equal(_bits(state["v"]), _bits(X[:, 3:6])) and np.array_equal(_bits(state["m"]), _bits(X[:, 6]))
    assert np.array_equal(_bits(state["var"]), _bits(X[:, 7]))
    lp = s.log_post()
    assert np.array_equal(_bits(lp), _bits([ch.log_post() for ch in ref.chains]))
    assert np.array_equal(_rng_n(s.checkpoint(), 7, 5, ladders * K), [ch.n.value for ch in ref.chains])
    st = info["steppers"][0]
    for j, name in enumerate(["mu", "s", "k"]):
        assert np.array_equal(_bits(st[name]["prop_log_scale"]), _bits([ch.pls[j] for ch in ref.chains])), name
        assert np.array_equal(st[name]["acceptance_count"], [ch.acc[j] for ch in ref.chains]), name
    assert np.array_equal(_bits(st["v"]["prop_log_scale"]), _bits(np.asarray([ch.pls[3:6] for ch in ref.chains]).T))
    t = info["tempering"]
    assert t["rounds"] == ref.rounds == 54 and t["temperatures"] == TEMPS
    assert np.array_equal(t["swap_accepts"], ref.accepts.sum(axis=0)) and t["swap_accepts"].sum() > 0
    assert list(t["swap_attempts"]) == [ladders * 27, ladders * 27, ladders * 27]
    assert np.allclose(t["swap_rate"], t["swap_accepts"] / t["swap_attempts"])


def test_tempered_statistics_sweep_follows_the_reference(gpu_pkg, orc):
    """amwg_stat_sweep_kernel<true> (config 2's Normal model, AMWG_JIT=0): its steps are decided from cached terms and one data pass
    (DESIGN.md §4), so a chain may leave the reference where exp(beta delta) lies within rounding of a uniform; the ladders that
    never meet such a tie (almost all) must equal the reference bit for bit, and the rounds must agree."""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    O = orc.lib()
    x = config2_data()[:64].tolist()
    params = {"mu": {"type": "real", "init": 180.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}

    def lp(st, d):
        l = 0
        l += ld.norm(st.mu, 0, 100)
        l += ld.unif(st.sigma, 0, 100)
        for i in range(len(d)):
            l += ld.norm(d[i], st.mu, st.sigma)
        return l

    def f(v):
        l = O.orc_ld_norm(v[0], 0, 100) + O.orc_ld_unif(v[1], 0, 100)
        for xi in x:
            l += O.orc_ld_norm(xi, v[0], v[1])
        return l
    ladders, seed = 16, 5
    with env(AMWG_JIT="0"):
        s = mcmc.AmwgSampler(params, lp, x, {"chains": ladders * 4, "seed": seed, "temperatures": TEMPS})
        assert "stat" in " ".join(s.program_summary()).lower() or s._program.stat_prog >= 0
        got = s.sample(40)
        state = s.state
    ref = temper_ref.RefLadder(orc, f, params, seed, [1.0 / t for t in TEMPS], ladders)
    draws = ref.sample(40, [0, 1])
    X = ref.states()
    same = 0
    for ell in range(ladders):
        c = slice(4 * ell, 4 * ell + 4)
        ok = (np.array_equal(_bits(got["mu"][:, ell]), _bits(draws[:, 0, ell])) and np.array_equal(_bits(got["sigma"][:, ell]), _bits(draws[:, 1, ell]))
              and np.array_equal(_bits(state["mu"][c]), _bits(X[c, 0])) and np.array_equal(_bits(state["sigma"][c]), _bits(X[c, 1])))
        same += ok
    assert same >= ladders - 2, "%d of %d ladders equal the reference" % (same, ladders)
    assert s.info()["tempering"]["rounds"] == ref.rounds == 40


def test_results_do_not_depend_on_how_ladders_are_split(gpu_pkg):
    """One handle of 48 chains, and two handles holding ladders [0, 6) and [6, 12) (first_chain 24): the same bits"""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    opts = {"seed": 12, "faithful": True, "temperatures": TEMPS}
    one = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=48))
    a = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=24))
    b = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=24, first_chain=24))
    for s in (one, a, b):
        s.burn(17)
    d1, da, db = one.sample(25), a.sample(25), b.sample(25)
    for name in ("mu", "s", "k", "v", "m", "var"):
        assert np.array_equal(_bits(d1[name]), _bits(np.concatenate([da[name], db[name]], axis=1))), name
        assert np.array_equal(_bits(one.state[name]), _bits(np.concatenate([a.state[name], b.state[name]], axis=0))), name
    ta, tb, t1 = a.info()["tempering"], b.info()["tempering"], one.info()["tempering"]
    assert np.array_equal(t1["swap_accepts"], ta["swap_accepts"] + tb["swap_accepts"]) and t1["rounds"] == ta["rounds"] == 42


# ---- the exact laws on a bimodal posterior ----------------------------------------------------------------------------------------
W, M = (0.3, 0.7), (-8.0, 8.0)


def _mixture(ld, mcmc):
    def lp(st, d=None):
        return mcmc.Math.log(0.3 * mcmc.Math.exp(ld.norm(st.x, -8, 1)) + 0.7 * mcmc.Math.exp(ld.norm(st.x, 8, 1)))
    return lp


def _log_mixture(x):
    return np.logaddexp(math.log(W[0]) + stats.norm.logpdf(x, M[0], 1), math.log(W[1]) + stats.norm.logpdf(x, M[1], 1))


def _tempered_cdf(beta):
    """the CDF of p^beta, normalised numerically on a fine grid"""
    grid = np.linspace(-200, 200, 800001)
    lw = beta * _log_mixture(grid)
    w = np.exp(lw - lw.max())
    c = np.cumsum((w[1:] + w[:-1]) * 0.5 * np.diff(grid))
    c = np.concatenate([[0.0], c / c[-1]])
    return lambda q: np.interp(q, grid, c)


def test_ladder_samples_a_bimodal_posterior_that_one_chain_cannot(gpu_pkg):
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    temps = [2.0 ** k for k in range(8)]
    n = 1 << 16
    params = {"x": {"type": "real", "init": -8.0}}
    s = mcmc.AmwgSampler(params, _mixture(ld, mcmc), None, {"chains": n, "seed": 2024, "temperatures": temps})
    s.burn(2000)
    s.stop_adaptation()                                              # then sample the laws with fixed proposal scales
    s.burn(1000)
    x = np.asarray(s.state["x"])
    cold = x[0::8]
    mix_cdf = lambda q: W[0] * stats.norm.cdf(q, M[0], 1) + W[1] * stats.norm.cdf(q, M[1], 1)
    assert stats.kstest(cold, mix_cdf).pvalue > 0.01
    assert abs(np.mean(cold > 0) - 0.7) < 0.03
    for r in range(8):
        p = stats.kstest(x[r::8], _tempered_cdf(1.0 / temps[r])).pvalue
        assert p > 0.01, (r, p)
    t = s.info()["tempering"]
    assert t["rounds"] == 3000 and np.all(t["swap_rate"] > 0.05)
    control = mcmc.AmwgSampler(params, _mixture(ld, mcmc), None, {"chains": n, "seed": 2024})
    control.burn(3000)
    # without the ladder almost every chain stays in the mode it started in (a few cross the 32-nat barrier when adaptation has grown
    # their proposal scale): the pooled draws would put about 0.03 of the mass in a mode that holds 0.7 of it
    assert np.mean(np.asarray(control.state["x"]) > 0) < 0.1


# ---- summaries ----------------------------------------------------------------------------------------------------------------------
def test_sample_summary_summarises_the_cold_chains(gpu_pkg):
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    opts = {"chains": 4 * 1024, "seed": 77, "temperatures": TEMPS}
    a = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts))
    b = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts))
    a.burn(50)
    b.burn(50)

    def loglik(st, d, i):
        return ld.norm(d[i], st.mu + 0.5 * st.m, st.s)
    summ = a.sample_summary(60, diagnostics=True, mcse=True, histogram={"bins": 16}, covariance=True, loo={"log_lik": loglik, "points": len(Y)})
    names = ["mu", "s", "k", "v", "m", "var"]
    entries = [e for nm in names for e in b._entries(nm)]
    block = b._sample_raw(60, 1, entries, 60).copy()                     # [rows, entries, 1024]: the twin's cold draws
    raw = {nm: b._shape_out(nm, block[:, [entries.index(e) for e in b._entries(nm)], :], b.cold_chains) for nm in names}
    # the summary code on that block, told the chain count explicitly: what sample_summary must have computed
    import torch
    from bayes_js_b200 import summary as sm
    probs = (0.025, 0.25, 0.5, 0.75, 0.975)
    red = sm.CudaBlockReducer(0)
    tb = torch.from_numpy(np.ascontiguousarray(block)).to("cuda:0")
    res = sm.summarise_block(red, tb, 60, 1024, probs, False, True)
    mc = sm.mcse_block(red, tb, 60, 1024, probs, res[0], res[1], res[3], False)
    for nm, e in (("mu", 0), ("s", 1), ("k", 2), ("var", 7)):
        r = summ[nm]
        for key in ("ess_mean", "ess_tail", "mcse_mean", "rhat_split"):
            assert _bits(r[key]) == _bits(res[4][0][key][e]), (nm, key)
        assert np.array_equal(_bits(r["mcse_quantile"]), _bits(mc["mcse_quantile"][:, e])), nm
        assert np.array_equal(_bits(r["ess_quantile"]), _bits(mc["ess_quantile"][:, e])) and _bits(r["mcse_sd"]) == _bits(mc["mcse_sd"][e]), nm
    # covariance over the 1024 cold chains, and PSIS-LOO over S = 60 x 1024 draws, against numpy
    X = np.concatenate([np.asarray(raw[nm], np.float64).reshape(60 * 1024, -1) for nm in names], axis=1)
    assert np.allclose(np.asarray(summ["covariance"]["cov"]), np.cov(X, rowvar=False), rtol=1e-9, atol=1e-12)
    import loo_ref
    mu, sd, m = (np.asarray(raw[nm], np.float64).reshape(-1) for nm in ("mu", "s", "m"))
    ll = np.stack([stats.norm.logpdf(y, mu + 0.5 * m, sd) for y in Y], axis=1)
    want = loo_ref.loo(ll)
    for key in ("elpd_loo", "p_loo", "elpd_waic", "p_waic"):
        assert np.isclose(summ["loo"][key], want[key], rtol=1e-9, atol=1e-9), key
    assert np.allclose(summ["loo"]["pointwise"]["pareto_k"], want["pointwise"]["pareto_k"], rtol=1e-6, atol=1e-9)
    assert summ["loo"]["n_draws"] == summ["covariance"]["n_draws"] == 60 * 1024
    for name in ("mu", "s", "k", "var"):
        d = np.asarray(raw[name], dtype=np.float64)
        r = summ[name]
        assert r["n_draws"] == d.size == 60 * 1024
        assert np.isclose(r["mean"], d.mean(), rtol=1e-12, atol=1e-12) and np.isclose(r["sd"], d.std(ddof=1), rtol=1e-10)
        assert np.allclose(r["quantiles"], np.quantile(d.reshape(-1), [0.025, 0.25, 0.5, 0.75, 0.975]), rtol=1e-12, atol=1e-12)
        assert int(np.sum(r["hist"])) + int(np.sum(r["hist_outside"])) == d.size
    assert np.array_equal(_bits(a.state["mu"]), _bits(b.state["mu"]))        # summary and sample advance the chains alike
    before = a.state["mu"].copy()
    rounds = a.info()["tempering"]["rounds"]
    with pytest.raises(ValueError, match="nested= is not available with options.temperatures"):
        a.sample_summary(10, nested=2)
    with pytest.raises(ValueError, match="ppc= is not available with options.temperatures"):
        a.sample_summary(10, ppc={"log_lik": loglik, "points": len(Y)})
    assert np.array_equal(_bits(a.state["mu"]), _bits(before)) and a.info()["tempering"]["rounds"] == rounds


def _rng_n(img, D, P, C_):
    """the stream positions of an image's chains (amwg_checkpoint.h layout, P <= 16)"""
    off = 56 + 24 * D + 16 * D * C_ + 8 * C_
    return np.frombuffer(bytes(img[off:off + 8 * C_]), dtype=np.uint64)


def test_checkpoint_mid_run_continues_bit_for_bit(gpu_pkg):
    """Stop mid-batch (mu adapts every 7 sweeps) on an odd round, restore into one handle and into two handles split at a ladder
    boundary: the continuation equals never stopping -- draws, state, info and the ladder's counters"""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    opts = {"seed": 19, "faithful": True, "temperatures": TEMPS, "params": {"mu": {"batch_size": 7}}}
    full = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=32))
    full.burn(11)
    img = full.checkpoint()
    assert full.info()["tempering"]["rounds"] == 11
    want = full.sample(20)
    want_info = full.info()
    one = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=32, seed=1))
    one.restore(img)
    lo = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=16, seed=2))
    hi = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=16, first_chain=16, seed=3))
    lo.restore(img)
    hi.restore(img)
    got1, glo, ghi = one.sample(20), lo.sample(20), hi.sample(20)
    for name in ("mu", "s", "k", "v", "m", "var"):
        assert np.array_equal(_bits(got1[name]), _bits(want[name])), name
        assert np.array_equal(_bits(np.concatenate([glo[name], ghi[name]], axis=1)), _bits(want[name])), name
    i1 = one.info()
    assert i1["tempering"]["rounds"] == want_info["tempering"]["rounds"] == 31
    assert np.array_equal(i1["tempering"]["swap_accepts"], want_info["tempering"]["swap_accepts"])
    assert np.array_equal(lo.info()["tempering"]["swap_accepts"] + hi.info()["tempering"]["swap_accepts"], want_info["tempering"]["swap_accepts"])
    for name in ("mu", "s", "k"):
        assert np.array_equal(_bits(i1["steppers"][0][name]["prop_log_scale"]), _bits(want_info["steppers"][0][name]["prop_log_scale"]))
    assert np.array_equal(_rng_n(one.checkpoint(), 7, 5, 32), _rng_n(full.checkpoint(), 7, 5, 32))
    # another ladder, an untempered sampler, and a ladder split across the handle's range are refused, and change nothing
    other = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, dict(opts, chains=32, temperatures=[1.0, 1.7, 3.1, 6.6]))
    plain = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": 32, "seed": 19, "faithful": True, "params": {"mu": {"batch_size": 7}}})
    for s_, msg in ((other, "restore: the image was taken with other temperatures"),
                    (plain, "restore: the image is of a tempered ladder (options.temperatures) and this sampler is not tempered")):
        before = s_.state["mu"].copy()
        with pytest.raises(mcmc.JsThrow) as e:
            s_.restore(img)
        assert str(e.value) == msg and np.array_equal(_bits(s_.state["mu"]), _bits(before))
    with pytest.raises(mcmc.JsThrow) as e:
        full.restore(plain.checkpoint())
    assert str(e.value) == "restore: this sampler is a tempered ladder (options.temperatures) and the image is not"


def test_ladder_is_set_before_the_chains_move(gpu_pkg):
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    L = gpu_pkg._ffi.lib()
    s = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": 8, "seed": 3})
    s.burn(1)
    beta = (C.c_double * 2)(1.0, 0.5)
    assert L.amwg_set_ladder(s._handle, beta, 2) != 0 and b"chains have moved" in L.amwg_last_error()
    s = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": 8, "seed": 3, "temperatures": [1, 2]})
    assert L.amwg_set_ladder(s._handle, beta, 2) != 0 and b"already has a ladder" in L.amwg_last_error()
    t = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": 6, "seed": 3})
    bad = (C.c_double * 4)(1.0, 0.5, 0.5, 0.1)
    assert L.amwg_set_ladder(t._handle, bad, 3) != 0 and b"strictly decreasing" in L.amwg_last_error()
    assert L.amwg_set_ladder(t._handle, beta, 4) != 0                          # 6 chains are not whole ladders of 4
    rounds = C.c_uint64(7)
    assert L.amwg_ladder_info(t._handle, C.byref(rounds), None) == 0 and rounds.value == 0


# ---- the JavaScript host ------------------------------------------------------------------------------------------------------------
def _js_native(gpu_pkg):
    from js_host import DeviceNative, _num_list
    from oracle.minijs.minijs import undefined

    class LadderNative(DeviceNative):
        """DeviceNative plus `set_ladder` / `ladder_info` (js/amwg_napi.cc), and `sample` sized for the recorded (cold) chains"""

        def __call__(self, host):
            o = super().__call__(host)
            it = host.it
            L = self.pkg._ffi.lib()
            K_of = {}

            def set_ladder(this, a):
                b = np.asarray(_num_list(a[1]), dtype=np.float64)
                if L.amwg_set_ladder(self.handles[a[0]], b.ctypes.data_as(C.POINTER(C.c_double)), b.size) != 0:
                    self._fail()
                K_of[a[0]] = b.size
                return undefined

            def ladder_info(this, a):
                rounds, acc = C.c_uint64(0), np.zeros(256, dtype=np.int64)
                K = L.amwg_ladder_info(self.handles[a[0]], C.byref(rounds), acc.ctypes.data_as(C.POINTER(C.c_int64)))
                if K < 0:
                    self._fail()
                r = it.new_object()
                r.put("rounds", float(rounds.value))
                r.put("accepts", it.new_array([float(v) for v in acc[:max(K - 1, 0)]]))
                return r

            def sample(this, a):
                n, thin, mon = int(a[1]), int(a[2]), np.asarray(_num_list(a[3]), dtype=np.int32)
                C_ = self.meta[a[0]][2] // K_of.get(a[0], 1)
                rows = 0 if n <= 0 else (n + thin - 1) // thin
                out = np.empty((max(rows, 1), max(mon.size, 1), C_))
                if L.amwg_sample(self.handles[a[0]], n, thin, mon.ctypes.data_as(C.POINTER(C.c_int32)), mon.size, out.ctypes.data) != 0:
                    self._fail()
                return it.new_array([float(v) for v in out[:rows, :mon.size].reshape(-1)])

            o.put("set_ladder", it.make_native("set_ladder", set_ladder))
            o.put("ladder_info", it.make_native("ladder_info", ladder_info))
            o.put("sample", it.make_native("sample", sample))
            return o
    return LadderNative(gpu_pkg)


JS_MODEL = r"""
var mix_post = function(st, d) {
  var l = 0;
  l += ld.norm(st.mu, 0, 5);
  l += ld.gamma(st.s, 2, 1);
  l += ld.norm(st.k, 2, 3);
  l += ld.bern(st.m, 0.3);
  for (var j = 0; j < 3; j++) { l += ld.norm(st.v[j], st.mu, st.s); }
  for (var i = 0; i < d.length; i++) { l += ld.norm(d[i], st.mu + 0.5 * st.m, st.s); }
  st.var = st.s * st.s;
  return l;
};
"""


def test_javascript_host_gives_the_python_hosts_bits(gpu_pkg):
    from js_host import JsHost, to_py
    from oracle.minijs.minijs import to_js
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc
    h = JsHost(native=_js_native(gpu_pkg))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.it.set_global("ld", h.load("distributions"))
    h.run(JS_MODEL)
    h.it.set_global("the_data", to_js(h.it, Y))
    h.run("""
      var P = {mu: {type: "real"}, s: {type: "real", lower: 0, init: 1.5}, k: {type: "int", lower: -20, upper: 20},
               v: {type: "real", dim: [3]}, m: {type: "binary"}};
      var S = new mcmc.AmwgSampler(P, mix_post, the_data, {chains: 32, seed: 61, faithful: true, temperatures: [1, 1.7, 3.1, 6.5]});
      S.burn(9);
      var d = S.sample(12);
      var inf = S.info();
      var err = "";
      try { new mcmc.AmwgSampler(P, mix_post, the_data, {chains: 30, temperatures: [1, 1.7, 3.1, 6.5]}); } catch (e) { err = e; }
      var err2 = "";
      try { new mcmc.AmwgSampler(P, mix_post, the_data, {chains: 32, temperatures: [1, 3, 2, 6.5]}); } catch (e) { err2 = e; }
      S.close();
    """)
    s = mcmc.AmwgSampler(PARAMS_MIX, _lp_mix(ld), Y, {"chains": 32, "seed": 61, "faithful": True, "temperatures": TEMPS})
    s.burn(9)
    p = s.sample(12)
    pi = s.info()
    js = to_py(h.get("d"))
    for name in ("mu", "s", "k", "v", "m", "var"):
        assert np.array_equal(_bits(js[name]), _bits(p[name])), name
    ji = to_py(h.get("inf"))
    assert ji["tempering"]["rounds"] == pi["tempering"]["rounds"] == 21
    assert np.array_equal(np.asarray(ji["tempering"]["swap_accepts"]), pi["tempering"]["swap_accepts"])
    assert list(ji["tempering"]["swap_attempts"]) == list(pi["tempering"]["swap_attempts"])
    for name in ("mu", "s", "k"):
        assert np.array_equal(_bits(ji["steppers"][0][name]["prop_log_scale"]), _bits(pi["steppers"][0][name]["prop_log_scale"]))
    assert h.get("err") == "options.temperatures: their number must divide options.chains"
    assert h.get("err2") == "options.temperatures must be strictly increasing"
