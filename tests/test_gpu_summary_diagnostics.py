"""Split-chain diagnostics (ESS, MCSE, split R-hat) of the on-device summary: amwg_summary_autocov against its numpy
restatement on an adversarial block, sample_summary(..., diagnostics=True) against the FFT restatement applied to the raw
draws of an identically seeded sampler, and AR(1) chains of known autocorrelation time uploaded to the device."""
import numpy as np
import pytest

import models
from conftest import NORM_DATA, config2_data
from ess_ref import ar1, autocov_records, fft_diagnostics

pytestmark = pytest.mark.gpu
KEYS = ("ess_mean", "ess_tail", "mcse_mean", "rhat_split")
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)


ADVERSARIAL = [
    (23, 1184 * 256 + 77, [(0, 11), (3, 7), (0, 1), (1, 10), (10, 1)]),     # more chains than kChainCtas * 256: grid-stride
    (71, 1000, [(0, 32), (3, 17), (17, 16), (19, 16), (34, 1)]),           # windows of more than 16 lags: two kernel passes
]


@pytest.mark.parametrize("rows,chains,windows", ADVERSARIAL)
def test_c_abi_autocov_on_an_adversarial_block(gpu_pkg, rows, chains, windows):
    """chains not a multiple of 256, odd rows, ties, +-inf, a constant column, windows at lag0 > 0 and of 1..32 lags: lag sums
    within rounding, moment records as the moments reduction's, two calls bit-identical"""
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    entries = 4
    x = ar1(0.5, rows, chains, entries, seed=8)
    x[:, 1] = np.round(2 * x[:, 1])
    x[:, 2] = np.exp(3 * x[:, 2]); x[4, 2, 9] = np.inf; x[7, 2, 100] = -np.inf
    x[:, 3] = 7.25
    thr = np.stack([np.quantile(np.moveaxis(x, 1, 0).reshape(entries, -1), p, axis=1) for p in (0.05, 0.95)], axis=1)
    thr[1] = (-1.0, 1.0)                                        # ties on both thresholds
    block = torch.from_numpy(x).to(torch.device("cuda", 0))
    red = CudaBlockReducer(0)
    fin = np.isfinite(x).all(axis=(0, 2))
    h = rows // 2
    for i, (lag0, n_lags) in enumerate(windows):
        t = None if i % 3 == 2 else thr
        got = red.autocov(block, t, lag0, n_lags)
        again = red.autocov(block, t, lag0, n_lags)
        assert np.array_equal(got.view(np.uint64), again.view(np.uint64)), (lag0, n_lags)
        want = autocov_records(x, t, lag0, n_lags)
        assert got.shape == want.shape
        assert np.array_equal(got[:, :, 0], want[:, :, 0])
        scale = np.maximum(np.abs(want[:, :, 3:4]), 1e-300)          # lag sums: rounding relative to sum d^2
        for e in range(entries):
            for s in range(got.shape[1]):
                if s == 0 and not fin[e]:
                    assert np.all(np.isnan(got[e, 0, 3:])) or not np.all(np.isfinite(got[e, 0, 3:]))
                    continue
                assert np.allclose(got[e, s, 1:3], want[e, s, 1:3], rtol=1e-11, atol=1e-300), (lag0, e, s)
                assert np.allclose(got[e, s, 3:], want[e, s, 3:], rtol=0, atol=1e-11 * scale[e, s, 0]), (lag0, e, s)
        assert got[3, 0, 1] == 7.25 and np.all(got[3, 0, 2:] == 0)
    L = gpu_pkg._ffi.lib()
    out = np.empty(64 * 40)
    p = block.data_ptr()
    bad = [(1, entries, chains, 0, 1), (rows, entries, chains, 0, 0), (rows, entries, chains, 0, 33), (rows, entries, chains, h - 1, 2),
           (rows, entries, chains, -1, 2)]
    for r, e, c, l0, n in bad:
        assert L.amwg_summary_autocov(0, p, r, e, c, None, l0, n, out.ctypes.data) != 0
        assert L.amwg_last_error().startswith(b"amwg_summary_autocov")
    assert L.amwg_summary_autocov(0, None, rows, entries, chains, None, 0, 2, out.ctypes.data) != 0
    assert b"null" in L.amwg_last_error()
    assert L.amwg_summary_autocov(0, p, rows, entries, chains, None, 0, 2, None) != 0
    assert L.amwg_summary_autocov(0, p, rows, entries, chains, None, 0, 40, out.ctypes.data) != 0
    assert b"n_lags" in L.amwg_last_error()


def _check(summ, raw, name):
    x = raw[name]                                              # [rows, chains, *dim]
    dim = x.shape[2:]
    flat = np.moveaxis(x.reshape(x.shape[0], x.shape[1], -1), 2, 1)
    want = fft_diagnostics(flat)
    shape = (lambda a: a.reshape(dim)) if dim else (lambda a: a[0])
    for k in KEYS:
        assert np.allclose(summ[name][k], shape(want[k]), rtol=1e-9, atol=0, equal_nan=True), (name, k, summ[name][k], want[k])


def _same(a, b):
    assert set(a) == set(b)
    for name in a:
        for k in a[name]:
            assert np.atleast_1d(np.asarray(a[name][k])).tobytes() == np.atleast_1d(np.asarray(b[name][k])).tobytes(), (name, k)


def test_diagnostics_match_the_raw_draws_config2_shape(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    mk = lambda: mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(1000)
    raw = a.sample(100)
    summ = b.sample_summary(100, PROBS, diagnostics=True)
    plain = c.sample_summary(100, PROBS)
    for name in ("mu", "sigma"):
        _check(summ, raw, name)
        assert summ[name]["ess_mean"] > 0 and summ[name]["rhat_split"] < 1.5
    _same(plain, {n: {k: v for k, v in d.items() if k not in KEYS} for n, d in summ.items()})
    sa, sb, sc = a.state, b.state, c.state
    for name in ("mu", "sigma"):
        assert np.array_equal(sa[name], sb[name]) and np.array_equal(sa[name], sc[name])


def test_diagnostics_with_thin_monitor_multidim_int_and_derived(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"x": {"type": "int", "dim": [2, 2], "lower": 0, "init": [[1, 10], [100, 1000]]}}
    mk = lambda: mcmc.AmwgSampler(pars, models.multivar_poisson_dens(ld), None, {"chains": 300, "seed": 5, "thin": 3})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(300)
    raw, summ, plain = a.sample(61), b.sample_summary(61, (0.1, 0.5, 0.9), diagnostics=True), c.sample_summary(61, (0.1, 0.5, 0.9))
    assert raw["x"].shape == (21, 300, 2, 2) and summ["x"]["ess_mean"].shape == (2, 2)
    _check(summ, raw, "x")
    _same(plain, {n: {k: v for k, v in d.items() if k not in KEYS} for n, d in summ.items()})
    assert np.array_equal(a.state["x"], b.state["x"]) and np.array_equal(a.state["x"], c.state["x"])
    pars = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    mk = lambda: mcmc.AmwgSampler(pars, models.norm_post_test(ld), NORM_DATA, {"chains": 257, "seed": 6, "monitor": ["var", "mu"]})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(200)
    raw, summ, plain = a.sample(40), b.sample_summary(40, diagnostics=True), c.sample_summary(40)
    assert set(summ) == {"var", "mu"}
    for name in ("var", "mu"):
        _check(summ, raw, name)
    _same(plain, {n: {k: v for k, v in d.items() if k not in KEYS} for n, d in summ.items()})
    short = b.sample_summary(9, diagnostics=True)              # fewer than 10 kept rows: NaN
    assert all(np.isnan(short["mu"][k]) for k in KEYS)


@pytest.mark.parametrize("phi,rows", [(0.9, 1000), (0.0, 1000), (-0.5, 4000)])
def test_ar1_known_answers_on_the_device(gpu_pkg, phi, rows):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer, summarise_block
    chains = 2000
    x = ar1(phi, rows, chains, 1, seed=10 + rows)
    block = torch.from_numpy(x).to(torch.device("cuda", 0))
    *_, (diag, windows) = summarise_block(CudaBlockReducer(0), block, rows, chains, PROBS, False, diagnostics=True)
    tau = (1 + phi) / (1 - phi)
    got = diag["ess_mean"][0] / (2 * chains * (rows // 2))
    assert abs(got * tau - 1) < 0.06, (phi, got * tau, windows)
    assert np.isclose(diag["ess_mean"][0], fft_diagnostics(x)["ess_mean"][0], rtol=1e-9)
