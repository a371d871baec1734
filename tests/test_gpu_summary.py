"""On-device posterior summaries (SURVEY 8(f).3) against numpy on the raw draws of an identically seeded sampler: exact
quantiles (order statistics are integers' work: bit-exact), moments within rounding of the different summation order."""
import ctypes as C

import numpy as np
import pytest

import models
from conftest import NORM_DATA, config2_data
from summary_ref import NumpyBlockReducer, numpy_summary

pytestmark = pytest.mark.gpu
PROBS = (0.0, 0.025, 0.25, 0.5, 0.75, 0.975, 1.0)


def _check(summary, raw, name, rows, probs=PROBS):
    x = raw[name]                                           # [rows, chains, *dim]
    dim = x.shape[2:]
    flat = x.reshape(x.shape[0], x.shape[1], -1)            # [rows, chains, entries]
    m0, s0, r0, q0 = numpy_summary(np.moveaxis(flat, 2, 1), probs)
    got = summary[name]
    shape = (lambda a: a.reshape(dim)) if dim else (lambda a: a[0])
    assert np.allclose(got["mean"], shape(m0), rtol=1e-12, atol=0)
    assert np.allclose(got["sd"], shape(s0), rtol=1e-10, atol=0)
    assert np.allclose(got["rhat"], shape(r0), rtol=1e-8, atol=0, equal_nan=True)
    want_q = q0.reshape((len(probs),) + dim) if dim else q0[:, 0]
    assert np.array_equal(np.asarray(got["quantiles"]), want_q), name
    assert got["n_draws"] == x.shape[0] * x.shape[1]


def test_summary_matches_numpy_on_the_raw_draws_config2_shape(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    a = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21})
    b = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21})
    a.burn(2500); b.burn(2500)
    raw = a.sample(50)
    summ = b.sample_summary(50, PROBS)
    for name in ("mu", "sigma"):
        _check(summ, raw, name, 50)
    assert abs(summ["mu"]["mean"] - np.mean(data)) < 0.05 and 1.0 <= summ["mu"]["rhat"] < 1.5
    # the chains advanced exactly as sample(50) advances them
    sa, sb = a.state, b.state
    assert np.array_equal(sa["mu"], sb["mu"]) and np.array_equal(sa["sigma"], sb["sigma"])


def test_summary_with_thin_monitor_multidim_int_and_derived(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"x": {"type": "int", "dim": [2, 2], "lower": 0, "init": [[1, 10], [100, 1000]]}}
    mk = lambda: mcmc.AmwgSampler(pars, models.multivar_poisson_dens(ld), None, {"chains": 300, "seed": 5, "thin": 3})
    a, b = mk(), mk()
    a.burn(100); b.burn(100)
    raw, summ = a.sample(31), b.sample_summary(31, (0.1, 0.5, 0.9))
    assert raw["x"].shape == (11, 300, 2, 2) and summ["x"]["quantiles"].shape == (3, 2, 2)
    _check(summ, raw, "x", 11, (0.1, 0.5, 0.9))
    # the reference's test model with a derived quantity (tests/test_data.js:80-91), monitoring a subset
    pars = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    mk = lambda: mcmc.AmwgSampler(pars, models.norm_post_test(ld), NORM_DATA, {"chains": 257, "seed": 6, "monitor": ["var", "mu"]})
    a, b = mk(), mk()
    a.burn(200); b.burn(200)
    raw, summ = a.sample(20), b.sample_summary(20)
    assert set(summ) == {"var", "mu"}
    for name in ("var", "mu"):
        _check(summ, raw, name, 20, (0.025, 0.25, 0.5, 0.75, 0.975))
    with pytest.raises(gpu_pkg.tracer.JsThrow):
        b.sample_summary(0)


def test_c_abi_reductions_on_an_adversarial_block(gpu_pkg):
    """ties, both zeros, infinities, 40 orders of magnitude, a constant column: the digit counts equal numpy's, count for count."""
    import torch
    from bayes_js_b200.summary import CudaBlockReducer, RadixSelect, quantile_targets
    rng = np.random.default_rng(3)
    rows, entries, chains = 13, 4, 1000
    x = rng.normal(0, 1, (rows, entries, chains))
    x[:, 1] = np.round(3 * x[:, 1]); x[0, 1, :5] = -0.0
    x[:, 2] = np.exp(20 * x[:, 2]) * np.sign(rng.normal(size=(rows, chains))); x[1, 2, 0] = np.inf; x[2, 2, 1] = -np.inf
    x[:, 3] = 7.25
    dev = torch.device("cuda", 0)
    block = torch.from_numpy(x).to(dev)
    red, ref = CudaBlockReducer(0), NumpyBlockReducer()
    ranks, _ = quantile_targets(rows * chains, PROBS)
    sel_d, sel_h = RadixSelect(entries, ranks), RadixSelect(entries, ranks)
    for p in range(8):
        table, which = sel_d.prefixes()
        cd = red.digit_counts(block, p, table).cpu().numpy()
        ch = ref.digit_counts(torch.from_numpy(x), p, table).numpy()
        for e in range(entries):                                # padded repeats of a prefix are not counted by the device
            assert np.array_equal(cd[e, which[e]], ch[e, which[e]]), (p, e)
        assert cd[:, 0].sum() == entries * rows * chains if p == 0 else True
        sel_d.advance(cd, which); sel_h.advance(ch, which)
    flat = np.sort(np.moveaxis(x, 1, 0).reshape(entries, -1), axis=1)
    assert np.array_equal(sel_d.values(), flat[:, ranks])     # by value: np.sort leaves -0.0 / +0.0 in arbitrary order, the key order is -0 < +0
    assert np.array_equal(sel_d.values().view(np.uint64), sel_h.values().view(np.uint64))
    fin = np.isfinite(x).all(axis=(0, 2))
    got, want = red.moments(block), ref.moments(torch.from_numpy(x))
    assert np.array_equal(got[:, 0], want[:, 0])
    assert np.allclose(got[fin, 1:], want[fin, 1:], rtol=1e-11, atol=1e-300)
    assert got[3, 1] == 7.25 and got[3, 2] == 0 and got[3, 3] == 0
    # argument checks come back as errors, not crashes
    L = gpu_pkg._ffi.lib()
    assert L.amwg_summary_digit_hist(0, block.data_ptr(), rows, entries, chains, 8, block.data_ptr(), 1, block.data_ptr()) != 0
    assert L.amwg_summary_digit_hist(0, block.data_ptr(), rows, entries, chains, 0, block.data_ptr(), 33, block.data_ptr()) != 0
    assert b"n_prefix" in L.amwg_last_error()
    assert L.amwg_summary_moments(0, block.data_ptr(), 0, entries, chains, got.ctypes.data) != 0


@pytest.mark.parametrize("device", [64, -1])
def test_every_reduction_refuses_a_device_index_out_of_range(gpu_pkg, device):
    """each device-taking summary entry point, with arguments that are otherwise valid, names itself and touches nothing"""
    import torch
    L = gpu_pkg._ffi.lib()
    blk = torch.zeros((4, 5, 7), dtype=torch.float64, device="cuda:0")
    p = blk.data_ptr()
    host = np.zeros(64)
    h = host.ctypes.data
    pairs, sel, skip = np.array([[0, 1]], dtype=np.int32), np.array([0, 1], dtype=np.int32), np.zeros(5, dtype=np.int32)
    calls = {"amwg_summary_moments": (p, 4, 5, 7, h),
             "amwg_summary_digit_hist": (p, 4, 5, 7, 0, p, 1, p),
             "amwg_summary_autocov": (p, 4, 5, 7, None, 0, 1, h),
             "amwg_summary_rank_sort": (p, 4, 5, 7, 0, float("nan"), p, p, None),
             "amwg_summary_rank_count": (p, 5, p, 5, p),
             "amwg_summary_rank_z": (p, p, 5, 5, p),
             "amwg_summary_finite_range": (p, 4, 5, 7, p, p),
             "amwg_summary_histogram": (p, 4, 5, 7, p, 8, p),
             "amwg_summary_histogram2d": (p, 4, 5, 7, pairs.ctypes.data, 1, p, 8, p),
             "amwg_summary_comoments": (p, 4, 5, 7, sel.ctypes.data, 2, h),
             "amwg_summary_nested": (p, 4, 5, 7, 0, 1, h),
             "amwg_summary_threshold_counts": (p, 4, 5, 7, h, p),
             "amwg_loo_reduce": (p, 4, 5, 7, h, h, h, 8, p, p, h),
             "amwg_loo_fit": (p, p, 1, 5, 8, h, h, skip.ctypes.data, h)}
    for name, args in calls.items():
        assert getattr(L, name)(device, *args) != 0, name
        assert L.amwg_last_error() == name.encode() + b": device index out of range"
    assert np.all(host == 0) and not blk.any()
