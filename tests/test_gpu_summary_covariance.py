"""Posterior covariance of sample_summary(..., covariance=...) on the GPU: the device record against an fsum reference within its
stated bound (tests/cov_ref.py), cov / corr / mean / rhat_multivariate against numpy and scipy on the raw draws of an identically
seeded sampler, every other key byte for byte unchanged, the chains advanced as sample(n) advances them, and the C ABI's checks."""
import numpy as np
import pytest

import cov_ref
import models
from conftest import config2_data

pytestmark = pytest.mark.gpu


def _bytes(v):
    return np.asarray(v).tobytes()


def _raw_block(raw, labels):
    """sample() output -> [rows, n, chains] in the order of the covariance labels"""
    cols = []
    for lab in labels:
        name, i = (lab, None) if isinstance(lab, str) else lab
        v = raw[name]
        rows, chains = v.shape[:2]
        v = v.reshape(rows, chains, -1)
        cols.append(v[:, :, 0 if i is None else i])
    return np.stack(cols, axis=1)


def _check_against_numpy(cov, x):
    """x [rows, n, chains]: cov, corr, mean, within, between and rhat_multivariate against numpy / scipy on the draws"""
    import scipy.linalg
    rows, n, C = x.shape
    flat = np.moveaxis(x, 1, 0).reshape(n, -1)
    bm, bB, bW = cov_ref.device_bound(x, range(n))
    M = rows * C
    # numpy.cov's own rounding is of the order of the device's: gamma_{M+2} sum |d_i||d_j| / (M - 1)
    d = np.abs(flat - flat.mean(axis=1, keepdims=True))
    b_np = cov_ref.gamma(M + 2) * (d @ d.T) / (M - 1)
    bound = (bW + rows * bB) / (M - 1) + b_np + 4 * cov_ref.U * np.abs(np.cov(flat))
    assert np.all(np.abs(cov["cov"] - np.cov(flat)) <= bound)
    assert np.all(np.abs(cov["mean"] - flat.mean(axis=1)) <= bm + cov_ref.gamma(M) * np.abs(flat).mean(axis=1))
    sd = np.sqrt(np.diag(np.cov(flat)))
    assert np.allclose(cov["corr"], np.corrcoef(flat), rtol=0, atol=1e-9)
    assert np.allclose(np.diag(cov["corr"]), 1.0, rtol=0, atol=1e-15)
    W = x.var(axis=0, ddof=1).mean(axis=1)
    within = np.mean([np.cov(x[:, :, c].T, ddof=1).reshape(n, n) for c in range(C)], axis=0)
    between = np.cov(x.mean(axis=0), ddof=1).reshape(n, n)
    assert np.allclose(np.diag(cov["within"]), W, rtol=1e-9, atol=0)
    assert np.allclose(cov["within"], within, rtol=0, atol=1e-9 * np.outer(sd, sd).max())
    assert np.allclose(cov["between"], between, rtol=0, atol=1e-9 * np.outer(sd, sd).max())
    lam = scipy.linalg.eigh(between, within, eigvals_only=True).max()
    want = (rows - 1) / rows + (C + 1) / C * lam
    assert abs(cov["rhat_multivariate"] - want) <= 1e-8 * want, (cov["rhat_multivariate"], want)
    assert cov["n_draws"] == M


@pytest.mark.parametrize("diagnostics", [False, True, "rank"])
def test_config2_covariance_matches_numpy_and_leaves_the_summary_alone(gpu_pkg, diagnostics):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    a, b, c = (mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 23}) for _ in range(3))
    for s in (a, b, c):
        s.burn(2500)
    hist = {"bins": 20, "pairs": [("mu", "sigma")]} if diagnostics is True else None
    raw = a.sample(50)
    got = b.sample_summary(50, (0.05, 0.5, 0.95), diagnostics=diagnostics, histogram=hist, covariance=True)
    base = c.sample_summary(50, (0.05, 0.5, 0.95), diagnostics=diagnostics, histogram=hist)
    cov = got["covariance"]
    assert cov["labels"] == ["mu", "sigma"]
    x = _raw_block(raw, cov["labels"])
    _check_against_numpy(cov, x)
    assert set(got) == set(base) | {"covariance"}
    for name in base:
        assert set(got[name]) == set(base[name])
        for key, val in base[name].items():
            assert _bytes(got[name][key]) == _bytes(val), (name, key)
    assert np.allclose(np.sqrt(np.diag(cov["cov"])), [got["mu"]["sd"], got["sigma"]["sd"]], rtol=1e-12, atol=0)
    sa, sb = a.state, b.state
    assert np.array_equal(sa["mu"], sb["mu"]) and np.array_equal(sa["sigma"], sb["sigma"])


def test_config4_shape_several_tile_bands(gpu_pkg):
    """65 entries (mu dim [64] + sigma) of config 4's hierarchical model: nine 8-entry blocks, 45 tiles over 16 warps"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    J, per = 64, 32
    g = np.repeat(np.arange(J), per)
    y = np.random.default_rng(64).normal(100, 20, J)[g] + np.random.default_rng(65).normal(0, 5, J * per)
    params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    mk = lambda: mcmc.AmwgSampler(params, models.hier_norm_post(ld), {"y": y, "g": g.astype(np.float64)}, {"chains": 1000, "seed": 4})
    a, b = mk(), mk()
    a.burn(200); b.burn(200)
    raw = a.sample(20)
    got = b.sample_summary(20, (0.5,), covariance=True)
    cov = got["covariance"]
    assert cov["labels"] == [("mu", i) for i in range(J)] + ["sigma"]
    x = _raw_block(raw, cov["labels"])
    _check_against_numpy(cov, x)
    assert np.array_equal(a.state["mu"], b.state["mu"])


def _int_model(ld):
    def log_post(par, data=None):
        lp = ld.norm(par.mu, 0, 10)
        lams = [[3, 5, 8], [1, 12, 20]]
        for i in range(2):
            for j in range(3):
                lp += ld.pois(par.x[i][j], lams[i][j])
        par.var = par.mu * par.mu
        return lp
    return log_post


def test_multidim_int_thin_monitor_derived_and_a_scattered_selection(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"mu": {"type": "real"}, "x": {"type": "int", "dim": [2, 3], "lower": 0, "init": [[3, 5, 8], [1, 12, 20]]}}
    mk = lambda: mcmc.AmwgSampler(pars, _int_model(ld), None, {"chains": 1000, "seed": 8, "thin": 3, "monitor": ["x", "var", "mu"]})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(300)
    raw = a.sample(31)                                             # 11 kept rows
    got = b.sample_summary(31, (0.5,), covariance=True)
    cov = got["covariance"]
    assert cov["labels"] == [("x", i) for i in range(6)] + ["var", "mu"]
    _check_against_numpy(cov, _raw_block(raw, cov["labels"]))
    sel = ["mu", ("x", 4), "var", ("x", 0)]
    got2 = c.sample_summary(31, (0.5,), covariance=sel)
    assert got2["covariance"]["labels"] == sel
    _check_against_numpy(got2["covariance"], _raw_block(raw, sel))
    assert np.array_equal(a.state["x"], b.state["x"]) and np.array_equal(a.state["x"], c.state["x"])


@pytest.mark.parametrize("n_sel", [1, 8, 9, 128])
def test_c_abi_comoments_on_synthetic_blocks(gpu_pkg, n_sel):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    red = CudaBlockReducer(0)
    rng = np.random.default_rng(n_sel)
    for rows, chains in ((1, 1), (1, 3), (7, 1), (7, 3), (5, 1001)):
        x = 1e6 + rng.normal(size=(rows, n_sel + 3, chains)) * np.linspace(0.5, 3, n_sel + 3)[None, :, None]
        sel = rng.permutation(n_sel + 3)[:n_sel].astype(np.int32)
        block = torch.from_numpy(x).to("cuda:0")
        rec = red.comoments(block, sel)
        cov_ref.check_record(rec, x, sel, (n_sel, rows, chains))
        assert _bytes(red.comoments(block, sel)) == _bytes(rec)                # two calls, same bits
    # non-finite draws: that entry's rows and columns are NaN, the others are untouched
    rows, chains = 4, 37
    x = rng.normal(size=(rows, n_sel + 2, chains))
    x[2, 0, 5] = np.nan
    x[1, 1, 0] = np.inf
    sel = np.arange(n_sel + 2, dtype=np.int32)[:max(n_sel, 2)]
    rec = red.comoments(torch.from_numpy(x).to("cuda:0"), sel)
    n = len(sel)
    B, W = rec[1 + n:1 + n + n * n].reshape(n, n), rec[1 + n + n * n:].reshape(n, n)
    bad = np.zeros(n, dtype=bool)
    bad[:2] = True
    for M in (B, W):
        assert np.all(np.isnan(M[bad])) and np.all(np.isnan(M[:, bad]))
        assert np.all(np.isfinite(M[np.ix_(~bad, ~bad)]))
    if n > 2:
        cov_ref.check_record(np.concatenate([[chains], rec[3:1 + n], B[2:, 2:].ravel(), W[2:, 2:].ravel()]), x, sel[2:])


def test_c_abi_comoments_refuses_bad_arguments(gpu_pkg):
    import torch
    L = gpu_pkg._ffi.lib()
    block = torch.zeros((3, 5, 7), dtype=torch.float64, device="cuda:0")
    p = block.data_ptr()
    out = np.full(1 + 129 + 2 * 129 * 129, 7.0)
    sel = np.arange(129, dtype=np.int32)
    s, o = sel.ctypes.data, out.ctypes.data
    cases = [((0, p, 3, 5, 7, s, 0, o), b"n_sel"), ((0, p, 3, 5, 7, s, 129, o), b"n_sel"), ((0, p, 0, 5, 7, s, 2, o), b"empty"),
             ((0, p, 3, 0, 7, s, 2, o), b"empty"), ((0, p, 3, 5, 0, s, 2, o), b"empty"), ((0, 0, 3, 5, 7, s, 2, o), b"null"),
             ((0, p, 3, 5, 7, None, 2, o), b"null"), ((0, p, 3, 5, 7, s, 2, None), b"null"), ((0, p, 3, 5, 7, s, 6, o), b"outside"),
             ((0, p, 1 << 40, 5, 1 << 13, s, 2, o), b"2^53"), ((64, p, 3, 5, 7, s, 2, o), b"device")]
    for args, msg in cases:
        assert L.amwg_summary_comoments(*args) != 0 and msg in L.amwg_last_error(), args
        assert np.all(out == 7.0)                                              # nothing written
    neg = np.array([0, -1], dtype=np.int32)
    assert L.amwg_summary_comoments(0, p, 3, 5, 7, neg.ctypes.data, 2, o) != 0 and b"outside" in L.amwg_last_error()


def test_rhat_multivariate_flags_separated_chains(gpu_pkg):
    """a bimodal posterior along the diagonal; half the chains start in each mode and stay there"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld

    def log_post(s, d=None):
        a = ld.norm(s.u, 5, 0.5) + ld.norm(s.v, 5, 0.5)
        b = ld.norm(s.u, -5, 0.5) + ld.norm(s.v, -5, 0.5)
        return mcmc.Math.log(mcmc.Math.exp(a) + mcmc.Math.exp(b))      # 20 sd between the modes: no chain crosses
    params = {"u": {"type": "real"}, "v": {"type": "real"}}
    C = 512
    mk = lambda: mcmc.AmwgSampler(params, log_post, None, {"chains": C, "seed": 17})
    a, b = mk(), mk()
    start = np.where(np.arange(C) < C // 2, 5.0, -5.0)
    for s in (a, b):
        s.set_state({"u": start, "v": start})
        s.burn(200)
    raw = a.sample(40)
    cov = b.sample_summary(40, (0.5,), covariance=True)["covariance"]
    x = _raw_block(raw, cov["labels"])
    assert cov["rhat_multivariate"] > 1.1
    _check_against_numpy(cov, x)
