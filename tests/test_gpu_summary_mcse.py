"""Monte Carlo standard errors of the quantiles and of the sd (sample_summary(..., mcse=True)) on the GPU:
amwg_summary_indicator_autocov equal to direct counting (tests/mcse_ref.py) on adversarial blocks, past the chain grid, at 16
thresholds and at a 64-lag window past lag0 = 0, under a chain permutation and in two calls; every refusal; amwg_summary_autocov_sq
within rounding of its numpy restatement; sample_summary(mcse=True) on config 2 against the raw draws of a twin sampler, with
every other key and the chains' state unchanged; AR(1) known answers; and config 2 at 2^20 chains against a torch restatement."""
import numpy as np
import pytest

import mcse_ref
import models
from conftest import NORM_DATA, config2_data
from ess_ref import autocov_records

pytestmark = pytest.mark.gpu
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)
MCSE_KEYS = ("ess_quantile", "mcse_quantile", "mcse_sd")
CHAIN_GRID = 1184 * 256


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to("cuda:0")


def _reducer():
    from bayes_js_b200.summary import CudaBlockReducer
    return CudaBlockReducer(0)


def _block(rows, chains, seed):
    """[rows, 5, chains]: ties on a half grid, +-0, +-inf among normals, a constant, AR(0.8)-like"""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, 5, chains))
    x[:, 0] = np.round(2 * rng.normal(size=(rows, chains))) / 2
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.5, -0.0, 0.0)
    x[:, 2] = rng.normal(size=(rows, chains))
    x[1, 2, 0], x[rows - 1, 2, chains - 1], x[rows // 2, 2, 1] = np.inf, -np.inf, np.inf
    x[:, 3] = 7.25
    z = rng.normal(size=(rows, chains))
    for r in range(1, rows):
        z[r] = 0.8 * z[r - 1] + 0.6 * z[r]
    x[:, 4] = z
    return x


def _thresholds(x, K, seed):
    rng = np.random.default_rng(seed)
    thr = np.empty((x.shape[1], K))
    for e in range(x.shape[1]):
        v = x[:, e, :].ravel()
        pool = [v.min(), np.nextafter(v.min(), -np.inf), v.max(), 0.0, -0.0] + list(rng.choice(v, size=16))
        thr[e] = pool[:K]
    return thr


def _ind(red, blk, thr, lag0, n_lags):
    got = red.indicator_autocov(blk, thr, lag0, n_lags)
    assert np.array_equal(red.indicator_autocov(blk, thr, lag0, n_lags), got)
    return got


@pytest.mark.parametrize("rows, chains, K, windows", [
    (10, 300, 5, [(0, 5), (2, 3)]),
    (127, 1000, 16, [(0, 63), (1, 62), (62, 1)]),
    (130, 4096 + 77, 1, [(0, 64), (1, 64), (64, 1)]),
    (300, 513, 16, [(70, 64), (86, 64), (149, 1)]),                 # 64-lag windows past lag0 = 0: two reads
    (12, CHAIN_GRID + 77, 5, [(0, 6)]),                            # grid stride
    (4201, 300, 5, [(0, 64), (2000, 64)]),                         # h >= 2048: the edge terms' warp sums in three limbs
])
def test_c_abi_indicator_sums_equal_direct_counting(gpu_pkg, rows, chains, K, windows):
    x = _block(rows, chains, rows)
    thr = _thresholds(x, K, rows)
    blk = _dev(x)
    red = _reducer()
    perm = np.random.default_rng(1).permutation(chains)
    blk_p = _dev(x[:, :, perm])
    for lag0, n_lags in windows:
        got = _ind(red, blk, thr, lag0, n_lags)
        assert np.array_equal(got, mcse_ref.indicator_sums(x, thr, lag0, n_lags)), (rows, chains, lag0, n_lags)
        assert np.array_equal(_ind(red, blk_p, thr, lag0, n_lags), got)


def test_c_abi_refusals(gpu_pkg):
    L = gpu_pkg._ffi.lib()
    rows, entries, chains = 20, 2, 100
    blk = _dev(np.zeros((rows, entries, chains)))
    p = blk.data_ptr()
    thr = np.zeros((entries, 16))
    out = np.zeros(entries * 16 * 130, dtype=np.int64)
    before = out.copy()
    bad = [(1, 2, 0, 1, b"rows must be at least 2"), (rows, 0, 0, 1, b"n_thresholds must be 1..16"),
           (rows, 17, 0, 1, b"n_thresholds must be 1..16"), (rows, 2, 0, 0, b"n_lags must be 1..64"),
           (rows, 2, 0, 65, b"n_lags must be 1..64"), (rows, 2, 9, 2, b"lag window"), (rows, 2, -1, 2, b"lag window")]
    for r, K, l0, n, msg in bad:
        assert L.amwg_summary_indicator_autocov(0, p, r, entries, chains, thr.ctypes.data, K, l0, n, out.ctypes.data) != 0
        err = L.amwg_last_error()
        assert err.startswith(b"amwg_summary_indicator_autocov: ") and msg in err, err
    for args in [(0, None, rows, entries, chains, thr.ctypes.data, 2, 0, 2, out.ctypes.data),
                 (0, p, rows, entries, chains, None, 2, 0, 2, out.ctypes.data),
                 (0, p, rows, entries, chains, thr.ctypes.data, 2, 0, 2, None)]:
        assert L.amwg_summary_indicator_autocov(*args) != 0
        assert L.amwg_last_error() == b"amwg_summary_indicator_autocov: null pointer"
    assert L.amwg_summary_indicator_autocov(9999, p, rows, entries, chains, thr.ctypes.data, 2, 0, 2, out.ctypes.data) != 0
    assert L.amwg_last_error().startswith(b"amwg_summary_indicator_autocov")
    assert L.amwg_summary_indicator_autocov(0, p, rows, 0, chains, thr.ctypes.data, 2, 0, 2, out.ctypes.data) != 0
    assert np.array_equal(out, before)
    c = np.zeros(entries)
    rec = np.zeros(entries * 40)
    assert L.amwg_summary_autocov_sq(0, p, rows, entries, chains, None, c.ctypes.data, 0, 2, rec.ctypes.data) != 0
    assert L.amwg_last_error() == b"amwg_summary_autocov_sq: null pointer"
    assert L.amwg_summary_autocov_sq(0, p, rows, entries, chains, c.ctypes.data, c.ctypes.data, 0, 33, rec.ctypes.data) != 0
    assert L.amwg_last_error().startswith(b"amwg_summary_autocov_sq: n_lags")


@pytest.mark.parametrize("rows, chains, windows", [(23, CHAIN_GRID + 77, [(0, 11), (3, 7)]), (71, 1000, [(0, 32), (19, 16)])])
def test_c_abi_autocov_sq_within_rounding(gpu_pkg, rows, chains, windows):
    x = np.ascontiguousarray(_block(rows, chains, rows + 1)[:, [0, 1, 3, 4]])      # ties, +-0, a constant, AR: all finite
    centre = x.mean(axis=(0, 2))
    scale = np.array([2.0, 0.5, 1.0, 1.0])
    red = _reducer()
    blk = _dev(x)
    y = ((x - centre[None, :, None]) * scale[None, :, None]) ** 2
    for lag0, n_lags in windows:
        got = red.autocov_sq(blk, centre, scale, lag0, n_lags)
        assert red.autocov_sq(blk, centre, scale, lag0, n_lags).tobytes() == got.tobytes()
        want = autocov_records(y, None, lag0, n_lags)
        assert np.array_equal(got[:, :, 0], want[:, :, 0])
        sc = np.maximum(np.abs(want[:, :, 3:4]), 1e-300)
        assert np.allclose(got[:, :, 1:3], want[:, :, 1:3], rtol=1e-11, atol=1e-300)
        assert np.allclose(got[:, :, 3:], want[:, :, 3:], rtol=0, atol=1e-11 * sc)


def _flat(raw, name):
    x = raw[name]                                              # [rows, chains, *dim]
    return np.moveaxis(x.reshape(x.shape[0], x.shape[1], -1), 2, 1)


def _check(summ, raw, name, probs):
    x = _flat(raw, name)
    dim = raw[name].shape[2:]
    q = np.asarray(summ[name]["quantiles"]).reshape(len(probs), -1)
    mean = np.atleast_1d(np.asarray(summ[name]["mean"])).ravel()
    sd = np.atleast_1d(np.asarray(summ[name]["sd"])).ravel()
    ess = mcse_ref.ess_quantile(x, q)
    mq = mcse_ref.mcse_quantile(x, probs, ess)
    msd = mcse_ref.mcse_sd(x, mean, sd)
    got_ess = np.asarray(summ[name]["ess_quantile"]).reshape(len(probs), -1)
    got_mq = np.asarray(summ[name]["mcse_quantile"]).reshape(len(probs), -1)
    assert got_ess.tobytes() == ess.tobytes(), (name, got_ess, ess)
    assert got_mq.tobytes() == mq.tobytes(), (name, got_mq, mq)
    assert np.allclose(np.atleast_1d(summ[name]["mcse_sd"]).ravel(), msd, rtol=1e-10, atol=0, equal_nan=True), name
    assert np.asarray(summ[name]["ess_quantile"]).shape == (len(probs),) + tuple(dim if dim else ())


def _same(a, b, drop=MCSE_KEYS):
    assert set(a) == set(b)
    for name in a:
        if not isinstance(a[name], dict):
            continue
        ka = {k for k in a[name] if k not in drop}
        assert ka == {k for k in b[name] if k not in drop}
        for k in ka:
            va, vb = a[name][k], b[name][k]
            if isinstance(va, dict):
                continue
            assert np.atleast_1d(np.asarray(va)).tobytes() == np.atleast_1d(np.asarray(vb)).tobytes(), (name, k)


def test_mcse_matches_the_raw_draws_config2_shape(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    mk = lambda: mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21})
    a, b = mk(), mk()
    for s in (a, b):
        s.burn(1000)
    raw = a.sample(100)
    summ = b.sample_summary(100, PROBS, mcse=True)
    for name in ("mu", "sigma"):
        _check(summ, raw, name, PROBS)
        assert np.all(summ[name]["mcse_quantile"] > 0) and summ[name]["mcse_sd"] > 0
    assert np.array_equal(a.sample(10)["mu"], b.sample(10)["mu"])


@pytest.mark.parametrize("diagnostics", [False, True, "rank"])
def test_every_other_key_keeps_its_bits(gpu_pkg, diagnostics):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    mk = lambda: mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 1024, "seed": 3})
    a, b = mk(), mk()
    for s in (a, b):
        s.burn(300)
    kw = dict(diagnostics=diagnostics, histogram={"bins": 20, "pairs": [("mu", "sigma")]}, covariance=True)
    plain = a.sample_summary(40, PROBS, **kw)
    with_mcse = b.sample_summary(40, PROBS, mcse=True, **kw)
    _same(plain, with_mcse)
    assert all(k in with_mcse["mu"] for k in MCSE_KEYS)
    sa, sb = a.sample(10), b.sample(10)
    assert np.array_equal(sa["mu"], sb["mu"]) and np.array_equal(sa["sigma"], sb["sigma"])


def test_mcse_with_thin_monitor_multidim_int_and_derived(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"x": {"type": "int", "dim": [2, 2], "lower": 0, "init": [[1, 10], [100, 1000]]}}
    mk = lambda: mcmc.AmwgSampler(pars, models.multivar_poisson_dens(ld), None, {"chains": 300, "seed": 5, "thin": 3})
    a, b = mk(), mk()
    for s in (a, b):
        s.burn(300)
    probs = (0.1, 0.5, 0.9)
    raw, summ = a.sample(61), b.sample_summary(61, probs, mcse=True)
    assert summ["x"]["mcse_quantile"].shape == (3, 2, 2) and summ["x"]["mcse_sd"].shape == (2, 2)
    _check(summ, raw, "x", probs)
    pars = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    mk = lambda: mcmc.AmwgSampler(pars, models.norm_post_test(ld), NORM_DATA, {"chains": 257, "seed": 6, "monitor": ["var", "mu"]})
    a, b = mk(), mk()
    for s in (a, b):
        s.burn(200)
    raw, summ = a.sample(40), b.sample_summary(40, PROBS, mcse=True)
    for name in ("var", "mu"):
        _check(summ, raw, name, PROBS)
    short = b.sample_summary(9, mcse=True)
    assert all(np.all(np.isnan(short["mu"][k])) for k in MCSE_KEYS)
    with pytest.raises(ValueError, match="mcse must be True or False"):
        b.sample_summary(20, mcse=1)


# ---- known answers ------------------------------------------------------------------------------------------------------------
# S' = M h = 2^14 chains x 1000 rows = 1.6e7 split draws; an ESS of S'/tau is estimated with a relative sd of about
# sqrt(2 (2 L + 1) / S') (L: the lags Geyer's sum runs over, < 100 here) < 0.5 %, and the 1000-row chains leave a truncation bias
# of phi^L; mcse_quantile at 1e8 iid draws rests on about 2 sqrt(S p (1 - p)) >= 4000 order statistics between its two ranks,
# a relative sd of 1.5 % or less at the probabilities below. 5 % is 3 sd or more of each.
def _ar1_device(phi, rows, chains, seed):
    import torch
    g = torch.Generator(device="cuda:0").manual_seed(seed)
    x = torch.empty((rows, 1, chains), dtype=torch.float64, device="cuda:0")
    x[0] = torch.randn((1, chains), generator=g, dtype=torch.float64, device="cuda:0") / np.sqrt(1 - phi * phi)
    for r in range(1, rows):
        x[r] = phi * x[r - 1] + torch.randn((1, chains), generator=g, dtype=torch.float64, device="cuda:0")
    return x


def _run(block, probs):
    from bayes_js_b200.summary import mcse_block, summarise_block
    rows, _, chains = block.shape
    red = _reducer()
    mean, sd, _, q = summarise_block(red, block, rows, chains, probs, False)
    return mcse_block(red, block, rows, chains, probs, mean, sd, q, False), sd


def _tau_indicator(phi, p, L=400):
    from scipy.stats import multivariate_normal, norm
    z = norm.ppf(p)
    rho = []
    for t in range(1, L):
        r = phi ** t
        if r < 1e-9:
            break
        c = multivariate_normal(mean=[0, 0], cov=[[1, r], [r, 1]]).cdf([z, z])
        rho.append((c - p * p) / (p * (1 - p)))
    return 1 + 2 * sum(rho)


@pytest.mark.parametrize("phi", [0.0, 0.5, 0.9])
def test_ar1_known_answers(gpu_pkg, phi):
    rows, chains = 1000, 1 << 14
    block = _ar1_device(phi, rows, chains, 11)
    out, sd = _run(block, (0.05, 0.5))
    Sp = 2 * chains * (rows // 2)
    tau_med = 1 + 2 * sum((2 / np.pi) * np.arcsin(phi ** t) for t in range(1, 2000))
    assert abs(out["ess_quantile"][1, 0] * tau_med / Sp - 1) < 0.05, (phi, out["ess_quantile"][1, 0], Sp / tau_med)
    tau05 = _tau_indicator(phi, 0.05)
    assert abs(out["ess_quantile"][0, 0] * tau05 / Sp - 1) < 0.05, (phi, out["ess_quantile"][0, 0], Sp / tau05)
    sigma = np.sqrt(1 / (1 - phi * phi))
    ess_y = Sp * (1 - phi * phi) / (1 + phi * phi)
    want = sigma / np.sqrt(2 * ess_y)
    assert abs(out["mcse_sd"][0] / want - 1) < 0.05, (phi, out["mcse_sd"][0], want)


def test_iid_mcse_quantile_known_answer(gpu_pkg):
    import torch
    from scipy.stats import norm
    rows, chains = 100, 1 << 20
    g = torch.Generator(device="cuda:0").manual_seed(5)
    block = torch.randn((rows, 1, chains), generator=g, dtype=torch.float64, device="cuda:0")
    probs = (0.05, 0.25, 0.5, 0.9)
    out, _ = _run(block, probs)
    S = rows * chains
    for i, p in enumerate(probs):
        want = np.sqrt(p * (1 - p) / S) / norm.pdf(norm.ppf(p))
        assert abs(out["mcse_quantile"][i, 0] / want - 1) < 0.05, (p, out["mcse_quantile"][i, 0], want)


# ---- full scale -----------------------------------------------------------------------------------------------------------------
def test_config2_full_scale_against_torch(gpu_pkg, monkeypatch):
    """config 2 at 2^20 chains x 100 rows: the indicator sums of the first window equal comparisons and sums formed by torch on
    the same block, and mcse_quantile equals the order statistics torch.kthvalue gives at the same ranks"""
    import torch
    import bayes_js_b200.summary as summ_mod
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    seen = {}

    class Capture(summ_mod.CudaBlockReducer):
        def indicator_autocov(self, block, thresholds, lag0, n_lags):
            out = super().indicator_autocov(block, thresholds, lag0, n_lags)
            seen.setdefault("calls", []).append((block, np.array(thresholds), lag0, n_lags, out))
            return out

    monkeypatch.setattr(summ_mod, "CudaBlockReducer", Capture)
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    s = mcmc.AmwgSampler(params, models.norm_post_readme(ld), config2_data().tolist(), {"chains": 1 << 20, "seed": 2})
    s.burn(1000)
    res = s.sample_summary(100, PROBS, mcse=True)
    block, thr, lag0, n_lags, got = seen["calls"][0]
    rows, entries, chains = block.shape
    h = rows // 2
    assert lag0 == 0 and n_lags == h
    for e in range(entries):
        xe = block[:, e, :]
        for k in range(thr.shape[1]):
            b = torch.cat([xe[:h], xe[rows - h:]], dim=1).T <= float(thr[e, k])      # [M, h]
            bi = b.to(torch.int64)
            c = bi.sum(dim=1)
            want = [int(c.sum()), int((c * c).sum())]
            P, G = [], []
            for t in range(n_lags):
                P.append(int((bi[:, :h - t] * bi[:, t:]).sum()))
                F = bi[:, :t].sum(dim=1)
                L = bi[:, h - t:].sum(dim=1) if t else torch.zeros_like(c)
                G.append(int((c * (F + L)).sum()))
            assert got[e, k].tolist() == want + P + G, (e, k)
    S = rows * chains
    from bayes_js_b200.summary import quantile_mcse_ranks
    for e, name in enumerate(("mu", "sigma")):
        ess = np.asarray(res[name]["ess_quantile"])[:, None]
        i1, i2, bad = quantile_mcse_ranks(ess, PROBS, S)
        assert not bad.any()
        flat = block[:, e, :].reshape(-1)
        for i in range(len(PROBS)):
            lo = float(torch.kthvalue(flat, int(i1[i, 0]) + 1).values)
            hi = float(torch.kthvalue(flat, int(i2[i, 0]) + 1).values)
            assert res[name]["mcse_quantile"][i] == (hi - lo) / 2, (name, i)
