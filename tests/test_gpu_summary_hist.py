"""Posterior histograms of sample_summary(..., histogram=...) on the GPU against numpy on the raw draws of an identically seeded
sampler: the counts are integers, so they must equal numpy.histogram / numpy.histogram2d count for count; every key the summary
returns without a histogram keeps its bits, and the chains advance as sample(n) advances them."""
import numpy as np
import pytest

import models
from conftest import config2_data

pytestmark = pytest.mark.gpu
PROBS = (0.0, 0.025, 0.25, 0.5, 0.75, 0.975, 1.0)


def _bytes(v):
    return np.asarray(v).tobytes()


@pytest.mark.parametrize("diagnostics", [False, True, "rank"])
def test_config2_histograms_match_numpy_and_leave_the_summary_alone(gpu_pkg, diagnostics):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    a, b, c = (mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21}) for _ in range(3))
    for s in (a, b, c):
        s.burn(2500)
    raw = a.sample(50)
    got = b.sample_summary(50, PROBS, diagnostics=diagnostics, histogram={"bins": 40, "pairs": [("mu", "sigma")], "pair_bins": 32})
    base = c.sample_summary(50, PROBS, diagnostics=diagnostics)
    for name in ("mu", "sigma"):
        v = raw[name].ravel()
        h, ed = np.histogram(v[np.isfinite(v)], bins=40)
        assert got[name]["hist"].dtype == np.int64 and got[name]["hist"].shape == (40,)
        assert np.array_equal(got[name]["hist"], h), name
        assert np.array_equal(got[name]["hist_edges"], ed), name            # by value
        assert np.array_equal(got[name]["hist_outside"], [0, 0, 0])
        assert got[name]["hist"].sum() == got[name]["n_draws"] == v.size
        for key, val in base[name].items():
            assert _bytes(got[name][key]) == _bytes(val), (name, key)
    mu, sg = raw["mu"].ravel(), raw["sigma"].ravel()
    want, xe, ye = np.histogram2d(mu, sg, bins=32, range=[(mu.min(), mu.max()), (sg.min(), sg.max())])
    pair = got[("mu", "sigma")]
    assert np.array_equal(pair["hist"], want.astype(np.int64)) and pair["hist"].dtype == np.int64
    assert np.array_equal(pair["xedges"], xe) and np.array_equal(pair["yedges"], ye)
    assert set(got) == set(base) | {("mu", "sigma")}
    sa, sb = a.state, b.state
    assert np.array_equal(sa["mu"], sb["mu"]) and np.array_equal(sa["sigma"], sb["sigma"])


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


def test_multidim_int_thin_monitor_and_derived(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"mu": {"type": "real"}, "x": {"type": "int", "dim": [2, 3], "lower": 0, "init": [[3, 5, 8], [1, 12, 20]]}}
    mk = lambda: mcmc.AmwgSampler(pars, _int_model(ld), None, {"chains": 1000, "seed": 8, "thin": 3, "monitor": ["x", "var"]})
    a, b = mk(), mk()
    a.burn(300); b.burn(300)
    raw = a.sample(31)                                             # 11 kept rows
    x, var = raw["x"], raw["var"]
    assert x.shape == (11, 1000, 2, 3)
    lo, hi = int(x.min()), int(x.max())
    k = hi - lo + 1
    vlo, vhi = np.quantile(var, [0.2, 0.8])                        # a range that leaves draws on both sides
    got = b.sample_summary(31, (0.5,), histogram={"bins": k, "range": {"x": (lo - 0.5, hi + 0.5), "var": (vlo, vhi)},
                                                  "pairs": [(("x", 3), "var")]})
    assert set(got) == {"x", "var", (("x", 3), "var")}
    assert got["x"]["hist"].shape == (2, 3, k) and got["x"]["hist_edges"].shape == (2, 3, k + 1) and got["x"]["hist_outside"].shape == (2, 3, 3)
    for i in range(2):
        for j in range(3):
            v = x[:, :, i, j].ravel()
            h, ed = np.histogram(v, bins=k, range=(lo - 0.5, hi + 0.5))
            assert np.array_equal(got["x"]["hist"][i, j], h) and np.array_equal(got["x"]["hist_edges"][i, j], ed)
            assert np.array_equal(got["x"]["hist"][i, j], np.bincount((v - lo).astype(int), minlength=k))     # unit bins
            assert np.array_equal(got["x"]["hist_outside"][i, j], [0, 0, 0])
    v = var.ravel()
    h, ed = np.histogram(v, bins=k, range=(vlo, vhi))
    assert np.array_equal(got["var"]["hist"], h) and np.array_equal(got["var"]["hist_edges"], ed)
    assert np.array_equal(got["var"]["hist_outside"], [(v < vlo).sum(), (v > vhi).sum(), 0])
    assert got["var"]["hist"].sum() + got["var"]["hist_outside"].sum() == got["var"]["n_draws"] == v.size
    want, xe, ye = np.histogram2d(x[:, :, 1, 0].ravel(), v, bins=50, range=[(lo - 0.5, hi + 0.5), (vlo, vhi)])
    pair = got[(("x", 3), "var")]
    assert np.array_equal(pair["hist"], want.astype(np.int64)) and np.array_equal(pair["xedges"], xe) and np.array_equal(pair["yedges"], ye)
    assert np.array_equal(a.state["x"], b.state["x"]) and np.array_equal(a.state["mu"], b.state["mu"])


def _pool(lo, hi, ks, rng):
    """edges of every bin count in ks, 1 ulp to each side, both zeros, subnormals, infinities, NaN and values past both ends"""
    v = [np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, -1e-310, np.inf, -np.inf, np.nan, lo - 1, hi + 1, 1e300, -1e300])]
    for k in ks:
        ed = np.linspace(lo, hi, k + 1)
        v += [ed, np.nextafter(ed, np.inf), np.nextafter(ed, -np.inf)]
    v.append(rng.uniform(lo, hi, 200))
    return np.concatenate(v)


def test_c_abi_histograms_on_an_adversarial_block(gpu_pkg):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    rng = np.random.default_rng(12)
    red = CudaBlockReducer(0)
    L = gpu_pkg._ffi.lib()
    ranges = [(-1.0, 1.0), (184.2, 185.1), (6.75, 7.75), (0.0, 1.0), (-3e-310, 2e-310)]
    chains = 1000                                                       # ragged: not a multiple of 256
    for rows in (1, 13):
        for bins, pb in ((1, 128), (7, 1), (4096, 37)):
            x = np.empty((rows, 5, chains))
            for e, (lo, hi) in enumerate(ranges):
                x[:, e] = rng.choice(_pool(lo, hi, (bins, pb), rng), size=(rows, chains))
            x[:, 2] = 7.25                                              # constant
            x[:, 3] = rng.choice([np.nan, np.inf, -np.inf], size=(rows, chains))     # no finite draw
            x[0, 3, 0] = np.nan
            block = torch.from_numpy(x).to("cuda:0")
            r, nf = (t.cpu().numpy() for t in red.finite_range(block))
            for e in range(5):
                v = x[:, e].ravel()
                f = v[np.isfinite(v)]
                assert np.array_equal(r[e], (f.min(), f.max()) if f.size else (np.inf, -np.inf)), (rows, e)
                assert np.array_equal(nf[e], [(v == -np.inf).sum(), (v == np.inf).sum(), np.isnan(v).sum()])
            edges = np.stack([np.linspace(lo, hi, bins + 1) for lo, hi in ranges])
            c = red.histogram(block, edges, bins).cpu().numpy()
            for e, (lo, hi) in enumerate(ranges):
                v = x[:, e].ravel()
                assert np.array_equal(c[e, :bins], np.histogram(v[~np.isnan(v)], bins=bins, range=(lo, hi))[0]), (rows, bins, e)
                assert np.array_equal(c[e, bins:], [(v < lo).sum(), (v > hi).sum(), np.isnan(v).sum()]), (rows, bins, e)
                assert c[e].sum() == v.size
            pedges = np.stack([np.linspace(lo, hi, pb + 1) for lo, hi in ranges])
            pairs = np.array([(0, 1), (1, 0), (0, 0), (2, 4), (4, 3), (1, 4)], dtype=np.int32)
            c2 = red.histogram2d(block, pairs, pedges, pb).cpu().numpy()
            for i, (a, b) in enumerate(pairs):
                want = np.histogram2d(x[:, a].ravel(), x[:, b].ravel(), bins=[pedges[a], pedges[b]])[0]
                assert np.array_equal(c2[i], want.astype(np.int64)), (rows, pb, a, b)
    # argument checks come back as errors, not crashes
    p = block.data_ptr()
    pr = np.array([[0, 5]], dtype=np.int32)
    assert L.amwg_summary_histogram(0, p, rows, 5, chains, p, 0, p) != 0 and b"bins" in L.amwg_last_error()
    assert L.amwg_summary_histogram(0, p, rows, 5, chains, p, 4097, p) != 0
    assert L.amwg_summary_histogram2d(0, p, rows, 5, chains, pr.ctypes.data, 1, p, 129, p) != 0
    assert L.amwg_summary_histogram2d(0, p, rows, 5, chains, pr.ctypes.data, 1, p, 8, p) != 0 and b"outside" in L.amwg_last_error()
    assert L.amwg_summary_histogram2d(0, p, rows, 5, chains, pr.ctypes.data, 0, p, 8, p) != 0
    assert L.amwg_summary_finite_range(0, p, 0, 5, chains, p, p) != 0


def test_histograms_of_a_large_block(gpu_pkg):
    """2^19 chains: more chain groups than CTAs per entry, so every thread walks several chains"""
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    rows, chains = 64, 1 << 19
    g = torch.Generator(device="cuda:0").manual_seed(5)
    block = torch.randn((rows, 2, chains), generator=g, dtype=torch.float64, device="cuda:0")
    block[:, 0] = 184.5 + 0.14 * block[:, 0]
    block[:, 1] = torch.exp(block[:, 1])
    block[3, 1, ::1000] = float("nan")
    x = block.cpu().numpy()
    red = CudaBlockReducer(0)
    r = red.finite_range(block)[0].cpu().numpy()
    ranges = []
    for e in range(2):
        v = x[:, e].ravel()
        f = v[np.isfinite(v)]
        assert np.array_equal(r[e], (f.min(), f.max()))
        ranges.append((f.min(), f.max()))
    edges = np.stack([np.linspace(lo, hi, 51) for lo, hi in ranges])
    c = red.histogram(block, edges, 50).cpu().numpy()
    for e in range(2):
        v = x[:, e].ravel()
        assert np.array_equal(c[e, :50], np.histogram(v[np.isfinite(v)], bins=50)[0])
        assert np.array_equal(c[e, 50:], [0, 0, np.isnan(v).sum()])
    pedges = np.stack([np.linspace(lo, hi, 129) for lo, hi in ranges])
    c2 = red.histogram2d(block, np.array([[0, 1]], dtype=np.int32), pedges, 128).cpu().numpy()
    want = np.histogram2d(x[:, 0].ravel(), x[:, 1].ravel(), bins=128, range=ranges)[0]
    assert np.array_equal(c2[0], want.astype(np.int64))


def test_refused_histograms_leave_the_chains_alone(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    u, w = (mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 300, "seed": 3}) for _ in range(2))
    u.burn(50); w.burn(50)
    refused = [0, 4097, 2.5, True, {"bins": 0}, {"bins": 4097}, {"bins": 2.5}, {"bins": True}, {"bins": 5, "pair_bins": 129},
               {"bins": 5, "range": {"mu": (2.0, 1.0)}}, {"bins": 5, "range": {"mu": (1.0, 1.0)}}, {"bins": 5, "range": {"mu": (0.0, np.inf)}},
               {"bins": 5, "range": {"nope": (0.0, 1.0)}}, {"pairs": [("mu", "nope")]}, {"pairs": [(("mu", 1), "sigma")]}]
    for spec in refused:
        with pytest.raises(ValueError):
            u.sample_summary(20, histogram=spec)
    ru, rw = u.sample(20), w.sample(20)
    assert _bytes(ru["mu"]) == _bytes(rw["mu"]) and _bytes(ru["sigma"]) == _bytes(rw["sigma"])
