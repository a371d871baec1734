"""Rank-normalised diagnostics of the on-device summary (diagnostics="rank"): the radix sort, merge-path rank counts and z
scatter entries against numpy, sample_summary(..., diagnostics="rank") against the scipy restatement applied to the raw draws
of an identically seeded sampler, and Vehtari et al.'s motivating cases on blocks uploaded to the device."""
import numpy as np
import pytest

import models
from conftest import NORM_DATA, config2_data
from rank_ref import canonical_keys, half_draws, rank_diagnostics_ref
from scipy.special import ndtri

pytestmark = pytest.mark.gpu
KEYS = ("ess_bulk", "rhat_rank")
TRUE_KEYS = ("ess_mean", "ess_tail", "mcse_mean", "rhat_split")
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)
DEV = 0


def _sort(block, entry, centre=np.nan):
    """-> (sorted keys uint64, indices, passes) of the device sort, and the canonical keys numpy computes."""
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    rows, _, chains = block.shape
    n = 2 * (rows // 2) * chains
    keys = torch.empty(2 * n, dtype=torch.int64, device=block.device)
    index = torch.empty(2 * n, dtype=torch.int32, device=block.device)
    passes = CudaBlockReducer(DEV).rank_sort(block, entry, centre, keys, index)
    v = half_draws(block[:, entry, :].cpu().numpy()).ravel()
    if not np.isnan(centre):
        v = np.abs(v - centre)
    return keys[:n].cpu().numpy().view(np.uint64), index[:n].cpu().numpy().view(np.uint32), passes, canonical_keys(v)


def _bits(rng, shape):
    """full-range bit patterns (NaNs replaced), with -0, +0, -inf and +inf mixed in: every byte varies, no pass is skipped"""
    u = rng.integers(0, 2 ** 63, size=shape, dtype=np.int64).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, size=shape).astype(np.uint64)
    x = u.view(np.float64).copy()
    x[np.isnan(x)] = 1.5
    flat = x.reshape(-1)
    flat[rng.choice(flat.size, 40, replace=False)] = np.repeat([-0.0, 0.0, -np.inf, np.inf], 10)
    return x


SORT_CASES = [
    ("narrow", 21, 4097),               # S not a multiple of any tile; config-2-like draws share their top bytes
    ("bits", 10, 3001),                 # full-range patterns with negatives, +-0 and +-inf: all eight passes
    ("constant", 12, 777),              # all keys equal: every pass skipped
    ("large", 20, 1 << 20),             # S > 2^24
]


@pytest.mark.parametrize("case,rows,chains", SORT_CASES)
def test_sort_entry_equals_numpy_sort(gpu_pkg, case, rows, chains):
    import torch
    rng = np.random.default_rng(rows + chains)
    if case == "bits":
        x = _bits(rng, (rows, 2, chains))
    elif case == "constant":
        x = np.full((rows, 2, chains), -3.5)
    else:
        x = 184.5 + 0.14 * rng.normal(size=(rows, 2, chains))
    block = torch.from_numpy(x).to(torch.device("cuda", DEV))
    for entry, centre in ((1, np.nan), (1, float(np.median(x[:, 1])))):
        got, idx, passes, want = _sort(block, entry, centre)
        assert np.array_equal(got, np.sort(want)), (case, entry, centre)
        assert np.array_equal(np.sort(idx), np.arange(want.size)), "indices are not a permutation"
        assert np.array_equal(want[idx], got), "indices do not reproduce the sorted keys"
        assert np.array_equal(idx, np.argsort(want, kind="stable")), "ties are not in index order"
        varying = sum(1 for d in range(8) if np.unique((want >> np.uint64(8 * d)) & np.uint64(255)).size > 1)
        assert passes == varying
        if case == "bits" and np.isnan(centre):
            assert passes == 8
        if case == "constant":
            assert passes == 0
        if case in ("narrow", "large") and np.isnan(centre):
            assert passes < 8
    again = _sort(block, 1)
    first = _sort(block, 1)
    assert np.array_equal(again[0], first[0]) and np.array_equal(again[1], first[1])


def _count(q, r):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    dev = torch.device("cuda", DEV)
    tq = torch.from_numpy(q.view(np.int64).copy()).to(dev)
    tr = torch.from_numpy(r.view(np.int64).copy()).to(dev)
    acc = torch.full((q.size,), 7, dtype=torch.int64, device=dev)        # the entry adds to what is there
    CudaBlockReducer(DEV).rank_count(tq, q.size, tr, r.size, acc)
    return acc.cpu().numpy() - 7


def test_count_entry_equals_searchsorted(gpu_pkg):
    rng = np.random.default_rng(5)
    q = np.sort(canonical_keys(rng.normal(size=300_001)))
    cases = {
        "self": q,
        "disjoint": np.sort(canonical_keys(rng.normal(size=70_000) + 100.0)),
        "interleaved": np.sort(np.concatenate([q[::3], canonical_keys(rng.normal(size=123_457))])),
        "one": q[150_000:150_001].copy(),
    }
    for name, r in cases.items():
        want = np.searchsorted(r, q, "left") + np.searchsorted(r, q, "right")
        assert np.array_equal(_count(q, r), want), name
    b = np.sort(canonical_keys(np.repeat([0.0, 1.0], 5_000_000)))    # a binary parameter: two tie groups of 5e6
    assert np.array_equal(_count(b, b), np.repeat([5_000_000, 15_000_000], 5_000_000))


def test_z_entry_is_within_8_ulp_and_deterministic(gpu_pkg):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer
    rng = np.random.default_rng(6)
    rows, chains = 30, 5001
    x = np.round(rng.normal(size=(rows, 1, chains)), 2)                  # ties
    dev = torch.device("cuda", DEV)
    block = torch.from_numpy(x).to(dev)
    red = CudaBlockReducer(DEV)
    n = 2 * (rows // 2) * chains
    keys = torch.empty(2 * n, dtype=torch.int64, device=dev)
    index = torch.empty(2 * n, dtype=torch.int32, device=dev)
    acc = torch.zeros(n, dtype=torch.int64, device=dev)
    red.rank_sort(block, 0, float("nan"), keys, index)
    red.rank_count(keys, n, keys, n, acc)
    zs = []
    for _ in range(2):
        z = torch.empty((2 * (rows // 2), 1, chains), dtype=torch.float64, device=dev)
        red.rank_z(acc, index, n, n, z)
        zs.append(z.cpu().numpy())
    assert zs[0].tobytes() == zs[1].tobytes()
    from scipy.stats import rankdata
    hd = half_draws(x[:, 0])
    want = ndtri((rankdata(hd.ravel(), method="average") - 0.375) / (n + 0.25)).reshape(hd.shape)
    ulp = np.spacing(np.abs(want))
    assert np.all(np.abs(zs[0][:, 0, :] - want) <= 8 * ulp)


def test_bad_arguments_name_the_entry(gpu_pkg):
    import torch
    L = gpu_pkg._ffi.lib()
    dev = torch.device("cuda", DEV)
    block = torch.zeros((10, 2, 16), dtype=torch.float64, device=dev)
    keys = torch.zeros(320, dtype=torch.int64, device=dev)
    index = torch.zeros(320, dtype=torch.int32, device=dev)
    acc = torch.zeros(160, dtype=torch.int64, device=dev)
    z = torch.zeros(160, dtype=torch.float64, device=dev)
    p, k, i, a, zp = block.data_ptr(), keys.data_ptr(), index.data_ptr(), acc.data_ptr(), z.data_ptr()
    nan = float("nan")
    sort_bad = [(0, p, 1, 2, 16, 0), (0, p, 10, 2, 16, 2), (0, p, 10, 2, 16, -1), (0, p, 10, 0, 16, 0), (0, None, 10, 2, 16, 0),
                (-1, p, 10, 2, 16, 0), (0, p, 2, 1, 1 << 31, 0)]
    for dv, bp, rows, entries, chains, e in sort_bad:
        assert L.amwg_summary_rank_sort(dv, bp, rows, entries, chains, e, nan, k, i, None) != 0
        assert L.amwg_last_error().startswith(b"amwg_summary_rank_sort"), L.amwg_last_error()
    assert L.amwg_summary_rank_sort(0, p, 10, 2, 16, 0, nan, None, i, None) != 0 and b"null" in L.amwg_last_error()
    assert L.amwg_summary_rank_sort(0, p, 2, 1, 1 << 31, 0, nan, k, i, None) != 0 and b"2^32" in L.amwg_last_error()
    for args in [(0, k, 0, k, 5, a), (0, k, 5, k, 0, a), (0, None, 5, k, 5, a), (0, k, 5, k, 5, None), (0, k, 1 << 32, k, 5, a), (99, k, 5, k, 5, a)]:
        assert L.amwg_summary_rank_count(*args) != 0
        assert L.amwg_last_error().startswith(b"amwg_summary_rank_count"), L.amwg_last_error()
    for args in [(0, a, i, 0, 5, zp), (0, a, i, 10, 5, zp), (0, None, i, 5, 5, zp), (0, a, i, 5, 5, None), (0, a, i, 1 << 32, 1 << 33, zp)]:
        assert L.amwg_summary_rank_z(*args) != 0
        assert L.amwg_last_error().startswith(b"amwg_summary_rank_z"), L.amwg_last_error()


def _check(summ, raw, name):
    x = raw[name]                                              # [rows, chains, *dim]
    dim = x.shape[2:]
    flat = np.moveaxis(x.reshape(x.shape[0], x.shape[1], -1), 2, 1)
    want = rank_diagnostics_ref(flat)
    shape = (lambda a: a.reshape(dim)) if dim else (lambda a: a[0])
    for k in KEYS:
        assert np.allclose(summ[name][k], shape(want[k]), rtol=1e-9, atol=0, equal_nan=True), (name, k, summ[name][k], want[k])


def _same(a, b):
    assert set(a) == set(b)
    for name in a:
        assert set(a[name]) == set(b[name])
        for k in a[name]:
            assert np.atleast_1d(np.asarray(a[name][k])).tobytes() == np.atleast_1d(np.asarray(b[name][k])).tobytes(), (name, k)


def _without_rank(summ):
    return {n: {k: v for k, v in d.items() if k not in KEYS} for n, d in summ.items()}


def test_rank_matches_the_raw_draws_config2_shape(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data().tolist()
    mk = lambda: mcmc.AmwgSampler(params, models.norm_post_readme(ld), data, {"chains": 4096, "seed": 21})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(1000)
    raw = a.sample(100)
    summ = b.sample_summary(100, PROBS, diagnostics="rank")
    true = c.sample_summary(100, PROBS, diagnostics=True)
    for name in ("mu", "sigma"):
        _check(summ, raw, name)
        assert summ[name]["ess_bulk"] > 0 and summ[name]["rhat_rank"] < 1.5
    _same(true, _without_rank(summ))
    for name in ("mu", "sigma"):
        assert np.array_equal(a.state[name], b.state[name]) and np.array_equal(a.state[name], c.state[name])
    with pytest.raises(ValueError, match="diagnostics"):
        b.sample_summary(20, diagnostics="bulk")


def test_rank_with_thin_int_multidim_and_derived(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    pars = {"x": {"type": "int", "dim": [2, 2], "lower": 0, "init": [[1, 10], [100, 1000]]}}
    mk = lambda: mcmc.AmwgSampler(pars, models.multivar_poisson_dens(ld), None, {"chains": 300, "seed": 5, "thin": 3})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(300)
    raw, summ, true = a.sample(61), b.sample_summary(61, (0.1, 0.5, 0.9), diagnostics="rank"), c.sample_summary(61, (0.1, 0.5, 0.9), diagnostics=True)
    assert raw["x"].shape == (21, 300, 2, 2) and summ["x"]["ess_bulk"].shape == (2, 2)
    _check(summ, raw, "x")
    _same(true, _without_rank(summ))
    assert np.array_equal(a.state["x"], b.state["x"]) and np.array_equal(a.state["x"], c.state["x"])
    pars = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    mk = lambda: mcmc.AmwgSampler(pars, models.norm_post_test(ld), NORM_DATA, {"chains": 257, "seed": 6, "monitor": ["var", "mu"]})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(200)
    raw, summ, true = a.sample(40), b.sample_summary(40, diagnostics="rank"), c.sample_summary(40, diagnostics=True)
    assert set(summ) == {"var", "mu"}
    for name in ("var", "mu"):
        _check(summ, raw, name)
    _same(true, _without_rank(summ))
    short = b.sample_summary(9, diagnostics="rank")            # fewer than 10 kept rows: NaN
    assert all(np.isnan(short["mu"][k]) for k in KEYS)


def _on_device(x):
    import torch
    from bayes_js_b200.summary import CudaBlockReducer, summarise_block
    block = torch.from_numpy(np.ascontiguousarray(x)).to(torch.device("cuda", DEV))
    rows, _, chains = x.shape
    *_, (diag, _) = summarise_block(CudaBlockReducer(DEV), block, rows, chains, PROBS, False, diagnostics="rank")
    return diag


def test_vehtari_cases_and_infinite_draws_on_the_device(gpu_pkg):
    rng = np.random.default_rng(12)
    rows, chains = 400, 64
    scale = rng.normal(size=(rows, 1, chains)) * np.where(np.arange(chains) < chains // 2, 1.0, 3.0)
    d = _on_device(scale)
    assert d["rhat_split"][0] < 1.01 and d["rhat_rank"][0] > 1.1
    shift = rng.normal(size=(rows, 1, chains)) + np.where(np.arange(chains) < chains // 2, 0.0, 2.0)
    d2 = _on_device(shift)
    assert d2["rhat_split"][0] > 1.1 and d2["rhat_rank"][0] > 1.1
    heavy = rng.standard_cauchy(size=(201, 3, 500))
    heavy[17, 0, 3] = np.inf
    heavy[4, 1, 9] = -np.inf
    heavy[:, 2] = np.where(rng.random((201, 500)) < 0.1, -0.0, np.round(heavy[:, 2]))
    heavy[9, 2, 2] = 0.0
    d3 = _on_device(heavy)
    assert np.isnan(d3["ess_mean"][0]) and np.isnan(d3["ess_mean"][1])
    assert np.all(np.isfinite(d3["ess_bulk"])) and np.all(np.isfinite(d3["rhat_rank"]))
    for x, d in ((scale, d), (shift, d2), (heavy, d3)):
        want = rank_diagnostics_ref(x)
        for k in KEYS:
            assert np.allclose(d[k], want[k], rtol=1e-9, atol=0, equal_nan=True), (k, d[k], want[k])
