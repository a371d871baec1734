"""The two base reductions of sample_summary on the GPU, held to exact references at the shapes and values where reductions go
wrong: amwg_summary_moments against the fsum restatement within its worst-case bound (tests/moments_ref.py), and the radix select
of amwg_summary_digit_hist by bits against the sorted order-preserving keys. Then NaN and infinite draws of derived quantities
through sample_summary, against numpy on the raw draws of an identically seeded handle."""
import numpy as np
import pytest

import moments_ref
from summary_ref import numpy_summary

pytestmark = pytest.mark.gpu
GRID = 1184 * 256                      # the chain-wise kernels' CTAs x threads: more chains than this and a thread walks two


def _block(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


def _moment_entries(rows, chains, seed):
    """[rows, 6, chains]: cancellation, config 2's mu, integers with ties and both zeros, values of about 1e150, subnormals
    (large ones: see moments_ref), a constant"""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, 6, chains))
    x[:, 0] = 1e6 + 1e-3 * rng.normal(size=(rows, chains))
    x[:, 1] = 184.5 + 0.14 * rng.normal(size=(rows, chains))
    x[:, 2] = np.round(3 * rng.normal(size=(rows, chains)))
    x[:, 2][x[:, 2] == 0] = np.where(rng.random(int((x[:, 2] == 0).sum())) < 0.5, -0.0, 0.0)
    x[:, 3] = 1e150 * (1 + 0.01 * rng.normal(size=(rows, chains)))
    x[:, 4] = 2.0 ** -1023 * (1 + rng.random((rows, chains)))
    x[:, 5] = -7.25
    return x


@pytest.mark.parametrize("rows, chains", [(1, 1), (1, 257), (7, 1), (8, 255), (9, 256), (13, 1001), (100, 4099), (3, GRID + 77),
                                          (2, 2 ** 20 + 3)])
def test_moments_within_the_worst_case_bound(gpu_pkg, rows, chains):
    from bayes_js_b200.summary import CudaBlockReducer
    x = _moment_entries(rows, chains, rows * 7 + chains)
    red = CudaBlockReducer(0)
    blk = _block(x)
    got = red.moments(blk)
    moments_ref.check_record(got, x, (rows, chains))
    assert red.moments(blk).tobytes() == got.tobytes()                  # the merge order is fixed: the same bits on every call
    assert got[5, 1] == -7.25 and got[5, 2] == 0 and got[5, 3] == 0      # a constant: both M2 exactly 0
    if rows == 1:
        assert np.all(got[:, 3] == 0)


# ---- the radix select, by bits ----------------------------------------------------------------------------------------------
def _select_block(kind):
    rng = np.random.default_rng(17)
    if kind == "grid-stride":                     # config 2's mu and integers with both zeros, a thread walks two chains
        rows, chains = 3, GRID + 77
        x = np.empty((rows, 2, chains))
        x[:, 0] = 184.5 + 0.14 * rng.normal(size=(rows, chains))
        x[:, 1] = np.round(2 * rng.normal(size=(rows, chains)))
        x[0, 1, ::7] = -0.0
        return x
    if kind == "ulps-and-decades":                # 1 + k ulp share their top seven bytes (they part in pass 7); 600 decades part in pass 0
        rows, chains = 5, 1000
        x = np.empty((rows, 2, chains))
        x[:, 0] = 1.0 + rng.integers(0, 256, (rows, chains)) * 2.0 ** -52
        x[:, 1] = 10.0 ** rng.uniform(-300, 300, (rows, chains)) * np.where(rng.random((rows, chains)) < 0.5, -1.0, 1.0)
        return x
    # subnormals with both zeros, both infinities and NaN of both signs; a normal entry with both zeros and infinities, half of
    # it +0; a plain normal entry
    rows, chains = 7, 333
    n = rows * chains
    specials = np.array([0.0, -0.0, 5e-324, -5e-324, np.inf, -np.inf, np.nan, np.uint64(0xFFF8000000000000).view(np.float64),
                         np.uint64(0x7FF0000000000123).view(np.float64), np.uint64(0xFFF00000000000FF).view(np.float64)])
    sub = rng.normal(size=n) * 1e-310
    sub[rng.integers(0, n, 600)] = rng.choice(specials, 600)
    mixed = rng.normal(size=n)
    mixed[:n // 2] = 0.0
    mixed[rng.integers(0, n, 40)] = rng.choice(specials[:6], 40)
    return np.stack([sub, mixed, rng.normal(size=n)]).reshape(3, rows, chains).transpose(1, 0, 2).copy()


def _grid(kind, M):
    if kind == "linspace41":                      # three selects: 16 + 16 + 9 probabilities
        return list(np.linspace(0, 1, 41))
    if kind == "distinct32":                      # 16 probabilities between two ranks each: 32 distinct order statistics
        lo = np.floor(np.linspace(0.05, 0.95, 16) * (M - 1))
        return list((lo + 0.5) / (M - 1))
    return list(0.5 + np.arange(16) * 1e-7)       # targets packed round the median: many share one prefix


@pytest.mark.parametrize("block_kind", ["grid-stride", "ulps-and-decades", "specials"])
def test_radix_select_by_bits(gpu_pkg, block_kind):
    """RadixSelect over the device's digit counts gives the order statistics of the sorted uint64 keys bit for bit (keys put -0
    below +0 and a NaN below -inf or above +inf by its sign, so the ranks are well defined); sample_summary's quantiles of the
    same block equal numpy.quantile's"""
    from bayes_js_b200.summary import MAX_PREFIXES, CudaBlockReducer, RadixSelect, double_to_key, quantile_targets, summarise_block
    x = _select_block(block_kind)
    rows, entries, chains = x.shape
    M = rows * chains
    red = CudaBlockReducer(0)
    blk = _block(x)
    flat = np.moveaxis(x, 1, 0).reshape(entries, -1)
    keys = np.sort(double_to_key(flat), axis=1)
    nonfinite = ~np.isfinite(flat).all(axis=1)
    for grid in ("linspace41", "distinct32", "shared"):
        probs = _grid(grid, M)
        full, padded = False, False
        for first in range(0, len(probs), MAX_PREFIXES // 2):
            ranks, _ = quantile_targets(M, probs[first:first + MAX_PREFIXES // 2])
            sel = RadixSelect(entries, ranks)
            for npass in range(8):
                table, which = sel.prefixes()
                n_uniq = [len(np.unique(t)) for t in table]
                full |= table.shape[1] == MAX_PREFIXES and MAX_PREFIXES in n_uniq
                padded |= min(n_uniq) < table.shape[1]
                sel.advance(red.digit_counts(blk, npass, table).cpu().numpy(), which)
            assert np.array_equal(sel.prefix, keys[:, ranks]), (grid, first)
        if grid == "distinct32":
            assert full                           # n_prefix = 32, an entry with 32 distinct prefixes: no padding in its row
        if grid == "shared":
            assert padded                         # an entry with fewer distinct prefixes than another: padded repeats
        with np.errstate(invalid="ignore"):
            mean, _sd, _rhat, q = summarise_block(red, blk, rows, chains, probs, False)
            want_q, want_mean = np.quantile(flat, probs, axis=1), flat[nonfinite].mean(axis=1)
        assert np.array_equal(q, want_q, equal_nan=True), grid
        assert _by_class(mean[nonfinite], want_mean, 0), grid     # a NaN draw: NaN; +inf and -inf: NaN; one infinity alone: itself


# ---- NaN and infinite draws through sample_summary ---------------------------------------------------------------------------
PROBS = (0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0)


def _by_class(got, want, rtol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    fin = np.isfinite(want)
    return (np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[np.isinf(want)], want[np.isinf(want)])
            and np.all(np.isfinite(got[fin])) and np.allclose(got[fin], want[fin], rtol=rtol, atol=0))


def test_nonfinite_derived_quantities_summarised_as_numpy(gpu_pkg):
    """lg = Math.log(mu) has NaN draws, inv = 1/(x*x) +inf only (x*x: an int state can be -0, and 1/-0 is -inf), both =
    1/(x - 1) - 1/(x - 2) +inf and -inf; mean, sd, rhat and quantiles equal numpy's on the raw draws, non-finite values by class.
    mu and x keep every key's bits against a handle that does not monitor the derived quantities."""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld

    def log_post(par, data=None):
        mu, x = par.mu, par.x
        lp = ld.norm(mu, 0.3, 1) + ld.pois(x, 0.5)
        par.lg = mcmc.Math.log(mu)
        par.inv = 1 / (x * x)
        par.both = 1 / (x - 1) - 1 / (x - 2)
        return lp

    params = {"mu": {"type": "real"}, "x": {"type": "int", "lower": 0}}
    mk = lambda **o: mcmc.AmwgSampler(params, log_post, None, dict({"chains": 2048, "seed": 31}, **o))
    a, b, c = mk(), mk(), mk(monitor=["mu", "x"])
    for s in (a, b, c):
        s.burn(200)
    rows = 40
    raw = a.sample(rows)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        summ = b.sample_summary(rows, PROBS, diagnostics=True, histogram=20)
    plain = c.sample_summary(rows, PROBS, diagnostics=True, histogram=20)
    assert set(summ) == {"mu", "x", "lg", "inv", "both"}
    assert {0.0, 1.0, 2.0} <= set(np.unique(raw["x"]).tolist())          # the draws that make inv and both infinite
    assert np.isnan(raw["lg"]).any() and np.isposinf(raw["inv"]).any() and not np.isneginf(raw["inv"]).any()
    assert np.isposinf(raw["both"]).any() and np.isneginf(raw["both"]).any() and not np.isnan(raw["both"]).any()
    wrong = []                                                            # every (name, key) that is not numpy's, then one assert
    for name in ("mu", "x", "lg", "inv", "both"):
        d = np.asarray(raw[name], dtype=np.float64)[:, None, :]          # [rows, 1, chains]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            m0, s0, r0, q0 = numpy_summary(d, PROBS)
        got = summ[name]
        for key, want, rtol in (("mean", m0, 1e-12), ("sd", s0, 1e-10), ("rhat", r0, 1e-8)):
            if not _by_class([got[key]], want, rtol):
                wrong.append((name, key, got[key], want[0]))
        if not np.array_equal(np.asarray(got["quantiles"]), q0[:, 0], equal_nan=True):
            wrong.append((name, "quantiles", got["quantiles"], q0[:, 0]))
        assert got["n_draws"] == rows * 2048
    assert not wrong, wrong
    assert np.isnan(summ["lg"]["quantiles"]).all() and summ["inv"]["mean"] == np.inf and np.isnan(summ["both"]["mean"])
    for name in ("mu", "x"):
        assert set(summ[name]) == set(plain[name])
        for key in summ[name]:
            assert np.asarray(summ[name][key]).tobytes() == np.asarray(plain[name][key]).tobytes(), (name, key)
    # the chains advanced exactly as sample(n) advances them
    for s in (b, c):
        assert all(np.asarray(a.state[k]).tobytes() == np.asarray(s.state[k]).tobytes() for k in ("mu", "x"))
