"""The covariance (K_c1..K_c4) and nested R-hat (K_n1, K_n2) reductions of sample_summary on the GPU, held to their references
(tests/cov_ref.py, tests/nested_ref.py) within the stated bounds at the shapes where the kernels change path: every block count
of the Gram kernel, chain counts where its 264 CTAs walk several 32-chain groups, chain-wise grids past 1184 x 256 threads,
superchain segments past the segment kernel's grid, shards cut inside a superchain, the measured production shapes, and
adversarial values. Every record is asked for twice and must keep its bits. Then the rule that a constant run is centred on its
value, end to end: an entry whose draws all equal one value has sd 0, exactly zero covariance rows and NaN R-hats."""
import numpy as np
import pytest

import cov_ref
import models
import nested_ref
from conftest import config2_data

pytestmark = pytest.mark.gpu

WALK = 264 * 32                      # amwg_comoments.cuh: kCoCtas x kCoChains, the chains one pass of the grid covers
CHAIN_GRID = 1184 * 256              # amwg_summary.cuh: kChainCtas x 256 threads


def _co_stage_rows(nb):
    return max(16 // nb, 1)


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to("cuda:0")


def _reducer():
    from bayes_js_b200.summary import CudaBlockReducer
    return CudaBlockReducer(0)


def _draws(rows, entries, chains, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(rows, entries, chains)) * rng.uniform(0.1, 3, size=(1, entries, 1))
    return offset + x + 0.3 * rng.normal(size=(1, entries, chains))


def _comoments(red, x, sel, what):
    blk = _dev(x)
    rec = red.comoments(blk, sel)
    assert red.comoments(blk, sel).tobytes() == rec.tobytes(), what                # a repeated call: the same bits
    return rec


def _split(rec, n):
    return rec[1:1 + n], rec[1 + n:1 + n + n * n].reshape(n, n), rec[1 + n + n * n:].reshape(n, n)


# ---- covariance ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb", range(1, 17))
@pytest.mark.parametrize("chains", [1001, WALK + 33])
def test_every_block_count(gpu_pkg, nb, chains):
    """nb = 1..16 blocks (reps 16..1, 1..9 tiles a warp, stages of 16 / nb rows), full and ragged selections, two stages and a
    ragged row; at WALK + 33 chains the first CTA walks two groups and the last group holds one chain"""
    red = _reducer()
    rows = 2 * _co_stage_rows(nb) + 1
    for n_sel in sorted({8 * nb, max(8 * nb - 5, 1)}):
        x = _draws(rows, n_sel + 2, chains, 97 * nb + n_sel + chains, 184.5)
        sel = np.random.default_rng(n_sel).permutation(n_sel + 2)[:n_sel].astype(np.int32)
        rec = _comoments(red, x, sel, (nb, n_sel, chains))
        cov_ref.check_record(rec, x, sel, (nb, n_sel, chains), exact=cov_ref.record(x, sel))


@pytest.mark.parametrize("chains", [WALK - 1, WALK, WALK + 1, 2 * WALK + 37, CHAIN_GRID + 77])
def test_walk_edges(gpu_pkg, chains):
    """around one and two passes of the grid walk, and past the chain-means kernel's grid; 1, 2 (16 and 8 reps), 24 (two reps),
    40 (15 tiles), 41 and 65 entries (2- and 3-slot warps)"""
    red = _reducer()
    for n_sel in (1, 2, 24, 40, 41, 65):
        x = _draws(3, n_sel, chains, chains + n_sel, 1e6)
        sel = np.arange(n_sel, dtype=np.int32)[::-1].copy()
        rec = _comoments(red, x, sel, (chains, n_sel))
        cov_ref.check_record(rec, x, sel, (chains, n_sel), exact=cov_ref.record(x, sel))


@pytest.mark.parametrize("n_sel, chains, rows", [(2, 1 << 20, 20), (65, 1 << 16, 20)])
def test_production_shapes(gpu_pkg, n_sel, chains, rows):
    """config 2's shape (two entries, 2^20 chains: 124 groups a CTA) and config 4's (65 entries, 2^16 chains: 8 groups a CTA)"""
    rng = np.random.default_rng(n_sel)
    x = 184.5 + 0.14 * rng.normal(size=(rows, n_sel, chains)) + 0.01 * rng.normal(size=(1, n_sel, chains))
    sel = np.arange(n_sel, dtype=np.int32)
    rec = _comoments(_reducer(), x, sel, n_sel)
    cov_ref.check_record(rec, x, sel, n_sel, exact=cov_ref.record(x, sel))


def _adversarial_block(rows, chains, seed):
    """[rows, 12, chains]: a normal entry, +-0, subnormals, +-1e150, 1e8 + 1e-3 z, the constants 0.1, 184.3 and 7.25, an entry
    constant within each chain, and two normal entries holding a NaN and a +inf at chains the grid walk reaches on its second group"""
    rng = np.random.default_rng(seed)
    z = lambda: rng.normal(size=(rows, chains))
    x = np.empty((rows, 12, chains))
    x[:, 0] = 3.0 + z()
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.5, -0.0, 0.0)              # +-0
    x[:, 2] = np.ldexp(np.round(rng.uniform(1, 2 ** 20, size=(rows, chains))), -1074)     # subnormals
    x[:, 3] = 1e150 * z()
    x[:, 4] = -1e150 + 1e135 * z()
    x[:, 5] = 1e8 + 1e-3 * z()                                                            # heavy cancellation
    x[:, 6] = 0.1
    x[:, 7] = 184.3
    x[:, 8] = 7.25
    x[:, 9] = rng.normal(size=(1, chains))                                                # constant within each chain
    x[:, 10] = 0.5 * x[:, 0] + z()
    x[:, 11] = z()
    x[rows // 2, 10, min(WALK + 5, chains - 3)] = np.nan
    x[0, 11, chains - 1] = np.inf
    return x


@pytest.mark.parametrize("chains", [WALK + 40, 2 * WALK + 37])
def test_adversarial_values(gpu_pkg, chains):
    from bayes_js_b200.summary import finalize_comoments
    rows = 5
    x = _adversarial_block(rows, chains, chains)
    n = x.shape[1]
    sel = np.arange(n, dtype=np.int32)
    rec = _comoments(_reducer(), x, sel, chains)
    m, B, W = _split(rec, n)
    bad = np.zeros(n, dtype=bool)
    bad[10:] = True
    # constants: their value as the mean, exactly zero rows and columns (against the finite entries); constant within chains: a
    # zero row of W only
    assert np.array_equal(m[6:9], [0.1, 184.3, 7.25])
    for M in (B, W):
        assert np.all(M[6:9][:, ~bad] == 0) and np.all(M[~bad][:, 6:9] == 0)
        assert np.all(M[1, ~bad] == 0) and np.all(M[~bad, 1] == 0)                        # +-0 centred: zeros
    assert np.all(W[9, ~bad] == 0) and np.all(W[~bad, 9] == 0) and B[9, 9] > 0
    # a NaN or +inf reached on a later group of the walk: that row and column NaN, as numpy.cov gives
    for M in (B, W):
        assert np.all(np.isnan(M[bad])) and np.all(np.isnan(M[:, bad]))
        assert np.all(np.isfinite(M[np.ix_(~bad, ~bad)]))
    with np.errstate(invalid="ignore", over="ignore"):
        want = np.cov(np.moveaxis(x, 1, 0).reshape(n, -1))
    fin = finalize_comoments(rec, rows)
    assert np.array_equal(np.isnan(fin["cov"][np.ix_(bad, bad)]), np.isnan(want[np.ix_(bad, bad)]))
    assert np.isnan(fin["rhat_multivariate"])
    # every finite entry within the bound. Higham's model has no underflow term, so the subnormal entry (2) is bounded apart: each
    # of its centres is off by at most 2^-1075 more in the device and in the reference, which a product with entry j carries as
    # 2^-1075 |d_j| twice, and each rounding of a product or sum in the subnormal range adds at most 2^-1075
    keep = np.arange(10, dtype=np.int32)
    sub = np.concatenate([[chains], m[keep], B[np.ix_(keep, keep)].ravel(), W[np.ix_(keep, keep)].ravel()])
    C, em, eB, eW = cov_ref.record(x, keep)
    bm, bB, bW = cov_ref.device_bound(x, keep)
    tiny = 2.0 ** -1074                                            # 2^-1075 itself is not a double: twice it
    xk = x[:, keep]
    xbar = xk.mean(axis=0)
    sW = np.abs(xk - xbar[None]).sum(axis=(0, 2))
    sB = np.abs(xbar - xbar.mean(axis=1, keepdims=True)).sum(axis=1)
    uW, uB = np.zeros((10, 10)), np.zeros((10, 10))
    uW[2] = uW[:, 2] = 4 * tiny * sW + (rows * chains + cov_ref.G_MAX + 8) * tiny
    uB[2] = uB[:, 2] = 4 * tiny * sB + (chains + cov_ref.G_MAX + 8) * tiny
    gm, gB, gW = _split(sub, len(keep))
    assert np.all(np.abs(gm - em) <= bm + (rows + chains) * tiny)
    assert np.all(np.abs(gB - eB) <= bB + uB) and np.all(np.abs(gW - eW) <= bW + uW)


# ---- nested R-hat --------------------------------------------------------------------------------------------------------------
def _nested(red, x, first, M, what):
    blk = _dev(x)
    got = red.nested(blk, first, M)
    assert red.nested(blk, first, M).tobytes() == got.tobytes(), what
    return got


@pytest.mark.parametrize("chains", [CHAIN_GRID + 77, 1 << 20])
@pytest.mark.parametrize("M", [1, 2, 64])
def test_nested_past_the_grids(gpu_pkg, chains, M):
    """K_n1 past 1184 x 256 chains, K_n2 past 1184 x 256 segments (M = 1 and 2 at 2^20 chains), whole superchains and a shard
    whose first chain cuts one at each end"""
    from bayes_js_b200.summary import finalize_nested, merge_nested_records
    red = _reducer()
    rows = 4
    x = _draws(rows, 2, chains, chains + M, 1e6)
    for first in (0, 3 * M + 1):
        got = _nested(red, x, first, M, (chains, M, first))
        exact, bound = nested_ref.check_record(got, x, first, M, (chains, M, first))
        if first % M == 0 and chains % M == 0:
            rh = finalize_nested(merge_nested_records([got], M, rows))
            lo, hi = nested_ref.rhat_interval(exact[:, :4], bound[:, :4])
            assert np.all((lo <= rh) & (rh <= hi)), (rh, lo, hi)


def test_nested_shard_inside_one_superchain(gpu_pkg):
    x = _draws(6, 3, 10, 5, 1e6)
    got = _nested(_reducer(), x, 5, 64, "inside")
    nested_ref.check_record(got, x, 5, 64, "inside")
    assert np.all(got[:, 0] == 0) and np.all(got[:, 4] == 0) and np.all(got[:, 5] == 10) and np.all(got[:, 9] == -1)


@pytest.mark.parametrize("M, chains", [(16, 4096), (64, CHAIN_GRID + 64 * 3)])
def test_nested_adversarial_values(gpu_pkg, M, chains):
    from bayes_js_b200.summary import finalize_nested, merge_nested_records
    rows = 5
    x = _adversarial_block(rows, chains, M)
    got = _nested(_reducer(), x, 0, M, (M, chains))
    # constants: their value and exact zeros; rhat_nested NaN
    assert np.array_equal(got[6:9, 1], [0.1, 184.3, 7.25]) and np.all(got[6:9, 2:4] == 0)
    assert np.all(got[1, 1:4] == 0)
    rh = finalize_nested(merge_nested_records([got], M, rows))
    assert np.all(np.isnan(rh[[1, 6, 7, 8, 10, 11]]))
    assert np.isnan(got[10, 1:4]).any() and not np.isfinite(got[11, 1:4]).all()
    fin = [0, 3, 4, 5, 9]                                           # the finite entries held to the bound
    exact, bound = nested_ref.record(x[:, fin], 0, M)
    assert np.array_equal(got[fin][:, [0, 4, 9]], exact[:, [0, 4, 9]])
    assert np.all(np.abs(got[fin] - exact) <= bound)
    lo, hi = nested_ref.rhat_interval(exact[:, :4], bound[:, :4])
    assert np.all((lo <= rh[fin]) & (rh[fin] <= hi))


# ---- end to end ----------------------------------------------------------------------------------------------------------------
def _check_cov_at_scale(cov, x):
    """x [rows, n, chains]: cov, corr, within, between and rhat_multivariate against numpy and scipy on the draws, vectorised over
    chains (tests/test_gpu_summary_covariance.py's check loops over them)"""
    import scipy.linalg
    rows, n, C = x.shape
    flat = np.moveaxis(x, 1, 0).reshape(n, -1)
    bm, bB, bW = cov_ref.device_bound(x, range(n))
    M = rows * C
    d = np.abs(flat - flat.mean(axis=1, keepdims=True))
    want = np.cov(flat)
    bound = (bW + rows * bB) / (M - 1) + cov_ref.gamma(M + 2) * (d @ d.T) / (M - 1) + 4 * cov_ref.U * np.abs(want)
    assert np.all(np.abs(cov["cov"] - want) <= bound)
    assert np.allclose(cov["corr"], np.corrcoef(flat), rtol=0, atol=1e-9)
    xb = x.mean(axis=0)                                                              # [n, C]
    dev = x - xb[None]
    within = np.einsum("ric,rjc->ij", dev, dev) / (C * (rows - 1))
    between = np.cov(xb)
    scale = np.outer(np.sqrt(np.diag(want)), np.sqrt(np.diag(want))).max()
    assert np.allclose(cov["within"], within, rtol=0, atol=1e-9 * scale)
    assert np.allclose(cov["between"], between, rtol=0, atol=1e-9 * scale)
    lam = scipy.linalg.eigh(between, within, eigvals_only=True).max()
    r = (rows - 1) / rows + (C + 1) / C * lam
    assert abs(cov["rhat_multivariate"] - r) <= 1e-8 * r


def test_config2_at_full_scale_with_covariance_and_nested(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    C, M, rows = 1 << 20, 64, 10
    mk = lambda: mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(ld), config2_data().tolist(),
                                  {"chains": C, "seed": 31, "init_radius": 2, "superchain_size": M})
    a, b, c = mk(), mk(), mk()
    for s in (a, b, c):
        s.burn(200)
    raw = a.sample(rows)
    got = b.sample_summary(rows, (0.05, 0.5, 0.95), covariance=True, nested=M)
    base = c.sample_summary(rows, (0.05, 0.5, 0.95))
    cov = got["covariance"]
    x = np.stack([np.asarray(raw[k], np.float64).reshape(rows, C, -1)[:, :, 0] for k in ("mu", "sigma")], axis=1)   # [rows, 2, C]
    assert cov["labels"] == ["mu", "sigma"]
    _check_cov_at_scale(cov, x)
    exact, bound = nested_ref.record(x, 0, M)
    lo, hi = nested_ref.rhat_interval(exact[:, :4], bound[:, :4])
    for e, k in enumerate(("mu", "sigma")):
        assert lo[e] <= got[k]["rhat_nested"] <= hi[e], (k, got[k]["rhat_nested"], lo[e], hi[e])
        assert set(got[k]) == set(base[k]) | {"rhat_nested"}
        for key, val in base[k].items():
            assert np.asarray(got[k][key]).tobytes() == np.asarray(val).tobytes(), (k, key)
    for k in ("mu", "sigma"):
        assert np.asarray(a.state[k]).tobytes() == np.asarray(b.state[k]).tobytes() == np.asarray(c.state[k]).tobytes()
    for s in (a, b, c):
        s.close()


def _constant_pool(rows, chains, seed):
    """[rows, 6, chains]: a normal entry, 0.1, 184.3 and 7.25 everywhere, chains stuck at their own values, a second normal"""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, 6, chains))
    x[:, 0] = rng.normal(size=(rows, chains))
    x[:, 1] = 0.1
    x[:, 2] = 184.3
    x[:, 3] = 7.25
    x[:, 4] = 0.1 * np.arange(chains)[None, :]
    x[:, 5] = 0.3 * x[:, 0] + rng.normal(size=(rows, chains))
    return x


@pytest.mark.parametrize("diagnostics", [True, "rank"])
@pytest.mark.parametrize("rows, chains", [(40, 64), (50, 4096)])
def test_constant_entries_through_the_block_summary(gpu_pkg, diagnostics, rows, chains):
    """sd 0, rhat, rhat_split and rhat_nested NaN, the value as the mean, zero covariance rows, NaN correlations and a NaN
    multivariate R-hat; chains stuck apart (W = 0 < B): rhat and rhat_split +inf"""
    from bayes_js_b200.summary import finalize_comoments, finalize_nested, merge_nested_records, summarise_block
    red = _reducer()
    x = _constant_pool(rows, chains, rows + chains)
    blk = _dev(x)
    mean, sd, rhat, q, (diag, _w) = summarise_block(red, blk, rows, chains, (0.05, 0.5, 0.95), False, diagnostics=diagnostics)
    assert np.array_equal(mean[1:4], [0.1, 184.3, 7.25]) and np.all(sd[1:4] == 0)
    assert np.all(np.isnan(rhat[1:4])) and np.all(np.isnan(diag["rhat_split"][1:4]))
    assert rhat[4] == np.inf and diag["rhat_split"][4] == np.inf
    assert np.all(np.isfinite(rhat[[0, 5]])) and np.all(np.isfinite(diag["rhat_split"][[0, 5]]))
    assert np.all(q[:, 1:4] == np.array([0.1, 184.3, 7.25])[None])
    fin = finalize_comoments(red.comoments(blk, np.arange(6, dtype=np.int32)), rows)
    for key in ("cov", "within", "between"):
        assert np.all(fin[key][1:4] == 0) and np.all(fin[key][:, 1:4] == 0), key
    assert np.all(np.isnan(fin["corr"][1:4])) and np.all(np.isnan(fin["corr"][:, 1:4]))
    assert np.isfinite(fin["corr"][0, 5]) and np.isnan(fin["rhat_multivariate"])
    rh = finalize_nested(merge_nested_records([red.nested(blk, 0, 16)], 16, rows))
    assert np.all(np.isnan(rh[1:4])) and np.all(np.isfinite(rh[[0, 4, 5]]))


def test_constant_derived_quantity_through_sample_summary(gpu_pkg):
    """a derived quantity that stays 0.1 (mu * 0 + 0.1 is 0.1 for every finite mu) is monitored and summarised like a parameter:
    sd 0, rhat NaN, zero covariance rows, and the multivariate R-hat of the whole selection NaN"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld

    def log_post(par, data):
        lp = ld.norm(par.mu, 0, 100) + ld.unif(par.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], par.mu, par.sigma)
        par.c = par.mu * 0 + 0.1
        return lp
    s = mcmc.AmwgSampler(models.PARAMS_NORM, log_post, config2_data().tolist()[:64], {"chains": 1024, "seed": 5})
    s.burn(200)
    out = s.sample_summary(40, (0.5,), diagnostics=True, covariance=True, nested=16)
    assert out["c"]["mean"] == 0.1 and out["c"]["sd"] == 0 and np.isnan(out["c"]["rhat"])
    assert np.isnan(out["c"]["rhat_split"]) and np.isnan(out["c"]["rhat_nested"])
    cov = out["covariance"]
    i = cov["labels"].index("c")
    assert np.all(cov["cov"][i] == 0) and np.all(np.isnan(cov["corr"][i])) and np.isnan(cov["rhat_multivariate"])
    assert np.isfinite(out["mu"]["rhat"]) and np.isfinite(out["mu"]["rhat_nested"])
    s.close()
