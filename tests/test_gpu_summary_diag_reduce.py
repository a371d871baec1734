"""The split-chain and rank reductions of sample_summary(..., diagnostics=True / "rank") on the GPU, held to exact references:
amwg_summary_autocov's records within tests/autocov_ref.py's bound at full scale and on adversarial blocks, the ESS and split
R-hat of the windowed Geyer driver inside the interval its decisions allow, amwg_summary_rank_z against Phi^-1 of its rounded
argument at 100 digits, amwg_summary_rank_count against closed-form counts past 2^31 merged keys, and the ESS and split R-hat
unchanged, bit for bit, when the draws are scaled by a power of two. Then the rank-normalised path end to end at 2^18 chains x
200 kept rows: ranks and z exact, the records of z within the bound, ess_bulk and rhat_rank inside their intervals. Every record
is asked for twice and must keep its bits."""
import numpy as np
import pytest

import autocov_ref
from ess_ref import ar1

pytestmark = pytest.mark.gpu
CHAIN_GRID = 1184 * 256                  # amwg_summary.cuh: kChainCtas x 256 threads


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to("cuda:0")


def _reducer():
    from bayes_js_b200.summary import CudaBlockReducer
    return CudaBlockReducer(0)


def _thr(x):
    return np.stack([np.quantile(np.moveaxis(x, 1, 0).reshape(x.shape[1], -1), p, axis=1) for p in (0.05, 0.95)], axis=1)


def _autocov(red, blk, thr, lag0, n_lags, what):
    got = red.autocov(blk, thr, lag0, n_lags)
    assert red.autocov(blk, thr, lag0, n_lags).tobytes() == got.tobytes(), what
    return got



@pytest.mark.parametrize("rows, chains, thresholds, windows", [
    (100, 1 << 20, True, [(0, 3), (17, 1)]),            # config 2's shape: 2^20 chains, four a thread
    (1000, CHAIN_GRID + 77, False, [(31, 1)]),          # every thread walks two chains of 500-draw halves
])
def test_records_at_full_scale(gpu_pkg, rows, chains, thresholds, windows):
    x = ar1(0.7, rows, chains, 1, rows)
    x = 184.5 + 0.14 * x
    thr = _thr(x) if thresholds else None
    blk = _dev(x)
    red = _reducer()
    for lag0, n_lags in windows:
        got = _autocov(red, blk, thr, lag0, n_lags, (rows, lag0))
        exact, bound = autocov_ref.record(x, thr, lag0, n_lags)
        autocov_ref.check_record(got, exact, bound, (rows, lag0))


class _Capture:
    """wraps the device reducer and keeps every autocov window it is asked for, as the summary path asks for them"""
    def __init__(self, red):
        self.red, self.calls = red, []

    def __getattr__(self, name):
        return getattr(self.red, name)

    def autocov(self, block, thresholds, lag0, n_lags):
        out = self.red.autocov(block, thresholds, lag0, n_lags)
        self.calls.append((None if thresholds is None else np.array(thresholds), lag0, n_lags, out))
        return out


def _lags_read(calls, h):
    """1 + the last lag GeyerESS reads over the captured windows' records, for every series: the window's lags past it are
    fetched but never used"""
    from bayes_js_b200.summary import GeyerESS
    rec = np.concatenate([calls[0][3]] + [g[:, :, 4:] for _, _, _, g in calls[1:]], axis=2)
    L = 1
    for e in range(rec.shape[0]):
        for s in range(rec.shape[1]):
            g = GeyerESS(rec[e, s], h)
            g.add(rec[e, s, 4:])
            L = max(L, g.t + 3)
    return min(L, rec.shape[2] - 4)


def _check_summary(x, diag, calls, name, series=(0, 1, 2)):
    """every captured window's lags that Geyer's loop reads within the bound; ess_mean, ess_tail and rhat_split inside the
    intervals (of the listed series) -> (decided, total)"""
    h = x.shape[0] // 2
    thr = calls[0][0]
    L = _lags_read(calls, h)
    exact, bound = autocov_ref.record(x, thr, 0, L, series)
    for t, l0, n, got in calls:
        assert np.array_equal(t, thr)
        if l0 >= L:
            continue
        k = min(n, L - l0)
        sl = list(range(4)) + list(range(4 + l0, 4 + l0 + k))
        autocov_ref.check_record(got[:, :, :4 + k], exact[:, :, sl], bound[:, :, sl], (name, l0))
    decided = total = 0
    for e in range(x.shape[1]):
        ivs = [autocov_ref.interval(exact[e, s], bound[e, s], h) if s in series else None for s in range(3)]
        total += len(series)
        decided += sum(iv is not None for iv in ivs)
        if ivs[0] is not None:
            assert autocov_ref.inside(diag["ess_mean"][e], ivs[0][0]), (name, e, diag["ess_mean"][e], ivs[0][0])
            assert autocov_ref.inside(diag["rhat_split"][e] ** 2, ivs[0][1]), (name, e)
        if ivs[1] is not None and ivs[2] is not None:
            lo = min(ivs[1][0][0], ivs[2][0][0]), min(ivs[1][0][1], ivs[2][0][1])
            assert autocov_ref.inside(diag["ess_tail"][e], lo), (name, e, diag["ess_tail"][e], lo)
    return decided, total


def test_long_chains_need_many_windows(gpu_pkg):
    """20000 rows x 64 chains of AR(0.995): Geyer's loop runs for hundreds of lags over many 32-lag windows; every window's record
    of the draws and of both indicators within the bound, ess_mean, ess_tail and rhat_split inside the intervals of the exact
    records"""
    from bayes_js_b200.summary import summarise_block
    rows, chains = 20000, 64
    x = ar1(0.995, rows, chains, 1, 12)
    cap = _Capture(_reducer())
    *_, (diag, windows) = summarise_block(cap, _dev(x), rows, chains, (0.5,), False, diagnostics=True)
    assert windows >= 8, windows
    decided, total = _check_summary(x, diag, cap.calls, "ar0.995")
    assert decided == total, (decided, total)


def _adversarial(rows, chains, seed):
    """[rows, 9, chains]: normal, +-0, subnormals, 1e8 + 1e-3 z, the constant 7.25, half-chains constant at values of their own,
    an entry holding +-inf, one holding a NaN, and 1e-300-scale draws whose squares underflow unless scaled"""
    rng = np.random.default_rng(seed)
    z = lambda: rng.normal(size=(rows, chains))
    x = np.empty((rows, 9, chains))
    x[:, 0] = 3.0 + z()
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.5, -0.0, 0.0)
    x[:, 2] = np.ldexp(np.round(rng.uniform(1, 2 ** 20, size=(rows, chains))), -1074)
    x[:, 3] = 1e8 + 1e-3 * z()
    x[:, 4] = 7.25
    h = rows // 2
    x[:h, 5] = rng.normal(size=(1, chains))
    x[h:, 5] = rng.normal(size=(1, chains))
    x[:, 6] = z(); x[2, 6, 5] = np.inf; x[3, 6, chains - 1] = -np.inf
    x[:, 7] = z(); x[0, 7, 1] = np.nan
    x[:, 8] = 1e-300 * ar1(0.5, rows, chains, 1, seed)[:, 0]
    return x


@pytest.mark.parametrize("rows, chains", [(23, 4096 + 77), (40, 2 * 4096 + 77)])
def test_adversarial_records(gpu_pkg, rows, chains):
    """the adversarial entries, with the pooled quantiles as thresholds, with thresholds at the minimum and the maximum, and
    without: every field of every finite series within the bound, the constant exactly, two calls the same bits"""
    x = _adversarial(rows, chains, rows)
    blk = _dev(x)
    red = _reducer()
    q = _thr(x)
    fl = np.moveaxis(x, 1, 0).reshape(x.shape[1], -1)
    with np.errstate(invalid="ignore"):
        ends = np.stack([fl.min(axis=1), fl.max(axis=1)], axis=1)
    for thr in (q, ends, None):
        for lag0, n_lags in ((0, 5), (3, 7)):
            got = _autocov(red, blk, thr, lag0, n_lags, (rows, lag0))
            exact, bound = autocov_ref.record(x, thr, lag0, n_lags)
            autocov_ref.check_record(got, exact, bound, (rows, lag0, thr is None))
            assert got[4, 0, 1] == 7.25 and np.all(got[4, 0, 2:] == 0)
            assert got[5, 0, 3] == 0 and got[5, 0, 2] > 0                          # half-chains stuck apart: W = 0 < B
            for e in (6, 7):
                assert not np.all(np.isfinite(got[e, 0, 2:]))


def test_adversarial_summary(gpu_pkg):
    from bayes_js_b200.summary import summarise_block
    rows, chains = 40, 4096 + 77
    x = _adversarial(rows, chains, 3)
    cap = _Capture(_reducer())
    *_, (diag, _w) = summarise_block(cap, _dev(x), rows, chains, (0.5,), False, diagnostics=True)
    assert diag["rhat_split"][5] == np.inf and np.isnan(diag["ess_mean"][5])
    assert np.isnan(diag["rhat_split"][4]) and diag["ess_mean"][4] == 2 * chains * (rows // 2)
    assert all(np.isnan(diag[k][e]) for k in ("ess_mean", "ess_tail", "rhat_split") for e in (6, 7))
    keep = [0, 2, 3, 8]
    decided, total = _check_summary(x[:, keep], {k: v[keep] for k, v in diag.items()},
                                    [(t[keep], l0, n, g[keep]) for t, l0, n, g in cap.calls], "adversarial")
    assert decided >= total - 1, (decided, total)


SCALES = (-1000, -560, -300, 0, 300, 511, 900)


def test_ess_and_rhat_do_not_depend_on_the_scale(gpu_pkg):
    """AR(0.6) draws times 2^j on the device: the bits of ess_mean, ess_tail and rhat_split of the unscaled draws (before the
    scaling, 2^-560 and 2^511 gave ESS 52572, four times the draws)"""
    from bayes_js_b200.summary import summarise_block
    x = ar1(0.6, 200, 64, 1, 3)
    res = {}
    for j in SCALES:
        *_, (d, _w) = summarise_block(_reducer(), _dev(np.ldexp(x, j)), 200, 64, (0.5,), False, diagnostics=True)
        res[j] = d
    for j in SCALES:
        for k in ("ess_mean", "ess_tail", "rhat_split"):
            assert res[j][k].tobytes() == res[0][k].tobytes(), (j, k, res[j][k], res[0][k])
    assert 3000 < res[0]["ess_mean"][0] < 3500


def test_scale_through_derived_quantities(gpu_pkg):
    """config 2's model with derived quantities mu * 2^-560 and mu * 2^511 (about 1e-166 and 1e156): their ess_mean, ess_tail and
    rhat_split have the bits of mu's"""
    import models
    from conftest import config2_data
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld

    def log_post(par, data):
        lp = ld.norm(par.mu, 0, 100) + ld.unif(par.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], par.mu, par.sigma)
        par.tiny = par.mu * 2.0 ** -560
        par.huge = par.mu * 2.0 ** 511
        return lp
    s = mcmc.AmwgSampler(models.PARAMS_NORM, log_post, config2_data().tolist()[:64], {"chains": 4096, "seed": 9})
    s.burn(200)
    out = s.sample_summary(60, (0.5,), diagnostics=True)
    s.close()
    assert 0 < out["mu"]["ess_mean"] < 2 * 4096 * 30
    for name in ("tiny", "huge"):
        for k in ("ess_mean", "ess_tail", "rhat_split"):
            assert np.float64(out[name][k]).tobytes() == np.float64(out["mu"][k]).tobytes(), (name, k, out[name][k], out["mu"][k])


def test_what_cannot_be_computed_is_nan_on_the_device(gpu_pkg):
    """an entry with q05 == q95 (not scaled) whose squares underflow, and one whose scaled outliers overflow: ESS and rhat_split
    NaN, never a finite value, while a normal entry beside them keeps finite values"""
    from bayes_js_b200.summary import summarise_block
    rng = np.random.default_rng(7)
    rows, chains = 40, 32
    x = np.empty((rows, 3, chains))
    x[:, 0] = ar1(0.5, rows, chains, 1, 8)[:, 0]
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.97, 1.0, 1.0 + rng.normal(size=(rows, chains))) * 2.0 ** -600
    x[:, 2] = np.where(rng.uniform(size=(rows, chains)) < 0.97, 1e-300 * rng.normal(size=(rows, chains)), 1e300)
    *_, (d, _w) = summarise_block(_reducer(), _dev(x), rows, chains, (0.5,), False, diagnostics=True)
    assert np.isfinite(d["ess_mean"][0]) and np.isfinite(d["rhat_split"][0])
    for e in (1, 2):
        assert np.isnan(d["ess_mean"][e]) and np.isnan(d["rhat_split"][e]), (e, d)


# ---- rank_z --------------------------------------------------------------------------------------------------------------------
# CUDA's documented bound for normcdfinv in double precision is 5 ulp, held at every z != 0; Phi^-1(0.5) = 0 exactly, and there
# the device must give 0. Measured on an H100 80GB HBM3 (700 W): at most 3 ulp over these ranks.
Z_ULP = 5.0


def _z_ok(z, want, ulp=Z_ULP):
    return z == 0 if want == 0 else abs(z - want) <= ulp * np.spacing(abs(want))


def test_rank_z_against_100_digit_inverse(gpu_pkg):
    import mpmath
    import torch
    mpmath.mp.dps = 100
    for total in (2, 3, 10, (1 << 20) + 1, (1 << 32) - 1, (1 << 40) + 7, (1 << 52) - 1):
        ranks = {1, 2, 3, total, total - 1, total - 2, total // 2, (total + 1) // 2, total // 2 + 1, total // 3}
        acc = sorted({2 * r - 1 for r in ranks if 1 <= r <= total} | {2 * r for r in ranks if 1 <= r < total})   # ties: even
        z = []
        for c in range(0, len(acc), total):                           # at most `total` draws a call
            part = acc[c:c + total]
            n = len(part)
            a = torch.tensor(part, dtype=torch.int64, device="cuda:0")
            idx = torch.arange(n - 1, -1, -1, dtype=torch.int32, device="cuda:0")
            zc = torch.full((n,), np.nan, dtype=torch.float64, device="cuda:0")
            _reducer().rank_z(a, idx, n, total, zc)
            z.extend(zc.cpu().numpy()[::-1])
        for i, v in enumerate(acc):
            p = ((v + 1) * 0.5 - 0.375) / (total + 0.25)             # the kernel's fp64 argument
            want = float(mpmath.sqrt(2) * mpmath.erfinv(2 * mpmath.mpf(p) - 1))
            assert _z_ok(z[i], want), (total, v, z[i], want)


# ---- rank_count ----------------------------------------------------------------------------------------------------------------
def _keys(n, div, odd, device, lo=0):
    import torch
    i = torch.arange(lo, lo + n, dtype=torch.int64, device=device)
    return 2 * torch.div(i, div, rounding_mode="floor") + odd


@pytest.mark.parametrize("nq, nr", [(5, 3000), (2047, 2049), (4096 * 3 + 1, 4096 * 3 + 1), ((1 << 30) + 12345, (1 << 30) + 54321)])
def test_rank_count_closed_form(gpu_pkg, nq, nr):
    """Q_i = 2 floor(i / 3), R_j = 2 floor(j / 5) + 1: acc[i] = 2 min(5 floor(i / 3), nr); against Q itself, #(Q < Q_i) +
    #(Q <= Q_i) = 3 a + min(3 a + 3, nq) with a = floor(i / 3). Q shorter than a tile, merged lengths off the tile, and past 2^31"""
    import torch
    dev = torch.device("cuda:0")
    q = _keys(nq, 3, 0, dev)
    r = _keys(nr, 5, 1, dev)
    acc = torch.zeros(nq, dtype=torch.int64, device=dev)
    red = _reducer()
    red.rank_count(q, nq, r, nr, acc)
    step = 1 << 27
    for lo in range(0, nq, step):
        a = torch.div(torch.arange(lo, min(lo + step, nq), dtype=torch.int64, device=dev), 3, rounding_mode="floor")
        assert torch.equal(acc[lo:lo + step], 2 * torch.clamp(5 * a, max=nr)), (nq, nr, lo)
    del r
    acc.zero_()
    red.rank_count(q, nq, q, nq, acc)
    for lo in range(0, nq, step):
        a = torch.div(torch.arange(lo, min(lo + step, nq), dtype=torch.int64, device=dev), 3, rounding_mode="floor")
        assert torch.equal(acc[lo:lo + step], 3 * a + torch.clamp(3 * a + 3, max=nq)), (nq, lo)


# ---- rank-normalised diagnostics end to end --------------------------------------------------------------------------------
def _recording_reducer_class(log):
    from bayes_js_b200.summary import CudaBlockReducer

    class Recording(CudaBlockReducer):
        """CudaBlockReducer that keeps, on the host, the draws block, every autocov window (with its block when that is a z-block
        asked for from lag 0) and the sorted key ends, as sample_summary drives it"""
        def moments(self, block):
            if "x" not in log:
                log["x"] = block.cpu().numpy()
            return super().moments(block)

        def autocov(self, block, thresholds, lag0, n_lags):
            out = super().autocov(block, thresholds, lag0, n_lags)
            z = block.cpu().numpy() if thresholds is None and lag0 == 0 else None
            log.setdefault("calls", []).append((None if thresholds is None else np.array(thresholds), lag0, n_lags, out, z))
            return out
    return Recording


def _expected_z(v):
    """v: the S ranked values in draw order -> Phi^-1((r - 3/8) / (S + 1/4)) with r the average rank (ties averaged, -0 = +0), and the
    argument; the ranks from a sort of v and two binary searches per value (torch on the device, exact integers)"""
    import torch
    from scipy.special import ndtri
    S = v.size
    t = torch.from_numpy(v + 0.0).to("cuda:0")
    srt = torch.sort(t).values
    acc = (torch.searchsorted(srt, t, right=False) + torch.searchsorted(srt, t, right=True)).cpu().numpy()
    del t, srt
    p = ((acc + 1) * 0.5 - 0.375) / (S + 0.25)
    return ndtri(p), p


def test_rank_diagnostics_end_to_end_config2(gpu_pkg, monkeypatch):
    """config 2's model and data through sample_summary(..., diagnostics="rank") at 2^18 chains x 200 kept rows (5.2e7 ranked draws
    an entry; at 2^20 chains the host-side exact reference alone takes over ten minutes): the
    device's z-blocks (bulk and folded) equal Phi^-1 of the exact average ranks within 16 ulp (the device's 5, scipy's ndtri's
    few), which pins every rank, since neighbouring ranks move z by more than 1e-9 of itself; the autocov records of z and of the
    draws within the bound on every lag Geyer's loop reads; ess_bulk, rhat_rank, ess_mean, ess_tail and rhat_split inside the
    intervals of the exact records"""
    import models
    from bayes_js_b200 import summary as summ
    from conftest import config2_data
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    log = {}
    monkeypatch.setattr(summ, "CudaBlockReducer", _recording_reducer_class(log))
    rows, chains = 200, 1 << 18
    s = mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(ld), config2_data().tolist(), {"chains": chains, "seed": 23})
    s.burn(1000)
    out = s.sample_summary(rows, (0.5,), diagnostics="rank")
    s.close()
    monkeypatch.undo()
    x = log.pop("x")
    h = rows // 2
    S = 2 * h * chains
    draw_calls = [c[:4] for c in log["calls"] if c[0] is not None]
    z_calls = [c for c in log["calls"] if c[0] is None]
    names = ["mu", "sigma"]
    diag = {k: np.array([out[n][k] for n in names]) for k in ("ess_mean", "ess_tail", "rhat_split")}
    decided, total = _check_summary(x, diag, draw_calls, "config2 draws")
    zi = 0
    for e, name in enumerate(names):
        v = x[:, e, :].ravel()                                   # rows [0, h) then [h, 2h): draw i = r chains + c
        med = np.quantile(v, 0.5)
        bulk = z_calls[zi]
        zi += 1
        more = []
        while zi < len(z_calls) and z_calls[zi][1] > 0:
            more.append(z_calls[zi])
            zi += 1
        fold = z_calls[zi]
        zi += 1
        assert (bulk[1], fold[1], fold[2]) == (0, 0, 1)
        for zc, vals in ((bulk, v), (fold, np.abs(v - med))):
            want, p = _expected_z(vals)
            got = zc[4].ravel()
            zero = want == 0
            assert np.all(got[zero] == 0), name
            ok = np.abs(got - want) <= 16 * np.spacing(np.abs(want))
            assert np.all(ok | zero), (name, np.argwhere(~(ok | zero))[:5], got[~(ok | zero)][:5], want[~(ok | zero)][:5])
            del want, p
        zb = bulk[4]
        L = _lags_read([(None, l0, n, o) for _, l0, n, o, _z in [bulk] + more], h)
        exact, bound = autocov_ref.record(zb, None, 0, L)
        autocov_ref.check_record(bulk[3][:, :, :4 + min(L, bulk[2])], exact[:, :, :4 + min(L, bulk[2])],
                                 bound[:, :, :4 + min(L, bulk[2])], (name, "z"))
        for _t, l0, n, o, _z in more:
            if l0 < L:
                k = min(n, L - l0)
                sl = list(range(4)) + list(range(4 + l0, 4 + l0 + k))
                autocov_ref.check_record(o[:, :, :4 + k], exact[:, :, sl], bound[:, :, sl], (name, "z", l0))
        fe, fb = autocov_ref.record(fold[4], None, 0, 1)
        autocov_ref.check_record(fold[3], fe, fb, (name, "folded z"))
        iv = autocov_ref.interval(exact[0, 0], bound[0, 0], h)
        rf = autocov_ref.ratio_interval(fe[0, 0], fb[0, 0], h)
        total += 2
        if iv is not None:
            decided += 1
            assert autocov_ref.inside(out[name]["ess_bulk"], iv[0]), (name, out[name]["ess_bulk"], iv[0])
        if iv is not None and rf is not None:
            decided += 1
            hi = max(iv[1][0], rf[0]), max(iv[1][1], rf[1])
            assert autocov_ref.inside(out[name]["rhat_rank"] ** 2, hi), (name, out[name]["rhat_rank"], hi)
    assert zi == len(z_calls)
    assert decided >= total - 1, (decided, total)
