"""Test infrastructure for the rank-normalised diagnostics of bayes_js_b200.summary (diagnostics="rank"):
- `rank_diagnostics_ref`: the estimator restated from the raw draws with scipy.stats.rankdata and scipy.special.ndtri over the
  half-chains and the FFT ESS / split R-hat of ess_ref, with the edge rules of summary.rank_diagnostics.
- `NumpyRankReducer`: a numpy stand-in for amwg_summary_rank_sort / _rank_count / _rank_z (plus the reductions of
  ess_ref.NumpyAutocovReducer), so the host driver and the ring of collectives run on CPU tensors.
Never imported by the product."""
import numpy as np
from scipy.special import ndtri
from scipy.stats import rankdata

from ess_ref import NumpyAutocovReducer, ess_fft, halves, rho_fft


def canonical_keys(v):
    """order-preserving uint64 keys with -0 made +0 (what the device sorts)."""
    v = np.where(v == 0.0, 0.0, np.asarray(v, dtype=np.float64))
    u = np.ascontiguousarray(v).view(np.uint64)
    sign = np.uint64(1 << 63)
    return np.where((u & sign) != 0, ~u, u | sign)


def half_draws(x):
    """x [rows, chains] -> [2h, chains]: rows [0, h) then rows [rows-h, rows), the ranked draws in z-block order."""
    rows = x.shape[0]
    h = rows // 2
    return np.concatenate([x[:h], x[rows - h:]], axis=0)


def z_scores(v):
    """z = Phi^-1((r - 3/8) / (S + 1/4)) of the values v (any shape) ranked among themselves."""
    flat = np.where(v == 0.0, 0.0, v).ravel()
    r = rankdata(flat, method="average")
    S = flat.size
    return ndtri((r - 0.375) / (S + 0.25)).reshape(v.shape)


def _rhat(y):
    with np.errstate(invalid="ignore", divide="ignore"):
        _, varplus, W = rho_fft(halves(y))
        return np.sqrt(varplus / W)


def rank_diagnostics_ref(x):
    """x [rows, entries, chains] -> {"ess_bulk", "rhat_rank"} per entry, straight from the draws."""
    rows, entries, chains = x.shape
    out = {k: np.full(entries, np.nan) for k in ("ess_bulk", "rhat_rank")}
    if rows < 10:
        return out
    h = rows // 2
    for e in range(entries):
        xe = x[:, e, :]
        if np.isnan(xe).any():
            continue
        hd = half_draws(xe)                                   # [2h, chains]: halves() of it are the split chains
        if np.all(hd == hd.ravel()[0]):
            out["ess_bulk"][e] = 2 * chains * h
            continue
        z = z_scores(hd)
        out["ess_bulk"][e] = ess_fft(z)
        rb = _rhat(z)
        med = np.quantile(xe.ravel(), 0.5)
        if not np.isfinite(med):
            continue
        f = np.abs(hd - med)
        if np.all(f == f.ravel()[0]):
            out["rhat_rank"][e] = rb
            continue
        out["rhat_rank"][e] = max(rb, _rhat(z_scores(f)))
    return out


class NumpyRankReducer(NumpyAutocovReducer):
    def __init__(self):
        super().__init__()
        self.sorts = []

    def rank_sort(self, block, entry, centre, keys, index):
        x = block.numpy()[:, entry, :]
        rows = x.shape[0]
        assert rows >= 2
        v = half_draws(x).ravel()
        if not np.isnan(centre):
            v = np.abs(v - centre)
        k = canonical_keys(v)
        n = k.size
        assert keys.numel() >= 2 * n and index.numel() >= 2 * n
        order = np.argsort(k, kind="stable")
        keys.numpy()[:n] = k[order].view(np.int64)
        index.numpy()[:n] = order.astype(np.int32)
        passes = sum(1 for d in range(8) if np.unique((k >> np.uint64(8 * d)) & np.uint64(255)).size > 1)
        self.sorts.append((entry, float(centre), passes))
        return passes

    def rank_count(self, q, nq, r, nr, acc):
        qk = q.numpy()[:nq].view(np.uint64)
        rk = r.numpy()[:nr].view(np.uint64)
        assert np.all(qk[1:] >= qk[:-1]) and np.all(rk[1:] >= rk[:-1])
        acc.numpy()[:nq] += np.searchsorted(rk, qk, "left") + np.searchsorted(rk, qk, "right")

    def rank_z(self, acc, index, n, total, z):
        a = acc.numpy()[:n]
        z.numpy().reshape(-1)[index.numpy()[:n]] = ndtri(((a + 1) / 2 - 0.375) / (total + 0.25))
