"""Test infrastructure: a numpy restatement of sample_summary(..., mcse=True) (bayes_js_b200.summary.mcse_block), straight from
the draws: the indicator sums C1, C2, P_t, G_t by direct counting (no bit tricks), the exact-rational GeyerESS inputs, ArviZ's
beta-rank rule with scipy, and mcse_sd from the halves. `NumpyMcseReducer` is a numpy stand-in for the device reductions
mcse_block calls, so the host path runs on CPU tensors. Never imported by the product."""
from fractions import Fraction

import numpy as np

from ess_ref import NumpyAutocovReducer, autocov_records, halves

BETA_PROBS = (0.1586553, 0.8413447)


def indicator_sums(x, thr, lag0, n_lags):
    """x [rows, entries, chains], thr [entries, K] -> int64 [entries, K, 2 + 2 n_lags] {C1, C2, P_t..., G_t...}"""
    rows, entries, chains = x.shape
    h = rows // 2
    thr = np.asarray(thr, dtype=np.float64).reshape(entries, -1)
    K = thr.shape[1]
    out = np.zeros((entries, K, 2 + 2 * n_lags), dtype=np.int64)
    for e in range(entries):
        for k in range(K):
            b = halves((x[:, e, :] <= thr[e, k]).astype(np.int64))       # [M, h]
            c = b.sum(axis=1)
            out[e, k, 0] = c.sum()
            out[e, k, 1] = (c * c).sum()
            for i in range(n_lags):
                t = lag0 + i
                out[e, k, 2 + i] = (b[:, :h - t] * b[:, t:]).sum()
                F = b[:, :t].sum(axis=1)
                L = b[:, h - t:].sum(axis=1) if t > 0 else np.zeros_like(c)
                out[e, k, 2 + n_lags + i] = (c * (F + L)).sum()
    return out


def geyer_inputs(sums, M, h, lag0):
    """one threshold's integer sums [2 + 2 n] -> the GeyerESS record [4 + n], every field an exact Fraction rounded once"""
    n = (len(sums) - 2) // 2
    C1, C2 = int(sums[0]), int(sums[1])
    rec = [float(M), float(Fraction(C1, M * h)), float(Fraction(M * C2 - C1 * C1, M * h * h)), float(Fraction(h * C1 - C2, h))]
    for i in range(n):
        t = lag0 + i
        P, G = int(sums[2 + i]), int(sums[2 + n + i])
        rec.append(float(Fraction(h * h * P - h * (2 * C2 - G) + (h - t) * C2, h * h)))
    return np.array(rec)


def ess_quantile(x, q):
    """x [rows, entries, chains], q [P, entries] -> ESS [P, entries] of 1[x <= q] from the whole lag range at once"""
    from bayes_js_b200.summary import GeyerESS
    rows, entries, chains = x.shape
    h, M = rows // 2, 2 * chains
    P = q.shape[0]
    out = np.full((P, entries), np.nan)
    if rows < 10:
        return out
    sums = indicator_sums(x, np.ascontiguousarray(q.T), 0, h)
    for e in range(entries):
        for p in range(P):
            s = sums[e, p]
            if s[0] == 0 or s[0] == M * h:
                out[p, e] = M * h
                continue
            rec = geyer_inputs(s, M, h, 0)
            g = GeyerESS(rec, h)
            g.add(rec[4:])
            out[p, e] = g.ess
    return out


def mcse_quantile(x, probs, ess):
    """ArviZ's _mcse_quantile with the given ess [P, entries] -> [P, entries]; NaN where ess is NaN"""
    from scipy.special import betaincinv
    rows, entries, chains = x.shape
    S = rows * chains
    out = np.full((len(probs), entries), np.nan)
    for e in range(entries):
        srt = np.sort(x[:, e, :].ravel())
        for i, p in enumerate(probs):
            es = ess[i, e]
            if not np.isfinite(es):
                continue
            a1, a2 = (betaincinv(es * p + 1, es * (1 - p) + 1, b) for b in BETA_PROBS)
            i1 = int(np.rint(max(a1 * S - 1, 0)))
            i2 = int(np.rint(min(a2 * S - 1, S - 1)))
            with np.errstate(invalid="ignore"):
                out[i, e] = (srt[i2] - srt[i1]) / 2
    return out


def ess_fft_direct(y):
    """ESS of y [rows, chains] by ess_ref's FFT estimator (independent of the windowed driver and of the record)"""
    from ess_ref import ess_fft
    return ess_fft(y)


def mcse_sd(x, mean, sd):
    """x [rows, entries, chains], the returned mean and sd per entry -> mcse_sd [entries], straight from the halves"""
    from ess_ref import geyer_tau, rho_fft
    rows, entries, chains = x.shape
    h = rows // 2
    out = np.full(entries, np.nan)
    if rows < 10:
        return out
    for e in range(entries):
        xe = x[:, e, :]
        if not np.all(np.isfinite(xe)):
            continue
        if sd[e] == 0:
            out[e] = 0.0
            continue
        s = 2.0 ** (1 - np.frexp(sd[e])[1])
        y = halves(((xe - mean[e]) * s) ** 2)
        M = y.shape[0]
        ybar = y.mean()
        v = ((y - ybar) ** 2).mean()
        rho, _, _ = rho_fft(y)
        ess_y = M * h / geyer_tau(rho, M, h)
        out[e] = np.sqrt(v / (4 * ybar * ess_y)) / s
    return out


class NumpyMcseReducer(NumpyAutocovReducer):
    """NumpyAutocovReducer plus the two mcse reductions, restated in numpy"""

    def __init__(self):
        super().__init__()
        self.indicator_windows = []

    def indicator_autocov(self, block, thresholds, lag0, n_lags):
        rows = block.shape[0]
        thr = np.asarray(thresholds, dtype=np.float64).reshape(block.shape[1], -1)
        assert 1 <= thr.shape[1] <= 16 and 1 <= n_lags <= 64 and 0 <= lag0 and lag0 + n_lags <= rows // 2
        self.indicator_windows.append((lag0, n_lags))
        return indicator_sums(block.numpy(), thr, lag0, n_lags)

    def autocov_sq(self, block, centre, scale, lag0, n_lags):
        x = block.numpy()
        with np.errstate(invalid="ignore", over="ignore"):
            y = ((x - np.asarray(centre)[None, :, None]) * np.asarray(scale)[None, :, None]) ** 2
        return autocov_records(y, None, lag0, n_lags)
