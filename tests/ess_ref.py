"""Test infrastructure for the split-chain diagnostics of bayes_js_b200.summary:
- `fft_diagnostics`: the estimator restated with full-length FFT autocovariances from the raw draws (no lag windows), as a
  user of sample() would compute it; independent of the windowed driver.
- `NumpyAutocovReducer`: a numpy stand-in for amwg_summary_autocov (plus the two reductions of summary_ref.NumpyBlockReducer),
  so the host path runs on CPU tensors.
Never imported by the product."""
import math

import numpy as np

from summary_ref import NumpyBlockReducer, run_means


def autocov_scale(q05, q95) -> float:
    """the power of two amwg_summary_autocov scales the draws series by (autocov_scale, csrc/amwg_autocov.cuh): 2^-ilogb(q95/2 -
    q05/2) clamped to [2^-1022, 2^1023]; 1 when that spread is 0 or not finite"""
    s = float(q95) * 0.5 - float(q05) * 0.5
    if not (0.0 < s <= 1.7976931348623157e308):
        return 1.0
    k = 1 - math.frexp(s)[1]                                  # -ilogb(s), subnormal s included
    return math.ldexp(1.0, min(max(k, -1022), 1023))


def halves(x):
    """x [rows, chains] -> [2*chains, h]: the first and the second half of every chain (middle row of odd rows dropped)."""
    rows = x.shape[0]
    h = rows // 2
    return np.concatenate([x[:h].T, x[rows - h:].T], axis=0)


def autocov_fft(y):
    """y [M, h] -> [M, h] acov_m(t) = (1/h) sum_{n<h-t} (y_n - ybar)(y_{n+t} - ybar), by zero-padded FFT."""
    M, h = y.shape
    d = y - y.mean(axis=1, keepdims=True)
    n = 1 << int(np.ceil(np.log2(2 * h)))
    f = np.fft.rfft(d, n=n, axis=1)
    return np.fft.irfft(f * np.conj(f), n=n, axis=1)[:, :h] / h


def rho_fft(y):
    """split-chain autocorrelations rho(t), t = 0..h-1, and (var+, W), from the half-chains y [M, h]."""
    M, h = y.shape
    acov = autocov_fft(y)
    W = h / (h - 1) * acov[:, 0].mean()
    B = y.mean(axis=1).var(ddof=1)
    varplus = (h - 1) / h * W + B
    return 1.0 - (W - acov.mean(axis=0)) / varplus, varplus, W


def geyer_tau(rho, M, h):
    """Geyer's initial positive then initial monotone sequence over rho(0..h-1), as written in the contract."""
    r = np.zeros(h + 2)
    r[0] = 1.0
    ev, od = 1.0, rho[1]
    r[1] = od
    t = 1
    while t < h - 3 and ev + od > 0:
        ev, od = rho[t + 1], rho[t + 2]
        if ev + od >= 0:
            r[t + 1], r[t + 2] = ev, od
        t += 2
    max_t = t - 2
    if ev > 0:
        r[max_t + 1] = ev
    t = 1
    while t <= max_t - 2:
        if r[t + 1] + r[t + 2] > r[t - 1] + r[t]:
            r[t + 1] = r[t + 2] = (r[t - 1] + r[t]) / 2
        t += 2
    tau = -1.0 + 2.0 * r[:max_t + 1].sum() + r[max_t + 1]
    return max(tau, 1.0 / np.log10(M * h))


def ess_fft(x):
    """ESS of x [rows, chains] (one series)."""
    y = halves(np.asarray(x, dtype=np.float64))
    M, h = y.shape
    rho, _, _ = rho_fft(y)
    return M * h / geyer_tau(rho, M, h)


def fft_diagnostics(x):
    """x [rows, entries, chains] -> {"ess_mean", "ess_tail", "mcse_mean", "rhat_split"} per entry, straight from the draws."""
    rows, entries, chains = x.shape
    out = {k: np.full(entries, np.nan) for k in ("ess_mean", "ess_tail", "mcse_mean", "rhat_split")}
    if rows < 10:
        return out
    h = rows // 2
    Mh = 2 * chains * h
    for e in range(entries):
        xe = x[:, e, :]
        flat = xe.ravel()
        if not np.isfinite(flat).all():
            continue
        lo, hi = np.quantile(flat, [0.05, 0.95])
        sd = flat.std(ddof=1) if flat.size > 1 else np.nan
        const = flat.min() == flat.max()
        ess = lambda y: Mh if y.min() == y.max() else ess_fft(y)
        out["ess_mean"][e] = Mh if const else ess_fft(xe)
        out["ess_tail"][e] = min(ess((xe <= lo).astype(float)), ess((xe <= hi).astype(float)))
        out["mcse_mean"][e] = 0.0 if const else sd / np.sqrt(out["ess_mean"][e])
        with np.errstate(invalid="ignore", divide="ignore"):
            _, varplus, W = rho_fft(halves(xe))
            out["rhat_split"][e] = np.sqrt(varplus / W)
    return out


def autocov_records(x, thresholds, lag0, n_lags):
    """numpy restatement of amwg_summary_autocov on x [rows, entries, chains] -> [entries, series, 4 + n_lags]; with thresholds,
    the draws series' centred values and means scaled by autocov_scale, as the device does."""
    rows, entries, chains = x.shape
    h = rows // 2
    ns = 1 if thresholds is None else 3
    out = np.empty((entries, ns, 4 + n_lags))
    for e in range(entries):
        series = [x[:, e, :]]
        if thresholds is not None:
            series += [(x[:, e, :] <= thresholds[e][0]).astype(float), (x[:, e, :] <= thresholds[e][1]).astype(float)]
        for s, ys in enumerate(series):
            y = halves(ys)
            m = run_means(y.T)                                 # a constant half-chain of draws is centred on its value
            d = y - m[:, None]
            if s == 0 and thresholds is not None:
                sc = autocov_scale(*thresholds[e])
                with np.errstate(over="ignore", invalid="ignore"):
                    m, d = m * sc, d * sc
            mean = run_means(m)                                # equal means: that value, as the Chan merge gives
            out[e, s, :4] = (y.shape[0], mean, ((m - mean) ** 2).sum(), (d * d).sum())
            for k in range(n_lags):
                t = lag0 + k
                out[e, s, 4 + k] = (d[:, :h - t] * d[:, t:]).sum()
    return out


class NumpyAutocovReducer(NumpyBlockReducer):
    def __init__(self):
        self.windows = []

    def autocov(self, block, thresholds, lag0, n_lags):
        rows = block.shape[0]
        assert 1 <= n_lags <= 32 and lag0 + n_lags <= rows // 2      # the device entry's argument checks
        self.windows.append((lag0, n_lags))
        return autocov_records(block.numpy(), thresholds, lag0, n_lags)


def ar1(phi, rows, chains, entries=1, seed=0):
    """[rows, entries, chains] stationary AR(1) chains with unit innovations: tau = (1 + phi) / (1 - phi)."""
    rng = np.random.default_rng(seed)
    eps = rng.normal(size=(rows, entries, chains))
    x = np.empty_like(eps)
    x[0] = eps[0] / np.sqrt(1 - phi * phi)
    for r in range(1, rows):
        x[r] = phi * x[r - 1] + eps[r]
    return x
