"""Test infrastructure: PSIS-LOO and WAIC restated in numpy from the papers (Vehtari, Gelman & Gabry 2017, "Practical Bayesian
model evaluation using leave-one-out cross-validation and WAIC"; Vehtari, Simpson, Gelman, Yao & Gabry 2024, "Pareto smoothed
importance sampling"; Zhang & Stephens 2009 for the generalised Pareto fit), in ArviZ's conventions, applied to a full
pointwise log-likelihood matrix ll[S, N]. Independent of the product: it sorts with numpy and sums with numpy."""
import math

import numpy as np

EPS = np.finfo(float).eps
LOG_TINY = np.log(np.finfo(float).tiny)


BLOCK_ELEMENTS = 1 << 24              # gpdfit's candidate matrix is formed in row blocks of at most this many elements


def gpdfit(x, block=None):
    """Zhang & Stephens (2009) with the weakly informative prior on k (prior_bs = 3, prior_k = 10); x ascending. -> (k, sigma).
    Candidates whose profile value L is not finite are left out (a b of exactly 0 in a tied tail, or every b infinite when a
    quarter of x is 0); ArviZ keeps them and gets NaN weights. With none left: (inf, nan), the tail is not smoothed.
    k(b) is the mean of log1p(-b x) over a [rows, n] block of candidates at a time: `block` rows (default: as many as keep the
    block within BLOCK_ELEMENTS), so n = 2^20 does not need the m x n matrix (8.8 GB)."""
    n = len(x)
    m = 30 + int(n ** 0.5)
    b = 1 - np.sqrt(m / (np.arange(1, m + 1, dtype=float) - 0.5))
    b /= 3 * x[int(n / 4 + 0.5) - 1]
    b += 1 / x[-1]
    rows = block or max(1, BLOCK_ELEMENTS // n)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        k = np.concatenate([np.log1p(-b[j:j + rows, None] * x).mean(axis=1) for j in range(0, m, rows)])
        L = n * (np.log(-(b / k)) - k - 1)
    fin = np.isfinite(L)
    if not fin.any():
        return np.inf, np.nan
    b, L = b[fin], L[fin]
    w = 1 / np.exp(L - L[:, None]).sum(axis=1)
    keep = w >= 10 * EPS
    w, b = w[keep], b[keep]
    w = w / w.sum()
    bp = np.sum(b * w)
    kp = np.log1p(-bp * x).mean()
    sigma = -kp / bp
    kp = (n * kp + 10 * 0.5) / (n + 10)
    return kp, sigma


def gpinv(p, k, sigma):
    if sigma <= 0:
        return np.full_like(p, np.nan)
    x = -np.log1p(-p) if abs(k) < EPS else np.expm1(-k * np.log1p(-p)) / k
    return x * sigma


def tail_length(S, r_eff):
    return int(math.ceil(min(0.2 * S, 3 * math.sqrt(S / r_eff))))


def psis_point(ll, r_eff=1.0):
    """One point: -> dict(lw (normalised smoothed log weights), k, tail (sorted indices of the tail draws), cut)."""
    S = len(ll)
    M = tail_length(S, r_eff)
    lw = np.min(ll) - ll
    order = np.argsort(lw, kind="stable")
    cut = max(lw[order[S - M - 1]], LOG_TINY)
    tail = np.flatnonzero(lw > cut)
    k = np.inf
    if len(tail) > 4:
        ti = tail[np.argsort(lw[tail], kind="stable")]
        n = len(ti)
        x = np.exp(lw[ti]) - np.exp(cut)
        k, sigma = gpdfit(x)
        if np.isfinite(k):
            lw = lw.copy()
            lw[ti] = np.log(gpinv(np.arange(0.5, n) / n, k, sigma) + np.exp(cut))
            lw[lw > 0] = 0
    m = np.max(lw)
    lw = lw - (m + np.log(np.sum(np.exp(lw - m))))
    return {"lw": lw, "k": k, "tail": np.sort(tail), "cut": cut}


def logsumexp(a):
    m = np.max(a)
    return m + np.log(np.sum(np.exp(a - m)))


def loo(ll, r_eff=1.0):
    """ll [S, N] -> the "loo" dict of sample_summary (plus "tails": the tail draws of each point)."""
    ll = np.asarray(ll, dtype=np.float64)
    S, N = ll.shape
    cols = {k: np.full(N, np.nan) for k in ("elpd_loo", "lppd", "p_loo", "elpd_waic", "p_waic", "pareto_k")}
    tails = []
    for i in range(N):
        x = ll[:, i]
        if not np.all(np.isfinite(x)):
            tails.append(None)
            continue
        r = psis_point(x, r_eff)
        lppd = logsumexp(x) - np.log(S)
        cols["lppd"][i] = lppd
        cols["p_waic"][i] = np.var(x)
        cols["elpd_waic"][i] = lppd - np.var(x)
        cols["elpd_loo"][i] = logsumexp(r["lw"] + x)
        cols["p_loo"][i] = lppd - cols["elpd_loo"][i]
        cols["pareto_k"][i] = r["k"]
        tails.append(r["tail"])
    thr = min(1 - 1 / np.log10(S), 0.7)
    out = {"elpd_loo": np.sum(cols["elpd_loo"]), "se_elpd_loo": np.sqrt(N * np.var(cols["elpd_loo"])), "p_loo": np.sum(cols["p_loo"]),
           "elpd_waic": np.sum(cols["elpd_waic"]), "se_elpd_waic": np.sqrt(N * np.var(cols["elpd_waic"])),
           "p_waic": np.sum(cols["p_waic"])}
    out["looic"], out["waic"] = -2 * out["elpd_loo"], -2 * out["elpd_waic"]
    out.update(pointwise=cols, pareto_k_threshold=thr, n_high_k=int(np.sum(cols["pareto_k"] > thr)), n_draws=S, points=N, tails=tails)
    return out
