"""Test infrastructure: LOO-PIT restated in numpy (Gabry, Simpson, Vehtari, Betancourt & Gelman 2019, "Visualization in Bayesian
workflow"; Säilynoja, Bürkner & Vehtari 2022; ArviZ's loo_pit) on the smoothed weights of tests/loo_ref.py's psis_point, with the
tie rule of DESIGN.md §4.9: the tail sorted by ascending lw splits into maximal runs of equal ll, and every draw of a run takes the
run's mean weight. Independent of the product: it sorts and sums with numpy."""
import numpy as np

import loo_ref


def point(ll, yrep, y, r_eff=1.0, tie_mean=True):
    """One point: ll, yrep [S], the observation y -> (pit, pit_equal, k). tie_mean=False leaves the tail's weights as psis_point
    ranks them (ties broken by draw index, a stable sort): ArviZ's loo_pit."""
    ll = np.asarray(ll, dtype=np.float64)
    yrep = np.asarray(yrep, dtype=np.float64)
    if not np.all(np.isfinite(ll)):
        return np.nan, np.nan, np.nan
    r = loo_ref.psis_point(ll, r_eff)
    w = np.exp(r["lw"])                                            # normalised: sums to 1 up to rounding
    if tie_mean and r["tail"].size:
        raw = np.min(ll) - ll
        ti = r["tail"][np.argsort(raw[r["tail"]], kind="stable")]     # ranks j = 0..n-1 of the tail
        v = ll[ti]
        start = np.flatnonzero(np.concatenate([[True], v[1:] != v[:-1]]))
        for a, b in zip(start, np.concatenate([start[1:], [len(v)]])):
            w[ti[a:b]] = np.sum(w[ti[a:b]]) / (b - a)
    D = np.sum(w)
    le = np.sum(w[yrep <= y]) / D
    eq = np.sum(w[yrep == y]) / D
    return min(1.0, le), min(1.0, eq), r["k"]


def loo_pit(ll, yrep, y, r_eff=1.0, tie_mean=True):
    """ll, yrep [S, N], y [N] -> {"pit", "pit_equal", "pareto_k"} [N] each, "pareto_k_threshold", "n_high_k"."""
    ll = np.asarray(ll, dtype=np.float64)
    S, N = ll.shape
    cols = {k: np.full(N, np.nan) for k in ("pit", "pit_equal", "pareto_k")}
    for i in range(N):
        cols["pit"][i], cols["pit_equal"][i], cols["pareto_k"][i] = point(ll[:, i], yrep[:, i], y[i], r_eff, tie_mean)
    thr = min(1 - 1 / np.log10(S), 0.7)
    with np.errstate(invalid="ignore"):
        n_high = int(np.sum(cols["pareto_k"] > thr))
    return dict(cols, pareto_k_threshold=thr, n_high_k=n_high)
