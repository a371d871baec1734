"""Reference for the nested R-hat of sample_summary(..., nested=M): the records of amwg_summary_nested restated from the definition
with math.fsum (every value within a few roundings of the exact one), and a worst-case forward-error bound for what the device
computes.

The bound follows the device's operations (csrc/amwg_nested.cuh), in the manner of tests/cov_ref.py (u = 2^-53,
gamma_k = k u / (1 - k u), Higham 3.1):
  chain     m^ = fl(fl(sum_r x_r) / N) is off the mean by at most dlt = gamma_{N+1} mean_r |x_r|. The two-pass M2 uses m^:
            sum_r (x_r - m^)^2 = sum_r (x_r - m)^2 + N (m - m^)^2 exactly, and the roundings of the differences, squares and the sum
            add at most gamma_{N+2} sum_r (|x_r - m| + dlt)^2.
  merge     Chan's merge of n records whose means lie in [lo, hi] (A = max |mean|, D = hi - lo), each mean off by at most e_v.
            A step's mean a + (b - a) nb / n is a convex combination: it adds at most 3 gamma_4 A, and inherited errors do not
            grow. A mean passes through at most L = n + 20 steps (the sequential merges in a thread, the 256- and 1024-thread
            trees), so its error is at most E = e_v + 3 L gamma_4 A. A step's M2 term w d^2 (w = na nb / n) has |d| <= D and d off
            by at most De = 2 E + u D; over the steps sum w <= n (1 + log2 n) (a binary merge tree). So the M2 is off by at most
            n (1 + log2 n) (2 D De + De^2) + gamma_{L+6} (n (1 + log2 n) (D + De)^2 + sum of the leaves' M2) + the leaves' M2
            errors, and a sum of the leaves' sum_w by at most gamma_L (sum of |sum_w|) + their errors.
  unit      B~_k + W-_k: two divisions and an addition, gamma_3 relative, on top of the errors of M2 / (M - 1) and sum_w / (M (N - 1)).
The superchain level merges the M chain records of a superchain; the total level merges the K unit records.
Values that all have the bits of the first, a finite one, have that value as their exact mean (and M2 = 0), at every level.

record_loop restates the records chain by chain with fsum; record() is the same vectorised over chains and superchains, for blocks
of 2^20 chains: each chain's sums by a compensated sum along the rows (Sum2, tests/moments_ref.py), a superchain's by Sum2 across
its M chains, and fsum only across the superchains. Sum2 is off by at most u |sum| + gamma_{n-1}^2 sum |x|, one rounding more
than fsum and far inside the bound; test_summary_nested_host checks the two forms against each other. Test infrastructure only."""
import math

import numpy as np

U = 2.0 ** -53


def gamma(k) -> float:
    k = float(k)
    return k * U / (1.0 - k * U)


def _chan_bound(means, e_v, m2_leaf, m2_err, sw_leaf, sw_err, steps=None):
    """Bounds (mean, M2, sum_w) of the Chan merge of len(means) records, as derived in the module docstring; `steps`: the most
    merge steps a mean passes through, when fewer than L = n + 20 are known."""
    n = len(means)
    L = n + 20 if steps is None else steps
    A = float(np.max(np.abs(means)))
    D = float(np.max(means) - np.min(means))
    E = float(np.max(e_v)) + 3 * L * gamma(4) * A
    De = 2 * E + U * D
    ws = n * (1 + math.log2(n)) if n > 1 else 0.0
    b_m2 = ws * (2 * D * De + De * De) + gamma(L + 6) * (ws * (D + De) ** 2 + float(np.sum(np.abs(m2_leaf)))) + float(np.sum(m2_err))
    b_sw = gamma(L) * float(np.sum(np.abs(sw_leaf))) + float(np.sum(sw_err))
    return E, b_m2, b_sw


def _same(v, axis=0):
    """whether the values along `axis` all have the bits of the first, a finite one: their exact mean is that value"""
    v = np.asarray(v, dtype=np.float64)
    first = np.take(v, [0], axis=axis)
    return np.all(v.view(np.uint64) == first.view(np.uint64), axis=axis) & np.isfinite(np.take(v, 0, axis=axis))


def _fmean(v):
    """mean of v with fsum, exact for values that all have the same bits"""
    v = np.asarray(v, dtype=np.float64)
    return float(v[0]) if _same(v) else math.fsum(v) / len(v)


def _chain(col):
    """exact (mean, M2) of one chain, and the device's error bounds for both"""
    N = len(col)
    m = _fmean(col)
    m2 = math.fsum((col - m) ** 2)
    dlt = gamma(N + 1) * float(np.mean(np.abs(col)))
    e_m2 = N * dlt * dlt + gamma(N + 2) * float(np.sum((np.abs(col - m) + dlt) ** 2))
    return m, m2, dlt, e_m2


def _superchain(x, e, c0, c1):
    """chain-level record (n, mean, M2, sum_w) of local chains [c0, c1) of entry e, exact, and its bounds"""
    ch = [_chain(np.asarray(x[:, e, c], dtype=np.float64)) for c in range(c0, c1)]
    means = np.array([c[0] for c in ch])
    mean = _fmean(means)
    m2 = math.fsum((means - mean) ** 2)
    sw = math.fsum([c[1] for c in ch])
    bm, bm2, bsw = _chan_bound(means, [c[2] for c in ch], [0.0], [0.0], [c[1] for c in ch], [c[3] for c in ch])
    return np.array([len(ch), mean, m2, sw]), np.array([0.0, bm, bm2, bsw])


def _chan_bound_v(means, e_v, sw_leaf, sw_err):
    """_chan_bound(means[k], e_v[k], [0.0], [0.0], sw_leaf[k], sw_err[k]) for every row k of the [K, n] arrays at once"""
    n = means.shape[1]
    L = n + 20
    A = np.max(np.abs(means), axis=1)
    D = np.max(means, axis=1) - np.min(means, axis=1)
    E = np.max(e_v, axis=1) + 3 * L * gamma(4) * A
    De = 2 * E + U * D
    ws = n * (1 + math.log2(n)) if n > 1 else 0.0
    b_m2 = ws * (2 * D * De + De * De) + gamma(L + 6) * (ws * (D + De) ** 2)
    b_sw = gamma(L) * np.sum(np.abs(sw_leaf), axis=1) + np.sum(sw_err, axis=1)
    return E, b_m2, b_sw


def record(x: np.ndarray, first_chain: int, M: int):
    """record_loop vectorised (module docstring): the complete superchains at once, the (at most two) cut ones by _superchain"""
    from moments_ref import _sum2
    x = np.asarray(x, dtype=np.float64)
    rows, entries, C = x.shape
    k0, k1 = first_chain // M, (first_chain + C - 1) // M
    kf, kl = -(-first_chain // M), (first_chain + C) // M - 1                    # the complete superchains [kf, kl]
    exact = np.zeros((entries, 14))
    bound = np.zeros((entries, 14))
    exact[:, [4, 9]] = -1.0
    if kl >= kf:
        K = kl - kf + 1
        d = x[:, :, kf * M - first_chain:(kl + 1) * M - first_chain]
        with np.errstate(invalid="ignore", over="ignore"):
            m = np.where(_same(d), d[0], _sum2(d) / rows)                       # [entries, chains]
            dev = d - m[None]
            m2c = _sum2(dev * dev)
            dlt = gamma(rows + 1) * np.mean(np.abs(d), axis=0)
            e_m2 = rows * dlt * dlt + gamma(rows + 2) * np.sum((np.abs(dev) + dlt[None]) ** 2, axis=0)
            for e in range(entries):
                cm = m[e].reshape(K, M)
                sk = np.where(_same(cm, axis=1), cm[:, 0], _sum2(cm.T) / M)       # superchain means
                m2 = _sum2(((cm - sk[:, None]) ** 2).T)
                sw = _sum2(m2c[e].reshape(K, M).T)
                bm, bm2, bsw = _chan_bound_v(cm, dlt[e].reshape(K, M), m2c[e].reshape(K, M), e_m2[e].reshape(K, M))
                bt = m2 / (M - 1) if M > 1 else np.zeros(K)
                wt = sw / (M * (rows - 1)) if rows > 1 else np.zeros(K)
                eb = (bm2 / (M - 1) if M > 1 else 0.0) + (bsw / (M * (rows - 1)) if rows > 1 else 0.0) + gamma(3) * (bt + wt)
                mean = _fmean(sk)
                exact[e, :4] = (K, mean, math.fsum((sk - mean) ** 2), math.fsum(bt + wt))
                tb = _chan_bound(sk, bm, [0.0], [0.0], bt + wt, eb)
                bound[e, :4] = (0.0, *tb)
    for k in sorted({k0, k1}):
        c0, c1 = max(k * M - first_chain, 0), min((k + 1) * M - first_chain, C)
        if c1 - c0 == M:
            continue
        slot = 0 if k == k0 else 1                                   # the first superchain, or the last when it is another one
        for e in range(entries):
            rec, b = _superchain(x, e, c0, c1)
            exact[e, 4 + 5 * slot:9 + 5 * slot] = (k, *rec)
            bound[e, 5 + 5 * slot:9 + 5 * slot] = b
    return exact, bound


def record_loop(x: np.ndarray, first_chain: int, M: int):
    """x [rows, entries, chains] of the global chains [first_chain, first_chain + chains) -> (exact [entries, 14], bound
    [entries, 14]) in amwg_summary_nested's layout: the complete superchains' (K, mean, M2, sum of B~_k + W-_k), then the cut
    records {id, chains, mean, M2, sum_w} of the first and the last superchain when the range cuts them."""
    rows, entries, C = x.shape
    k0, k1 = first_chain // M, (first_chain + C - 1) // M
    exact = np.zeros((entries, 14))
    bound = np.zeros((entries, 14))
    for e in range(entries):
        units, ubnd = [], []
        cuts = []
        for k in range(k0, k1 + 1):
            c0, c1 = max(k * M - first_chain, 0), min((k + 1) * M - first_chain, C)
            rec, b = _superchain(x, e, c0, c1)
            if c1 - c0 < M:
                cuts.append((k, rec, b))
                continue
            bt = rec[2] / (M - 1) if M > 1 else 0.0
            wt = rec[3] / (M * (rows - 1)) if rows > 1 else 0.0
            eb = (b[2] / (M - 1) if M > 1 else 0.0) + (b[3] / (M * (rows - 1)) if rows > 1 else 0.0) + gamma(3) * (bt + wt)
            units.append((rec[1], bt + wt))
            ubnd.append((b[1], eb))
        if units:
            means = np.array([v[0] for v in units])
            K = len(units)
            mean = _fmean(means)
            exact[e, :4] = (K, mean, math.fsum((means - mean) ** 2), math.fsum([v[1] for v in units]))
            bm, bm2, bsw = _chan_bound(means, [b[0] for b in ubnd], [0.0], [0.0], [v[1] for v in units], [b[1] for b in ubnd])
            bound[e, :4] = (0.0, bm, bm2, bsw)
        for slot in range(2):
            exact[e, 4 + 5 * slot] = -1.0
        for k, rec, b in cuts:
            slot = 0 if k == k0 else 1                               # the first superchain, or the last when it is another one
            exact[e, 4 + 5 * slot:9 + 5 * slot] = (k, *rec)
            bound[e, 5 + 5 * slot:9 + 5 * slot] = b
    return exact, bound


def rhat_nested(x: np.ndarray, M: int) -> np.ndarray:
    """The definition over whole superchains of x [rows, entries, chains] (global chains from 0), with fsum: per entry
    sqrt(1 + B^ / W^); NaN when K < 2, W^ = 0 or a draw is not finite."""
    rows, entries, C = x.shape
    K = C // M
    out = np.full(entries, np.nan)
    for e in range(entries):
        d = np.asarray(x[:, e, :], dtype=np.float64)
        if K < 2 or not np.all(np.isfinite(d)):
            continue
        cm = np.array([math.fsum(d[:, c]) / rows for c in range(C)])
        sk = np.array([math.fsum(cm[k * M:(k + 1) * M]) / M for k in range(K)])
        xb = math.fsum(sk) / K
        Bh = math.fsum((sk - xb) ** 2) / (K - 1)
        Wh = 0.0
        terms = []
        for k in range(K):
            bt = math.fsum((cm[k * M:(k + 1) * M] - sk[k]) ** 2) / (M - 1) if M > 1 else 0.0
            wt = (math.fsum(math.fsum((d[:, c] - cm[c]) ** 2) for c in range(k * M, (k + 1) * M)) / (M * (rows - 1))) if rows > 1 else 0.0
            terms.append(bt + wt)
        Wh = math.fsum(terms) / K
        if Wh > 0:
            out[e] = math.sqrt(1.0 + Bh / Wh)
    return out


def rhat_interval(rec: np.ndarray, bnd: np.ndarray):
    """(lo, hi) of rhat_nested over every total-level record within `bnd` of the exact `rec` ([entries, 4] each), plus the few
    roundings of finalize_nested."""
    K, m2, sw = rec[:, 0], rec[:, 2], rec[:, 3]
    with np.errstate(invalid="ignore", divide="ignore"):
        Blo, Bhi = np.maximum(m2 - bnd[:, 2], 0) / (K - 1), (m2 + bnd[:, 2]) / (K - 1)
        Wlo, Whi = np.maximum(sw - bnd[:, 3], 0) / K, (sw + bnd[:, 3]) / K
        lo = np.sqrt(1 + Blo / Whi) * (1 - gamma(6))
        hi = np.sqrt(1 + Bhi / Wlo) * (1 + gamma(6))
    return lo, hi


def check_record(got, x: np.ndarray, first_chain: int, M: int, what=""):
    """got [entries, 14] from the device (or its host build) against record(): ids and counts equal, values within the bound."""
    exact, bound = record(x, first_chain, M)
    got = np.asarray(got)
    for cols in ((0,), (4, 5), (9, 10)):
        assert np.array_equal(got[:, cols], exact[:, cols]), (what, cols, got[:, cols], exact[:, cols])
    err = np.abs(got - exact)
    ok = (err <= bound) | (np.isnan(got) & np.isnan(exact))
    assert np.all(ok), (what, np.argwhere(~ok)[:5], (err / np.where(bound > 0, bound, 1))[~ok][:5])
    return exact, bound
