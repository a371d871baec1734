"""Reference for the split-chain records of amwg_summary_autocov (the ESS and split R-hat of sample_summary(..., diagnostics=True) and
the rank-normalised ones of diagnostics="rank"), a worst-case bound for what the device computes, and the estimators' decisions
taken over that bound.

record() restates the records from the draws:
  - the half-chain means bit for bit as the device forms them (csrc/amwg_autocov.cuh): a strictly sequential sum in row order
    divided by h, with run_mean's constant rule, and the indicators' counts over h. So the centred values fl(v - m) (times the
    draws series' power of two, ess_ref.autocov_scale) and the indicator values are the device's bits; all the remaining error is in
    the accumulation.
  - every lag sum sum_m sum_n d_mn d_m,n+t near exactly: each product rounded once in double (off by at most u of itself; when a
    product could leave the normal doubles, in x86 extended precision instead: 64-bit significand, exponents to 2^16383), the
    products summed in extended precision (numpy's pairwise sum and the chunk sums add at most (64 + log2 n) 2^-64 sum |.|), then
    one rounding to double. Off the exact sum by at most 3 u sum |d_n d_n+t|.
  - the moment fields: M exactly, the mean and the M2 of the (scaled) half-chain means with fsum, sum_w = the lag-0 sum.
  - the indicators' lag sums from integer pair counts (indicator_lag_sums), to the same precision and far faster.
bound() follows the device (u = 2^-53, gamma_k = k u / (1 - k u), Higham 3.1; nested_ref):
  lag sum   each thread adds its products by a sequential fma over its ceil(C / (chain_ctas(C) 256)) chains x 2 halves x h terms,
            then cta_sum's 8-level tree over 256 threads, then amwg_merge_sums_kernel's strided sum of <= 5 of the <= 1184 CTA partials
            per thread and another 8-level tree: at most n = 2 cpt h + 21 roundings on any path, so gamma_{n+1} sum |d_n d_n+t|,
            plus the reference's own 3 u of it.
  record    the four fields through nested_ref._chan_bound with leaf means exact and leaf sum_w off by gamma_h of their size, at
            most 2 cpt + 20 merge steps (a thread's halves, the 256-thread tree, K_m2's two strided merges and 1024-thread tree).
  Higham's model has no underflow term: every field also gets (n + M) 2^-1074 of absolute slack, which covers the subnormal
  products and means of an unscaled series and is far below every normal value.
interval() carries those bounds through GeyerESS (bayes_js_b200/summary.py) as intervals: rho(t), var+ and W, then every
comparison of Geyer's initial positive and initial monotone steps and the tau floor. It returns the interval of the ESS and of
var+ / W, or None when a comparison falls inside its interval (undecided). Test infrastructure only."""
import math

import numpy as np

from ess_ref import autocov_scale, halves
from nested_ref import U, _chan_bound, gamma

TINY = 2.0 ** -1074
XP = np.longdouble
assert np.finfo(XP).nmant >= 63, "the exact lag sums need an extended-precision long double (64-bit significand)"


def chain_ctas(C: int) -> int:
    return min((C + 255) // 256, 1184)                           # csrc/amwg_summary.cuh


def device_means(y: np.ndarray) -> np.ndarray:
    """y [M, h] -> the device's half-chain means: a sequential sum in row order over h, then run_mean's rule"""
    M, h = y.shape
    s = np.zeros(M)
    with np.errstate(invalid="ignore", over="ignore"):
        for n in range(h):
            s = s + y[:, n]
        m = s / h
    same = np.all(y.view(np.uint64) == y[:, :1].view(np.uint64), axis=1) & np.isfinite(y[:, 0])
    return np.where(same, y[:, 0], m)


def centred(x: np.ndarray, thr, e: int, s: int):
    """the device's centred values [M, h] and half-chain means [M] of series s of entry e (s = 0: the draws, scaled when thresholds
    are given; s = 1, 2: the indicators of thr[e][0], thr[e][1])"""
    y = halves(np.asarray(x[:, e, :], dtype=np.float64))
    M, h = y.shape
    with np.errstate(invalid="ignore", over="ignore"):
        if s == 0:
            m = device_means(y)
            d = y - m[:, None]
            if thr is not None:
                sc = autocov_scale(*thr[e])
                d, m = d * sc, m * sc
            return d, m
        q = thr[e][s - 1]
        m = (y <= q).sum(axis=1).astype(np.float64) / h
        return np.where(y <= q, 1.0 - m[:, None], -m[:, None]), m


def lag_sum(d: np.ndarray, t: int, wide=None):
    """-> (sum_m sum_n d_mn d_m,n+t within 3 u sum |.| of exact, sum |d_mn d_m,n+t|): the sums in extended precision, the products
    too when `wide` (module docstring); wide=None decides from d"""
    M, h = d.shape
    if wide is None:
        wide = needs_wide(d)
    tot, ab = XP(0), XP(0)
    step = max(1, (1 << 23) // h)                               # half-chains at a time: bounded temporaries at 2^21 half-chains
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(0, M, step):
            a = d[c:c + step, :h - t]
            p = (a.astype(XP) if wide else a) * d[c:c + step, t:]
            tot += p.astype(XP).sum()
            ab += np.abs(p).sum()
    return float(tot), float(ab)


def needs_wide(d: np.ndarray) -> bool:
    """whether a product of two values of d could leave the normal doubles: some |d| >= 2^500, or a nonzero one below 2^-500"""
    a = np.abs(d)
    with np.errstate(invalid="ignore"):
        return not (np.nanmax(a, initial=0.0) < 2.0 ** 500 and np.all((a >= 2.0 ** -500) | (a == 0) | np.isnan(a)))


def indicator_lag_sums(x: np.ndarray, thr, e: int, s: int, lags):
    """lag_sum of indicator series s (1, 2) of entry e at every lag in `lags`, from integer pair counts: a half-chain's centred
    indicator takes two values, A = fl(1 - m) and B = -m, so sum_n d_n d_n+t = A^2 N11 + A B (N10 + N01) + B^2 N00 with N the
    counts of the (bit, bit) pairs at lag t. N11 is an integer autocorrelation of 0/1 sequences, formed by FFT and rounded
    (every count is below 2^31, the FFT's error below 1/4, asserted); the rest follow from prefix counts. The combination runs in
    extended precision, as lag_sum."""
    y = halves(np.asarray(x[:, e, :], dtype=np.float64))
    M, h = y.shape
    b = (y <= thr[e][s - 1]).astype(np.float64)
    m = b.sum(axis=1) / h
    A, B = (1.0 - m).astype(XP), (-m).astype(XP)
    n = 1 << int(np.ceil(np.log2(2 * h)))
    f = np.fft.rfft(b, n=n, axis=1)
    ac = np.fft.irfft(f * np.conj(f), n=n, axis=1)[:, :h]
    n11 = np.rint(ac)
    assert np.max(np.abs(ac - n11)) < 0.25
    cs = np.concatenate([np.zeros((M, 1)), np.cumsum(b, axis=1)], axis=1)          # cs[:, k] = ones among the first k
    tot, ab = [], []
    for t in lags:
        first, last = cs[:, h - t], cs[:, h] - cs[:, t]                            # ones among n < h - t, and among n >= t
        c11 = n11[:, t]
        c10 = first + last - 2 * c11
        c00 = (h - t) - c11 - c10
        terms = np.stack([A * A * c11.astype(XP), A * B * c10.astype(XP), B * B * c00.astype(XP)])
        tot.append(float(terms.sum()))
        ab.append(float(np.abs(terms).sum()))
    return tot, ab


def record(x: np.ndarray, thr, lag0: int, n_lags: int, series=None):
    """x [rows, entries, chains] -> (exact [entries, series, 4 + n_lags], bound [same]) for amwg_summary_autocov(x, thr, lag0, n_lags);
    only the series listed in `series` when given (the others' bounds NaN: not checked)"""
    rows, entries, C = x.shape
    h = rows // 2
    ns = 1 if thr is None else 3
    cpt = -(-C // (chain_ctas(C) * 256))
    n_ops = 2 * cpt * h + 21
    steps = 2 * cpt + 20
    exact = np.zeros((entries, ns, 4 + n_lags))
    bound = np.zeros((entries, ns, 4 + n_lags))
    for e in range(entries):
        for s in range(ns):
            if series is not None and s not in series:
                exact[e, s, 0] = 2 * C
                bound[e, s] = np.nan
                continue
            d, m = centred(x, thr, e, s)
            M = d.shape[0]
            slack = (n_ops + M) * TINY
            with np.errstate(invalid="ignore", over="ignore"):
                sw_leaf = np.sum(d * d, axis=1)
                if not np.all(np.isfinite(m)):
                    mean = m2 = np.nan                           # not checked: the bound below is NaN
                else:
                    mean = float(m[0]) if np.all(m.view(np.uint64) == m[:1].view(np.uint64)) else math.fsum(m) / M
                    m2 = math.fsum((m - mean) ** 2)
            lags = [0] + list(range(lag0, lag0 + n_lags))
            if s == 0:
                wide = needs_wide(d)
                sums = [lag_sum(d, t, wide) for t in lags]
            else:
                sums = list(zip(*indicator_lag_sums(x, thr, e, s, lags)))
            sw = sums[0][0]
            exact[e, s, :4] = (M, mean, m2, sw)
            if np.all(np.isfinite(d)) and np.all(np.isfinite(m)):
                bm, bm2, bsw = _chan_bound(m, [0.0], [0.0], [0.0], sw_leaf, gamma(h) * sw_leaf, steps=steps)
                bound[e, s, :4] = (0.0, bm + slack, bm2 + slack, bsw + 3 * U * abs(sw) + slack)
            else:
                bound[e, s, :4] = np.nan
            for k in range(n_lags):
                tot, ab = sums[1 + k]
                exact[e, s, 4 + k] = tot
                bound[e, s, 4 + k] = (gamma(n_ops + 1) + 3 * U) * ab + slack if np.isfinite(ab) else np.nan
    return exact, bound


def check_record(got, exact, bound, what=""):
    """got (the device's or the host build's record) against record()'s: M equal, every finite field within the bound; a series
    with a non-finite centred value only where the device's is not finite too"""
    got = np.asarray(got)
    assert got.shape == exact.shape, (what, got.shape, exact.shape)
    assert np.array_equal(got[:, :, 0], exact[:, :, 0]), what
    fin = np.isfinite(bound)
    err = np.abs(got - exact)
    ok = ~fin | (err <= bound)
    assert np.all(ok), (what, np.argwhere(~ok)[:5], (err / np.where(bound > 0, bound, 1))[~ok][:5])
    return float(np.max(np.where(fin & (bound > 0), err / np.where(bound > 0, bound, 1), 0.0)))


# ---- Geyer's decisions over the bound -------------------------------------------------------------------------------------------
class Undecided(Exception):
    pass


def _add(a, b):
    return (a[0] + b[0], a[1] + b[1])


def _div(a, b):                                                  # b > 0
    qs = (a[0] / b[0], a[0] / b[1], a[1] / b[0], a[1] / b[1])
    return (min(qs), max(qs))


def _pad(a, rel):                                                # the host's own roundings: rel times the magnitude
    w = rel * max(abs(a[0]), abs(a[1]))
    return (a[0] - w, a[1] + w)


def _gt(a, b):
    """a > b for every value of the intervals (True), for none (False), else Undecided"""
    if a[0] > b[1]:
        return True
    if a[1] <= b[0]:
        return False
    raise Undecided


def _ge(a, b):
    if a[0] >= b[1]:
        return True
    if a[1] < b[0]:
        return False
    raise Undecided


def _wv(rec, bnd, h: int):
    M, _mean, m2, sw = rec[:4]
    W = (max(sw - bnd[3], 0.0) / (M * (h - 1)), (sw + bnd[3]) / (M * (h - 1)))
    B = (max(m2 - bnd[2], 0.0) / (M - 1), (m2 + bnd[2]) / (M - 1))
    W, B = _pad(W, 2 * U), _pad(B, 2 * U)
    return W, _pad(_add(((h - 1) / h * W[0], (h - 1) / h * W[1]), B), 4 * U)


def ratio_interval(rec, bnd, h: int):
    """(lo, hi) of var+ / W (the square of rhat_split, and of either half of rhat_rank) over the bound, or None when W may be 0"""
    W, V = _wv(rec, bnd, h)
    if not W[0] > 0:
        return None
    return _pad(_div(V, W), 8 * U)                               # and sqrt then squared by the caller


def interval(rec, bnd, h: int):
    """rec, bnd: one series' [4 + n] exact record and bound, the lags 0..n-1. -> (ess (lo, hi), var+ / W (lo, hi)), or None when
    undecided. Raises ValueError when the lags run out before Geyer's loop ends."""
    Mh = rec[0] * h
    W, V = _wv(rec, bnd, h)
    if not W[0] > 0:
        return None
    ratio = ratio_interval(rec, bnd, h)
    sums = rec[4:]
    rho = []
    for t in range(len(sums)):
        s = ((sums[t] - bnd[4 + t]) / Mh, (sums[t] + bnd[4 + t]) / Mh)
        num = (W[0] - s[1], W[1] - s[0])
        q = _div(num, V)
        w = 8 * U * (1.0 + max(abs(q[0]), abs(q[1])))       # the host's roundings of 1 - (W - s) / var+
        rho.append((1.0 - q[1] - w, 1.0 - q[0] + w))
    zero = (0.0, 0.0)
    try:
        r = [(1.0, 1.0), rho[1]]
        ev, od, t = (1.0, 1.0), rho[1], 1
        while t < h - 3 and _gt(_add(ev, od), zero):
            if t + 2 >= len(rho):
                raise ValueError("more lags needed")
            ev, od = rho[t + 1], rho[t + 2]
            r.extend([zero] * (t + 3 - len(r)))
            if _ge(_add(ev, od), zero):
                r[t + 1], r[t + 2] = ev, od
            t += 2
        max_t = t - 2
        r.extend([zero] * (max_t + 2 - len(r)))
        if _gt(ev, zero):
            r[max_t + 1] = ev
        t = 1
        while t <= max_t - 2:
            a, b = _add(r[t + 1], r[t + 2]), _add(r[t - 1], r[t])
            if _gt(a, b):
                r[t + 1] = r[t + 2] = _pad((b[0] / 2, b[1] / 2), 2 * U)
            t += 2
        acc = (0.0, 0.0)
        for v in r[:max_t + 1]:
            acc = _add(acc, v)
        tau = _add((-1.0 + 2.0 * acc[0], -1.0 + 2.0 * acc[1]), r[max_t + 1])
        w = gamma(max_t + 4) * (1.0 + 2.0 * sum(max(abs(v[0]), abs(v[1])) for v in r[:max_t + 2]))
        tau = (tau[0] - w, tau[1] + w)                           # the host's roundings of the sum
        floor = 1.0 / np.log10(Mh)
        floor = (floor * (1 - 4 * U), floor * (1 + 4 * U))
        if _gt(tau, floor):
            ess = (Mh / tau[1], Mh / tau[0])
        else:
            ess = (Mh / floor[1], Mh / floor[0])
    except Undecided:
        return None
    return _pad(ess, 2 * U), ratio


def inside(v, iv) -> bool:
    return iv[0] <= v <= iv[1]
