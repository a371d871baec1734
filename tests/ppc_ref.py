"""Restatement of the posterior predictive checks of sample_summary(..., ppc=...) (DESIGN.md §4.8), independent of the product:
the samplers of csrc/amwg_ppc.cuh written from the papers over the oracle's primitives (its Philox stream orc_stream_uniform and
fdlibm orc_log / orc_exp), the per-dataset statistics and the "ppc" dict from a matrix of replicated data. Python floats are
IEEE-754 doubles and every operation below is one rounding, as on the device (--fmad=false)."""
import math

import mpmath
import numpy as np

FAMILIES = ["norm", "lnorm", "cauchy", "laplace", "logis", "exp", "weibull", "pareto", "unif", "gamma", "invgamma", "beta", "t",
            "bern", "pois", "binom", "nbinom"]
ARITY = {"exp": 1, "bern": 1, "pois": 1, "t": 3}
STREAM_BASE = 1 << 62
POINT_SHIFT = 16
NAN = float("nan")

mpmath.mp.prec = 200
LOG_FACTORIAL = [float(mpmath.loggamma(k + 1)) for k in range(128)]          # correctly rounded (checked in the tests)


def position(row, points, i):
    return STREAM_BASE + ((row * points + i) << POINT_SHIFT)


class Philox:
    """uniforms of global chain `chain` from stream position `pos` on"""

    def __init__(self, O, seed, chain, pos):
        self.O, self.seed, self.chain, self.pos, self.n = O, seed, chain, pos, pos
        self.end = pos + (1 << POINT_SHIFT)

    def u(self):
        v = self.O.orc_stream_uniform(self.seed, self.chain, self.n)
        self.n += 1
        return v

    def spent(self):
        return self.n > self.end

    def used(self):
        return self.n - self.pos


class Tape:
    def __init__(self, O, tape):
        self.O, self.t, self.n = O, list(tape), 0

    def u(self):
        v = self.t[self.n] if self.n < len(self.t) else 0.5
        self.n += 1
        return v

    def spent(self):
        return self.n > len(self.t)

    def used(self):
        return self.n


def rnorm(s):
    """mcmc.js:43-54, v / u"""
    log = s.O.orc_log
    while True:
        u = s.u()
        v = 1.7156 * (s.u() - 0.5)
        x = u - 0.449871
        y = abs(v) + 0.386595
        q = x * x + y * (0.19600 * y - 0.25472 * x)
        if not (q > 0.27597 and (q > 0.27846 or v * v > -4 * log(u) * u * u)):
            return v / u


def log_factorial(O, k):
    if k < 128.0:
        return LOG_FACTORIAL[int(k)]
    r = 1.0 / k
    r2 = r * r
    return (k + 0.5) * O.orc_log(k) - k + 0.91893853320467274178 + r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0)))


def expo(s):
    return -s.O.orc_log(1.0 - s.u())


def gamma_mt(s, a):
    """Marsaglia & Tsang (2000), ACM TOMS 26(3), without the squeeze"""
    log = s.O.orc_log
    d = a - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * d)
    while not s.spent():
        while True:
            x = rnorm(s)
            v = 1.0 + c * x
            if not (v <= 0.0 and not s.spent()):
                break
        v = v * v * v
        U = s.u()
        lv = log(v) if v > 0 else NAN
        if log(U) < 0.5 * x * x + d - d * v + d * lv:
            return d * v
    return NAN


def gamma1(s, a):
    if a >= 1.0:
        return gamma_mt(s, a)
    g = gamma_mt(s, a + 1.0)
    return g * s.O.orc_exp(s.O.orc_log(s.u()) / a)


def pois(s, lam):
    O = s.O
    if lam < 10.0:
        L = O.orc_exp(-lam)
        p, k = 1.0, -1.0
        while True:
            k += 1.0
            p = p * s.u()
            if not (p > L and not s.spent()):
                return k
    # PTRS: W. Hoermann, Insurance: Mathematics and Economics 12 (1993) 39-45
    slam, loglam = math.sqrt(lam), O.orc_log(lam)
    b = 0.931 + 2.53 * slam
    a = -0.059 + 0.02483 * b
    lia = O.orc_log(1.1239 + 1.1328 / (b - 3.4))
    vr = 0.9277 - 3.6224 / (b - 2.0)
    while not s.spent():
        U = s.u() - 0.5
        V = s.u()
        us = 0.5 - abs(U)
        k = math.floor((2.0 * a / us + b) * U + lam + 0.43) if us > 0 else -math.inf
        k = float(k)
        if k < 0.0:
            continue
        if us >= 0.07 and V <= vr:
            return k
        if us < 0.013 and V > us:
            continue
        if O.orc_log(V) + lia - O.orc_log(a / (us * us) + b) <= -lam + k * loglam - log_factorial(O, k):
            return k
    return NAN


def binom_low(s, n, q):
    O = s.O
    if n * q < 10.0:
        qn = O.orc_exp(n * O.orc_log(1.0 - q))
        r = q / (1.0 - q)
        g = r * (n + 1.0)
        while not s.spent():
            U, f, k = s.u(), qn, 0.0
            while True:
                if U < f:
                    return k
                if k >= n:
                    break
                U = U - f
                k += 1.0
                f = f * (g / k - r)
        return NAN
    # BTRS: W. Hoermann, J. Statist. Comput. Simul. 46 (1993) 101-110
    spq = math.sqrt(n * q * (1.0 - q))
    b = 1.15 + 2.53 * spq
    a = -0.0873 + 0.0248 * b + 0.01 * q
    c = n * q + 0.5
    vr = 0.92 - 4.2 / b
    alpha = (2.83 + 5.1 / b) * spq
    lpq = O.orc_log(q / (1.0 - q))
    m = float(math.floor((n + 1.0) * q))
    h = log_factorial(O, m) + log_factorial(O, n - m)
    while not s.spent():
        U = s.u() - 0.5
        V = s.u()
        us = 0.5 - abs(U)
        k = float(math.floor((2.0 * a / us + b) * U + c)) if us > 0 else -math.inf
        if k < 0.0 or k > n:
            continue
        if us >= 0.07 and V <= vr:
            return k
        if O.orc_log(V * alpha / (a / (us * us) + b)) <= h - log_factorial(O, k) - log_factorial(O, n - k) + (k - m) * lpq:
            return k
    return NAN


def draw(family, args, s):
    """one replicated observation; NaN outside the family's domain (csrc/amwg_ppc.cuh lists them)"""
    O = s.O
    n = ARITY.get(family, 2)
    a = [float(v) for v in args[:n]] + [0.0] * (3 - n)
    if not all(math.isfinite(v) for v in a[:n]):
        return NAN
    a0, a1, a2 = a
    f = family
    if f in ("norm", "lnorm"):
        if not a1 > 0:
            return NAN
        x = rnorm(s) * a1 + a0
        if f == "lnorm":
            x = O.orc_exp(x)
    elif f == "cauchy":
        if not a1 > 0:
            return NAN
        z1 = rnorm(s)
        z2 = rnorm(s)
        x = a0 + a1 * z1 / z2 if z2 != 0 else a0 + math.copysign(math.inf, a1 * z1) * math.copysign(1.0, z2)
    elif f == "laplace":
        if not a1 > 0:
            return NAN
        e1 = expo(s)
        e2 = expo(s)
        x = a0 + a1 * (e1 - e2)
    elif f == "logis":
        if not a1 > 0:
            return NAN
        while True:
            U = s.u()
            if not (U == 0.0 and not s.spent()):
                break
        x = a0 + a1 * (O.orc_log(U) - O.orc_log(1.0 - U))
    elif f == "exp":
        if not a0 > 0:
            return NAN
        x = expo(s) / a0
    elif f == "weibull":
        if not (a0 > 0 and a1 > 0):
            return NAN
        x = a1 * O.orc_exp(O.orc_log(expo(s)) / a0)
    elif f == "pareto":
        if not (a0 > 0 and a1 > 0):
            return NAN
        x = a0 * O.orc_exp(expo(s) / a1)
    elif f == "unif":
        if not a0 < a1:
            return NAN
        x = a0 + (a1 - a0) * s.u()
    elif f == "gamma":
        if not (a0 > 0 and a1 > 0):
            return NAN
        x = gamma1(s, a0) / a1
    elif f == "invgamma":
        if not (a0 > 0 and a1 > 0):
            return NAN
        g = gamma1(s, a0)
        x = a1 / g if g != 0 else math.inf
    elif f == "beta":
        if not (a0 > 0 and a1 > 0):
            return NAN
        X = gamma1(s, a0)
        Y = gamma1(s, a1)
        x = X / (X + Y) if X + Y != 0 else NAN
    elif f == "t":
        if not (a1 > 0 and a2 > 0):
            return NAN
        z = rnorm(s)
        g = gamma1(s, a2 / 2.0)
        x = a0 + a1 * z / math.sqrt(2.0 * g / a2)
    elif f == "bern":
        if not 0.0 <= a0 <= 1.0:
            return NAN
        x = 1.0 if s.u() < a0 else 0.0
    elif f == "pois":
        if not a0 >= 0:
            return NAN
        x = pois(s, a0)
    elif f == "binom":
        if not (a0 >= 0 and a0 == math.floor(a0) and 0.0 <= a1 <= 1.0):
            return NAN
        flip = a1 > 0.5
        k = binom_low(s, a0, 1.0 - a1 if flip else a1)
        x = a0 - k if flip else k
    elif f == "nbinom":
        if not (a0 > 0 and 0.0 < a1 <= 1.0):
            return NAN
        rate = a1 / (1.0 - a1) if a1 < 1.0 else math.inf
        lam = gamma1(s, a0) / rate
        x = pois(s, lam)
    else:
        raise ValueError(family)
    return NAN if s.spent() else x


def draw_at(O, family, args, seed, chain, row, points, i):
    """-> (y_rep, uniforms used) of (kept row, point i) of global chain `chain`"""
    s = Philox(O, seed, chain, position(row, points, i))
    x = draw(family, args, s)
    return x, s.used()


# ---- the statistics and the "ppc" dict ------------------------------------------------------------------------------------------
STATS = ("mean", "sd", "min", "max")


def _nanmin(a, b):
    return NAN if (a != a or b != b) else (a if a < b else b)


def _nanmax(a, b):
    return NAN if (a != a or b != b) else (a if a > b else b)


def dataset_stats(y):
    """(mean, sd, min, max) of one dataset, points in index order: sequential Welford, sd = sqrt(M2 / (N - 1)) (NaN for N = 1)"""
    m = M2 = 0.0
    mn = mx = NAN
    for j, v in enumerate(y, 1):
        v = float(v)
        d = v - m
        m += d / j
        M2 += d * (v - m)
        mn = v if j == 1 else _nanmin(mn, v)
        mx = v if j == 1 else _nanmax(mx, v)
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = float(np.sqrt(np.float64(M2) / np.float64(len(y) - 1))) if len(y) > 1 else NAN
    return m, sd, mn, mx


def counts(draws, t):
    """(#<, #==, #>, #NaN) of the draws against the threshold t"""
    d = np.asarray(draws, dtype=np.float64)
    return int(np.sum(d < t)), int(np.sum(d == t)), int(np.sum(d > t)), int(np.sum(np.isnan(d)))


def ppc(yrep, y, probs, family="norm"):
    """yrep [S, N] (every kept draw's replicated dataset), y [N] -> the "ppc" dict as numpy computes it (mean and sd pooled,
    quantiles numpy.quantile's linear rule)"""
    S, N = yrep.shape
    c = np.array([counts(yrep[:, i], y[i]) for i in range(N)])
    with np.errstate(invalid="ignore"):
        pw = {"mean": yrep.mean(axis=0), "sd": yrep.std(axis=0, ddof=1), "n_below": c[:, 0], "n_equal": c[:, 1],
              "pit": (c[:, 0] + c[:, 1]) / S, "n_nan": c[:, 3]}
    T = np.array([dataset_stats(row) for row in yrep])                # [S, 4]
    obs = dataset_stats(y)
    stats = {}
    for k, name in enumerate(STATS):
        ct = counts(T[:, k], obs[k])
        stats[name] = {"observed": obs[k], "mean": T[:, k].mean(), "sd": T[:, k].std(ddof=1),
                       "quantiles": np.quantile(T[:, k], probs), "n_greater": ct[2], "n_equal": ct[1], "n_nan": ct[3],
                       "p_value": (ct[2] + ct[1]) / S}
    return {"family": family, "points": N, "n_draws": S, "pointwise": pw, "stats": stats, "T": T}


def dataset_stats_many(Y):
    """dataset_stats of every row of Y [S, N] at once: the same sequential operations, each elementwise over the rows"""
    Y = np.asarray(Y, dtype=np.float64)
    S, N = Y.shape
    m = np.zeros(S)
    M2 = np.zeros(S)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for j in range(N):
            v = Y[:, j]
            d = v - m
            m = m + d / float(j + 1)
            M2 = M2 + d * (v - m)
        sd = np.sqrt(M2 / np.float64(N - 1)) if N > 1 else np.full(S, NAN)
    return np.stack([m, sd, Y.min(axis=1), Y.max(axis=1)], axis=1)          # numpy's min / max propagate NaN like js_min / js_max
