"""The predictive-check samplers of csrc/amwg_ppc.cuh, compiled for the host, across each family's domain: every switch between
algorithms with its neighbours on both sides (pois lambda = 10, binom size q = 10 and prob = 1/2, gamma shape = 1, t df = 2), counts
up to 1e18, binomial q down to 1e-15, shapes and degrees of freedom down to 1e-3, nbinom prob from 1e-300 to 1 - 2^-53, scales
that put the draws among the subnormals or past DBL_MAX, and unif over (-1e308, 1e308).

Each of the GRID's 72 points takes 1e5 draws from fixed seeds and is held to the law of the fp64-rounded variate, not of the real
one: a draw of 0, +-inf, or 1.0 for beta, has the probability that the exact variate rounds there.
  * No draw is NaN, and no draw takes more than 2^12 uniforms (the stream reserves 2^16 per draw).
  * Continuous laws: each atom cell (0, +-inf, beta's 1.0) by a two-sided binomial test against its probability, computed by
    mpmath at 160 bits at the rounding boundaries (2^-1075, 2^1024 - 2^970, 1 - 2^-54); the other draws by a chi-square over
    cells whose edges are scipy quantiles and whose probabilities are mpmath's CDF at each edge's rounding boundary.
  * Discrete laws: a chi-square over cells at quantiles, probabilities from scipy's CDF or, where the sd exceeds 1e3, from an
    Edgeworth expansion (error O(1 / sd^2)), which test_scipy_cdfs_agree_with_mpmath_at_the_extremes holds to scipy and mpmath.
    nbinom at prob < 1e-6 is held to its gamma limit, as a continuous law (the CDFs differ by O(prob)).
  * Where the fourth moment exists and the excess kurtosis is at most 50: the standardised mean, and the sample variance
    against its exact sampling sd sqrt((mu4 / sigma^4 - (n - 3) / (n - 1)) / n), two-sided normal tests. KS at 1e5 draws cannot
    see a 2 % error in the sd; this can.
Every statistical check must give p > 1e-6. The 72 points make 362 checks in all (CHECKS; a test holds the number here to the
grid). Besides: 100 draws of every point bit for bit against tests/ppc_ref.py, the samplers' log1p and log-factorial differences
against mpmath, and scipy's quantiles and CDFs at the extreme points against mpmath."""
import ctypes as C
import math
import os
import subprocess

import mpmath
import numpy as np
import pytest
from scipy import stats as st

import ppc_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 20261017
CHAIN = 3
N_DRAWS = 100000
P_MIN = 1e-6
MAX_USED = 1 << 12
N_CELLS = 40
PREC = 160
INF = math.inf
DMAX = float(np.finfo(np.float64).max)
nxt = np.nextafter


def _build(out_dir):
    out = os.path.join(str(out_dir), "libppc_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "ppc_host.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("ppc_domain_host")))
    lib.hs_ppc_draws.restype = C.c_uint64
    lib.hs_ppc_draws.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]
    lib.hs_ppc_draw.restype = C.c_double
    lib.hs_ppc_draw.argtypes = [C.c_int, C.c_void_p] + [C.c_uint64] * 5 + [C.POINTER(C.c_uint64)]
    return lib


def host_draws(H, fam, p, n=N_DRAWS):
    """-> (n draws at row 0, points 0 .. n - 1 of chain CHAIN, the most uniforms any took)"""
    out = np.empty(n)
    a = np.ascontiguousarray(list(p) + [0.0] * (3 - len(p)), dtype=np.float64)
    most = H.hs_ppc_draws(ppc_ref.FAMILIES.index(fam), a.ctypes.data, SEED, CHAIN, n, out.ctypes.data)
    return out, int(most)


# ---- the grid ------------------------------------------------------------------------------------------------------------------
def _around(x):
    return [nxt(x, -INF), x, nxt(x, INF)]


LARGE = [1e8, 1e12, 1e14, 1e15, 2.0 ** 53, 1e18]
GRID = (
    [("pois", (lam,)) for lam in _around(10.0) + LARGE]
    + [("binom", (40.0, q)) for q in _around(0.25)]                                      # size q = 10
    + [("binom", (20.0, q)) for q in _around(0.5)] + [("binom", (100.0, q)) for q in _around(0.5)]     # prob = 1/2
    + [("binom", (float(round(m / 0.3)), 0.3)) for m in LARGE]
    + [("binom", (1e14, 0.3)), ("binom", (1e15, 0.3)), ("binom", (1e18, 0.5)), ("binom", (1e15, 1.0 - 5e-15))]
    + [("binom", (1e15, 5e-15)), ("binom", (5e15, 1e-15)), ("binom", (3e13, 2e-13)), ("binom", (1e9, 5e-9))]   # inversion, tiny q
    + [("nbinom", (2.0, 1e-300)), ("nbinom", (2.0, 1e-12)), ("nbinom", (2.0, 1.0 - 2.0 ** -53)), ("nbinom", (0.5, 1e-12))]
    + [("gamma", (a, 1.0)) for a in _around(1.0) + [1e-3, 3e-3, 2e-2]] + [("gamma", (2e-2, 1e-300)), ("gamma", (3.0, 1e300))]
    + [("invgamma", (a, 1.0)) for a in (1e-3, 3e-3, 2e-2)]
    + [("beta", (a, a)) for a in (1e-3, 3e-3, 2e-2)] + [("beta", (1e-3, 2.0)), ("beta", (2.0, 3e-3))]
    + [("beta", (a, 1.0)) for a in _around(1.0)]
    + [("t", (0.0, 1.0, df)) for df in (0.01, 0.05, 1.0, 1e300) + tuple(_around(2.0))]
    + [("weibull", (0.01, 1.0)), ("pareto", (1.0, 0.01))]
    + [("norm", (0.0, 1e-320)), ("exp", (1e300,)), ("exp", (1e-300,)), ("cauchy", (0.0, 1e300)), ("logis", (0.0, 1e300))]
    + [("unif", (-1e308, 1e308)), ("unif", (-DMAX, DMAX)), ("laplace", (0.0, 1e300))]
)
GRID = [(f, tuple(float(v) for v in p)) for f, p in GRID]


def _id(point):
    return "%s%r" % (point[0], point[1])


# ---- the exact laws --------------------------------------------------------------------------------------------------------------
def _mp(x):
    return mpmath.mpf(float(x))


def rounds_up_at(t):
    """the real at which round-to-nearest passes from the double t to the next one above (t = -inf: where -inf ends)"""
    over = mpmath.mpf(2) ** 1024 - mpmath.mpf(2) ** 970
    t = float(t)
    if t == -INF:
        return -over
    if t == DMAX:
        return over
    return (_mp(t) + _mp(nxt(t, INF))) / 2


def _ncdf(x):
    """mpmath's ncdf, which overflows far out: beyond 1e4 sd the tail (e^(-5e7)) is below any probability here"""
    return mpmath.mpf(0) if x < -1e4 else mpmath.mpf(1) if x > 1e4 else mpmath.ncdf(x)


def _t_cdf(x, df):
    if df > 1e10:
        return _ncdf(x)
    tail = mpmath.betainc(df / 2, mpmath.mpf(1) / 2, 0, df / (df + x * x), regularized=True) / 2
    return tail if x < 0 else 1 - tail


def exact_cdf(fam, p):
    """-> the exact CDF of the real variate at an mpf, or None for the discrete laws (nbinom at prob < 1e-6 is its gamma limit,
    whose CDF is within O(prob) of nbinom's)"""
    a = [_mp(v) for v in p]
    pos = lambda f: (lambda t: mpmath.mpf(0) if t <= 0 else f(t))
    if fam == "norm":
        return lambda t: _ncdf((t - a[0]) / a[1])
    if fam == "cauchy":
        return lambda t: mpmath.mpf(1) / 2 + mpmath.atan((t - a[0]) / a[1]) / mpmath.pi
    if fam == "laplace":
        return lambda t: mpmath.exp((t - a[0]) / a[1]) / 2 if t < a[0] else 1 - mpmath.exp(-(t - a[0]) / a[1]) / 2
    if fam == "logis":
        return lambda t: 1 / (1 + mpmath.exp(-(t - a[0]) / a[1]))
    if fam == "exp":
        return pos(lambda t: -mpmath.expm1(-a[0] * t))
    if fam == "weibull":
        return pos(lambda t: -mpmath.expm1(-(t / a[1]) ** a[0]))
    if fam == "pareto":
        return lambda t: mpmath.mpf(0) if t <= a[0] else 1 - (a[0] / t) ** a[1]
    if fam == "unif":
        return lambda t: min(max((t - a[0]) / (a[1] - a[0]), mpmath.mpf(0)), mpmath.mpf(1))
    if fam == "gamma":
        return pos(lambda t: mpmath.gammainc(a[0], 0, a[1] * t, regularized=True))
    if fam == "invgamma":
        return pos(lambda t: mpmath.gammainc(a[0], a[1] / t, mpmath.inf, regularized=True))
    if fam == "beta":
        return pos(lambda t: mpmath.mpf(1) if t >= 1 else mpmath.betainc(a[0], a[1], 0, t, regularized=True))
    if fam == "t":
        return lambda t: _t_cdf((t - a[0]) / a[1], a[2])
    if fam == "nbinom" and p[1] < 1e-6:
        return pos(lambda t: mpmath.gammainc(a[0], 0, t * a[1] / (1 - a[1]), regularized=True))
    return None


class _HalvedUniform:
    """the uniform law's quantiles where max - min overflows"""

    def __init__(self, lo, hi):
        self.lo, self.hi = lo, hi

    def ppf(self, u):
        return 2.0 * (0.5 * self.lo + (0.5 * self.hi - 0.5 * self.lo) * np.asarray(u))


def scipy_law(fam, p):
    a = p
    return {"norm": lambda: st.norm(a[0], a[1]), "cauchy": lambda: st.cauchy(a[0], a[1]), "laplace": lambda: st.laplace(a[0], a[1]),
            "logis": lambda: st.logistic(a[0], a[1]), "exp": lambda: st.expon(scale=1 / a[0]),
            "weibull": lambda: st.weibull_min(a[0], scale=a[1]), "pareto": lambda: st.pareto(a[1], scale=a[0]),
            "unif": lambda: _HalvedUniform(a[0], a[1]), "gamma": lambda: st.gamma(a[0], scale=1 / a[1]),
            "invgamma": lambda: st.invgamma(a[0], scale=a[1]), "beta": lambda: st.beta(a[0], a[1]),
            "t": lambda: st.t(min(a[2], 1e10), a[0], a[1]), "pois": lambda: st.poisson(a[0]),
            "binom": lambda: st.binom(a[0], a[1]),
            "nbinom": lambda: (st.gamma(a[0], scale=(1 - a[1]) / a[1]) if a[1] < 1e-6 else st.nbinom(a[0], a[1]))}[fam]()


def moments(fam, p, split=False):
    """-> (mean, sd, excess kurtosis) of the law, or None where the fourth moment does not exist; split: the mean as two
    doubles, hi + lo (1e15 - 4.996 is not a double, and its rounding moves the standardised mean of 1e6 draws by 2 sd)"""
    with mpmath.workprec(PREC):
        a = [_mp(v) for v in p]
        if fam == "norm":
            m = (a[0], a[1], 0)
        elif fam == "exp":
            m = (1 / a[0], 1 / a[0], 6)
        elif fam == "logis":
            m = (a[0], a[1] * mpmath.pi / mpmath.sqrt(3), mpmath.mpf(6) / 5)
        elif fam == "laplace":
            m = (a[0], a[1] * mpmath.sqrt(2), 3)
        elif fam == "unif":
            m = ((a[0] + a[1]) / 2, (a[1] - a[0]) / mpmath.sqrt(12), -mpmath.mpf(6) / 5)
        elif fam == "gamma":
            m = (a[0] / a[1], mpmath.sqrt(a[0]) / a[1], 6 / a[0])
        elif fam == "beta":
            s = a[0] + a[1]
            ab = a[0] * a[1]
            m = (a[0] / s, mpmath.sqrt(ab / (s * s * (s + 1))), 6 * ((a[0] - a[1]) ** 2 * (s + 1) - ab * (s + 2)) / (ab * (s + 2) * (s + 3)))
        elif fam == "t" and a[2] > 4:
            m = (a[0], a[1] * (mpmath.sqrt(a[2] / (a[2] - 2)) if a[2] < 1e100 else 1), 6 / (a[2] - 4))
        elif fam == "pois":
            m = (a[0], mpmath.sqrt(a[0]), 1 / a[0]) if a[0] > 0 else None
        elif fam == "binom":
            v = a[0] * a[1] * (1 - a[1])
            m = (a[0] * a[1], mpmath.sqrt(v), (1 - 6 * a[1] * (1 - a[1])) / v)
        elif fam == "nbinom":
            q = 1 - a[1]
            m = (a[0] * q / a[1], mpmath.sqrt(a[0] * q) / a[1], 6 / a[0] + a[1] ** 2 / (a[0] * q))
        else:
            return None
        if m is None:
            return None
        mean = (float(m[0]), float(m[0] - float(m[0]))) if split else float(m[0])
        return (mean, float(m[1]), float(m[2]))


def _merge_small(obs, exp, n):
    """adjacent cells pooled until each expects >= 5 draws"""
    co, ce, ao, ae = [], [], 0.0, 0.0
    for o, e in zip(obs, exp):
        ao, ae = ao + o, ae + e
        if ae * n >= 5:
            co.append(ao)
            ce.append(ae)
            ao = ae = 0.0
    if ae > 0 or ao > 0:
        if ce:
            co[-1] += ao
            ce[-1] += ae
        else:
            co.append(ao)
            ce.append(ae)
    return np.array(co), np.array(ce)


def _chi_square(obs, prob):
    """p of the chi-square of the counts against the cell probabilities, renormalised to the cells' total; 0 if a draw lies
    where the law puts no mass (a beta draw above 1, say)"""
    n = obs.sum()
    if np.any(obs[prob == 0] > 0):
        return 0.0
    if n == 0:
        return 1.0
    co, ce = _merge_small(obs, prob / prob.sum(), n)
    if len(co) < 2:
        return 1.0
    return float(st.chisquare(co, ce * n).pvalue)


def _continuous_cells(fam, p, F):
    """-> (edges, P(fl(X) <= edge) for each edge, indices of the atom cells). Cell j holds edges[j-1] < x <= edges[j]; the last
    cell, x > edges[-1], is +inf."""
    special = [-INF, DMAX]
    atoms = {-INF, DMAX}                                 # cells ending at -inf (x = -inf) and beyond DMAX (x = +inf)
    lower_support = fam in ("exp", "weibull", "pareto", "gamma", "invgamma", "beta", "nbinom")
    if lower_support:
        special.append(0.0)
        atoms.add(0.0)
    if fam == "beta":
        special += [float(nxt(1.0, 0.0)), 1.0]
        atoms.add(1.0)
    G = {e: F(rounds_up_at(e)) for e in special}
    lo_mass = max(float(G[e]) for e in special if e in (-INF, 0.0))
    hi_edge = float(nxt(1.0, 0.0)) if fam == "beta" else DMAX
    hi_mass = float(G[hi_edge])
    with np.errstate(all="ignore"):
        u = lo_mass + (hi_mass - lo_mass) * np.arange(1, N_CELLS) / N_CELLS
        q = scipy_law(fam, p).ppf(u)
    lo_edge = 0.0 if lower_support else -INF
    inner = sorted({float(v) for v in q if np.isfinite(v) and lo_edge < v < hi_edge} - set(special))
    edges = sorted(set(special) | set(inner))
    for e in inner:
        G[e] = F(rounds_up_at(e))
    return np.array(edges), [G[e] for e in edges], [i for i, e in enumerate(edges) if e in atoms and e != DMAX] + [len(edges)]


def _edgeworth_cdf(k, mu, sd, skew):
    """P(X <= k) of an integer law from its first three cumulants; the error is O(1 / sd^2)"""
    z = (k + 0.5 - mu) / sd
    return st.norm.cdf(z) - st.norm.pdf(z) * skew * (z * z - 1) / 6


def _skew(fam, p):
    return 1 / math.sqrt(p[0]) if fam == "pois" else (1 - 2 * p[1]) / math.sqrt(p[0] * p[1] * (1 - p[1]))


def _discrete_cells(fam, p):
    """pois and binom with sd > 1e3 by the Edgeworth expansion (scipy's CDF there is off by up to 1e-8, and NaN at some points
    above 2^53); below, scipy. Beyond 2^53 a cell edge e stands for the integers that round to at most e: P(X <= e) moves by
    less than ulp(e) / sd (1e-7), far below what 1e6 draws resolve."""
    mu, sd, _ = moments(fam, p)
    u = np.arange(1, N_CELLS) / N_CELLS
    if sd > 1e3:
        edges = np.unique(np.floor(mu + sd * st.norm.ppf(u)))
        G = _edgeworth_cdf(edges, mu, sd, _skew(fam, p))
    else:
        d = scipy_law(fam, p)
        edges = np.unique(d.ppf(u))
        G = d.cdf(edges)
    return edges, [mpmath.mpf(float(v)) for v in G], []


def law_checks(x, fam, p):
    """-> [(name, p-value)] of every statistical check of the draws x against the law of (fam, p)"""
    out = []
    n = len(x)
    with mpmath.workprec(PREC):
        F = exact_cdf(fam, p)
        edges, G, atoms = _continuous_cells(fam, p, F) if F is not None else _discrete_cells(fam, p)
        G = G + [mpmath.mpf(1)]
        prob = np.array([float(G[0])] + [float(G[j] - G[j - 1]) for j in range(1, len(G))])
    obs = np.bincount(np.searchsorted(edges, x, side="left"), minlength=len(prob)).astype(float)
    for j in atoms:
        what = "x = %s" % ("+inf" if j == len(edges) else edges[j])
        if prob[j] == 0.0:
            out.append((what, 1.0 if obs[j] == 0 else 0.0))
        else:
            out.append((what, float(st.binomtest(int(obs[j]), n, prob[j]).pvalue)))
    rest = np.array([j for j in range(len(prob)) if j not in atoms])
    out.append(("chi-square", _chi_square(obs[rest], prob[rest])))
    m = moments(fam, p, split=True)
    if m is not None and m[2] <= 50:
        (hi, lo), sd, kurt = m
        with np.errstate(over="ignore"):
            y = ((x - hi) - lo) / sd
        zm = y.mean() * math.sqrt(n)
        var_sd = math.sqrt((3.0 + kurt - (n - 3.0) / (n - 1.0)) / n)
        zv = (y.var(ddof=1) - 1.0) / var_sd
        out.append(("standardised mean %.3g" % zm, float(2 * st.norm.sf(abs(zm)))))
        out.append(("standardised variance %.3g" % zv, float(2 * st.norm.sf(abs(zv)))))
    return out


def check_draws(x, fam, p):
    assert not np.any(np.isnan(x)), (fam, p, int(np.isnan(x).sum()))
    res = law_checks(x, fam, p)
    bad = [(what, pv) for what, pv in res if not pv > P_MIN]
    assert not bad, (fam, p, bad)
    return len(res)


CHECKS = 362                                             # the docstring's count: no-NaN-and-budget + law_checks, over the GRID


@pytest.mark.parametrize("point", GRID, ids=_id)
def test_draws_follow_the_rounded_law(H, point):
    fam, p = point
    x, most = host_draws(H, fam, p)
    assert most < MAX_USED, (fam, p, most)
    check_draws(x, fam, p)


def test_the_docstring_counts_every_check():
    n = 0
    for fam, p in GRID:
        with mpmath.workprec(PREC):
            F = exact_cdf(fam, p)
            edges, G, atoms = _continuous_cells(fam, p, F) if F is not None else _discrete_cells(fam, p)
        m = moments(fam, p)
        n += 1 + len(atoms) + 1 + (2 if m is not None and m[2] <= 50 else 0)
    assert len(GRID) == 72 and n == CHECKS, (len(GRID), n)


def test_host_draws_equal_the_restatement_across_the_grid(H, orc):
    """100 draws of every grid point at random (chain, row, point), bit for bit and uniform for uniform"""
    O = orc.lib()
    rng = np.random.default_rng(11)
    for fam, p in GRID:
        a = np.ascontiguousarray(list(p) + [0.0] * (3 - len(p)), dtype=np.float64)
        for _ in range(100):
            g, r, N = int(rng.integers(0, 1 << 22)), int(rng.integers(0, 50)), int(rng.integers(1, 5000))
            i = int(rng.integers(0, N))
            used = C.c_uint64()
            got = H.hs_ppc_draw(ppc_ref.FAMILIES.index(fam), a.ctypes.data, SEED, g, r, N, i, C.byref(used))
            want, wused = ppc_ref.draw_at(O, fam, p, SEED, g, r, N, i)
            assert np.float64(got).tobytes() == np.float64(want).tobytes() and used.value == wused, (fam, p, g, r, i, got, want)


def _helper(H, name, nargs):
    f = getattr(H, name)
    f.restype = C.c_double
    f.argtypes = [C.c_double] * nargs
    return f


def test_log1p_is_within_a_few_ulp(H, orc):
    """Goldberg's log1p against mpmath, where js_log(1 + x) loses every bit (|x| < 2^-53) and around it"""
    O = orc.lib()
    log1p = _helper(H, "hs_ppc_log1p", 1)
    xs = [5e-324, -5e-324, 1e-300, 2.0 ** -60, -2.0 ** -54, 1e-16, -1e-16, 1.1e-16, 3e-15, -5e-15, 1e-12, -1e-9, 3e-8, -0.25,
          0.5, -0.5, 0.999, 10.0, 1e10, 1e300, -(1 - 2.0 ** -53)]
    with mpmath.workprec(PREC):
        for x in xs:
            got = log1p(x)
            exact = mpmath.log1p(_mp(x))
            assert abs(_mp(got) - exact) <= 4 * 2.0 ** -52 * abs(exact), (x, got)
            assert got == ppc_ref.log1p(O, x)


def test_log_factorial_differences_against_mpmath(H, orc):
    """log (i + e)! - log i! for i from 10 to 1e18 and steps of the size PTRS and BTRS take (e up to 10 sd), within a few ulp of
    |e| log i once both are >= 128 (log i! itself is 4e19 at 1e18); i above 2^53 stands for itself (an integer double)"""
    O = orc.lib()
    diff = _helper(H, "hs_ppc_log_factorial_diff", 2)
    cases = [(10.0, 5.0), (100.0, 50.0), (127.0, 1.0), (128.0, -1.0), (1000.0, -999.0), (5e5, 3e3)]
    for i in (1e8, 1e12, 1e15, 2.0 ** 53, 3e16, 1e18):
        s = math.sqrt(i)
        cases += [(i, float(math.floor(k * s))) for k in (-10.0, -1.0, 0.001, 1.0, 7.0)] + [(i, 1.0), (i, -1.0), (i, 0.0)]
    with mpmath.workprec(PREC):
        for i, e in cases:
            got = diff(i, e)
            exact = mpmath.loggamma(_mp(i) + e + 1) - mpmath.loggamma(_mp(i) + 1)
            tol = 8 * 2.0 ** -52 * (abs(e) * math.log(i) + 1)
            if min(i, i + e) < 128:                          # the plain difference of two log factorials below 128
                tol += 4 * 2.0 ** -52 * math.lgamma(max(i, i + e) + 1)
            assert abs(_mp(got) - exact) <= tol, (i, e, got, float(exact))
            assert got == ppc_ref.log_factorial_diff(O, i, e)


EXTREME_CONTINUOUS = [("gamma", (1e-3, 1.0), (0.55, 0.7, 0.9, 0.99)), ("invgamma", (2e-2, 1.0), (0.02, 0.1, 0.2, 0.3)),
                      ("beta", (3e-3, 3e-3), (0.1, 0.3, 0.45, 0.52)), ("t", (0.0, 1.0, 0.05), (0.01, 0.3, 0.6, 0.97)),
                      ("nbinom", (2.0, 1e-12), (0.01, 0.3, 0.6, 0.99)), ("nbinom", (2.0, 1e-300), (0.01, 0.5, 0.99))]
EXTREME_DISCRETE = [("pois", (1e8,)), ("pois", (1e12,)), ("pois", (1e15,)), ("pois", (1e18,)), ("binom", (1e15, 0.3)),
                    ("binom", (1e18, 0.5)), ("binom", (float(round(2.0 ** 53 / 0.3)), 0.3))]


@pytest.mark.parametrize("fam, p, us", EXTREME_CONTINUOUS, ids=lambda v: repr(v))
def test_scipy_quantiles_agree_with_mpmath_at_the_extremes(fam, p, us):
    """the cell edges are scipy's quantiles: mpmath's CDF at them gives back the probabilities asked for (and for nbinom at a
    tiny prob, scipy's own nbinom CDF agrees with the gamma limit the cells use)"""
    with mpmath.workprec(PREC):
        F = exact_cdf(fam, p)
        for u in us:
            q = float(scipy_law(fam, p).ppf(u))
            assert abs(float(F(_mp(q))) - u) < 1e-7, (fam, p, u, q)
            if fam == "nbinom" and p[1] > 1e-100:
                assert abs(float(st.nbinom(p[0], p[1]).cdf(math.floor(q))) - u) < 1e-7, (fam, p, u, q)


@pytest.mark.parametrize("point", EXTREME_DISCRETE, ids=_id)
def test_scipy_cdfs_agree_with_mpmath_at_the_extremes(point):
    """the large discrete cells' probabilities are the Edgeworth expansion: it agrees with scipy's CDF wherever that is finite,
    and at 1e8 with mpmath's incomplete gamma (beyond, mpmath does not finish)"""
    fam, p = point
    mu, sd, _ = moments(fam, p)
    d = scipy_law(fam, p)
    for z in (-3.0, -1.0, 0.0, 0.5, 2.5):
        k = math.floor(mu + z * sd)
        want = _edgeworth_cdf(k, mu, sd, _skew(fam, p))
        got = float(d.cdf(k))
        assert math.isnan(got) or abs(got - want) < 2e-8, (fam, p, z, got, want)
        if fam == "pois" and p[0] <= 1e8:
            with mpmath.workprec(PREC):
                exact = float(mpmath.gammainc(k + 1, p[0], mpmath.inf, regularized=True))
            assert abs(exact - want) < 1e-8, (fam, p, z, exact, want)
