"""Extended-precision reference for the factorised likelihood plates (csrc amwg_kernels.cu: PLATE_NORM_IID, PLATE_NORM_GROUPED,
PLATE_POIS_LOGLIN), with a worst-case forward-error bound for the fp64 operations the kernels perform.

Every value is the sum, in numpy.longdouble (>= 63-bit significand), of the exact per-row terms of the reference's likelihood loop
at a given state; lfactorial comes from the oracle's restatement of the reference's Lanczos lfactorial (orc_ld_lfactorial), so
the value is what distributions.js computes, without its rounding. The bound adds up, term by term, what each fp64 operation of
the kernel (and of the host precomputation it relies on) can contribute. A test passes when |kernel - value| <= bound, and every
case also checks that the bound is below 1e-3 of the median of what the kernel sums per row (exp(eta_i) for the Poisson plate, whose
other parts are precomputed on the host; (x_i - mean_i)^2 / (2 sd^2) for the Normal plates, whose n (c0 - log sd) is formed from
n): a dropped, duplicated or stale row, or a value from another chain, moves the result by far more than the bound.

Test infrastructure only (CPU); used by the GPU value tests and self-checked against the oracle's term-by-term models."""
import numpy as np

LD = np.longdouble
U = 2.0 ** -53                  # unit roundoff of fp64
TINY = 2.0 ** -1074             # an ulp of the subnormal range
JS_PI = 3.141592653589793      # Math.PI: ld.norm uses the double, not pi


def require_extended():
    """The bounds below are of the order of u = 2^-53 times the magnitudes involved; a reference with a 53-bit significand
    would be as wrong as the kernel it checks. Fail instead of quietly losing the precision."""
    nmant = np.finfo(LD).nmant
    assert nmant >= 63, f"numpy.longdouble has a {nmant}-bit significand on this platform; the plate reference needs >= 63"


def gamma(k) -> float:
    """gamma_k = k u / (1 - k u): bound on the relative error of k chained fp64 roundings (Higham, Accuracy and Stability, 3.1)"""
    k = float(k)
    return k * U / (1.0 - k * U)


class Value:
    """value (longdouble), bound (float) and the median per-row summand of the kernel (for the sensitivity check), per chain."""

    def __init__(self, value, bound, row_median):
        self.value = np.asarray(value, dtype=LD)
        self.bound = np.asarray(bound, dtype=np.float64)
        self.row_median = np.asarray(row_median, dtype=np.float64)

    def check(self, got, what=""):
        """|got - value| <= bound for every chain, and bound < 1e-3 x the median per-row summand."""
        got = np.asarray(got, dtype=np.float64)
        assert got.shape == self.value.shape, (what, got.shape, self.value.shape)
        assert np.all(np.isfinite(self.value)), what
        assert np.all(self.bound < 1e-3 * self.row_median), (what, float(np.max(self.bound / self.row_median)))
        err = np.abs(got.astype(LD) - self.value).astype(np.float64)
        bad = ~(err <= self.bound)
        assert not bad.any(), (what, int(bad.sum()), "chains off; worst err/bound", float(np.max(err / self.bound)),
                               "first", int(np.argmax(bad)), float(got[bad][0]), float(self.value[bad][0]))


def lfactorial_ref(orc, y) -> np.ndarray:
    """orc_ld_lfactorial (the reference's Lanczos lgamma(y + 1), distributions.js:63-82) per entry, as doubles"""
    L = orc.lib()
    y = np.asarray(y, dtype=np.float64)
    vals, inv = np.unique(y, return_inverse=True)
    return np.array([L.orc_ld_lfactorial(float(v)) for v in vals])[inv].reshape(y.shape)


def _lfactorial_host_bound(y) -> np.ndarray:
    """How far the host's lfactorial (tracer._lfactorial_host_vec, numpy log) can be from orc_ld_lfactorial (the oracle's log): the
    same fp64 operations in the same order, on logs that may differ by 1 ulp each, and every later rounding then differs by up to
    an ulp of its result. 4 u times the sum of the magnitudes of the intermediate values covers both."""
    x = np.asarray(y, dtype=np.float64) + 1.0
    ser = np.full_like(x, 1.000000000190015)
    yy = x.copy()
    for c in (76.18009172947146, -86.50532032941677, 24.01409824083091, -1.231739572450155, 0.1208650973866179e-2, -0.5395239384953e-5):
        yy = yy + 1.0
        ser = ser + abs(c) / yy
    tmp = x + 5.5
    big = (x + 0.5) * np.log(tmp)
    return 4 * U * (tmp + big + np.abs(np.log(2.5066282746310005 * ser / x)) + np.abs(tmp - big) + 1.0)


# ---- priors (scalar terms of log_post), as the device computes them: NORM_K / UNIF_K with device-folded constants ------------
def norm_term(x, mean, sd):
    """ld.norm(x, mean, sd) for one state component per chain: (value, bound). The device evaluates k1 - (x - mean)^2 / k2 with
    k1 = -0.5 log(2 pi) - log(sd) and k2 = 2 sd sd folded once (two logs within 1 ulp, a product, a difference), then a difference,
    a square, a quotient and a difference."""
    x, mean, sd = (np.asarray(v, dtype=LD) for v in (x, mean, sd))
    c = LD(-0.5) * np.log(LD(2) * LD(JS_PI))
    k1 = c - np.log(sd)
    q = (x - mean) ** 2 / (LD(2) * sd * sd)
    v = k1 - q
    b = 4 * U * (np.abs(c) + np.abs(np.log(sd))) + 5 * U * q + U * np.abs(v)
    return v, b.astype(np.float64)


def unif_term(x, lo, hi):
    """ld.unif(x, lo, hi) inside the support: the folded constant log(1 / (hi - lo)): three roundings and a 1-ulp log"""
    v = np.log(LD(1) / (LD(hi) - LD(lo))) * np.ones(np.shape(x), dtype=LD)
    assert np.all((np.asarray(x) >= lo) & (np.asarray(x) <= hi))
    return v, (4 * U * (np.abs(v) + 1)).astype(np.float64)


def combine(terms):
    """lp = ((0 + t_1) + t_2) + ...: the program adds its terms in the user's order. terms: [(value, bound, row_median or None)];
    the result's bound is the terms' bounds plus gamma_m times the sum of their magnitudes (the running sums are bounded by it)."""
    value = sum(t[0] for t in terms)
    mag = sum(np.abs(t[0]).astype(np.float64) + t[1] for t in terms)
    bound = sum(t[1] for t in terms) + gamma(len(terms)) * mag
    meds = [t[2] for t in terms if len(t) > 2 and t[2] is not None]
    assert meds, "at least one plate: its rows set the sensitivity"
    return Value(value, bound, np.minimum.reduce(meds))


def per_state(fn, states):
    """Evaluate fn([U, D] distinct states) -> Value once per distinct row of `states` [C, D] (chains share their initial state)."""
    u, inv = np.unique(np.asarray(states, dtype=np.float64), axis=0, return_inverse=True)
    inv = np.asarray(inv).reshape(-1)
    r = fn(u)
    return Value(r.value[inv], r.bound[inv], r.row_median[inv])


# ---- PLATE_POIS_LOGLIN ----------------------------------------------------------------------------------------------------
def pois_loglin(orc, y, X, beta, partials=2, chunk=64):
    """sum_i ld.pois(y_i, exp(eta_i)), eta_i = sum_k X_ik beta_k, per chain (beta: [C, K]) -> (value, bound, median exp(eta_i)).

    The plate computes beta . (X^T y) - sum_i exp(eta_i) - sum_i lfactorial(y_i) (csrc pois_plate_k). Its error is at most:
      Xt  the host's X^T y in fp64 (numpy): gamma_n sum_i |X_ik y_i| per k, times |beta_k|; then the K-term fma chain beta . (X^T y):
          gamma_K sum_k |beta_k (X^T y)_k|;
      eta the K-term fma chain of each row (register path) or the DMMA.8x8x4 dot product (K = 8 on the ring): |d eta_i| <= gamma_K
          sum_k |X_ik beta_k| =: a_i, which is a relative error of expm1(a_i) ~ K u a_i in exp(eta_i);
      exp the table exp (exp_acc_fast) or the library exp (beyond |eta| = 690): within 2 ulp, i.e. 4 u exp(eta_i), plus 2 ulp of
          the subnormal range below exp(-708);
      acc the accumulation of the perturbed exp(eta_i) into `partials` partial sums (2: s0/s1 of the register and global paths; 8:
          the row classes of a lane in the DMMA form), then their combination: gamma_(n/partials + log2(partials) + 2) sum_i exp;
      lf  the host's lfactorial constant: per row _lfactorial_host_bound, then numpy's sum: gamma_n sum_i |lfactorial(y_i)|;
      out the two differences (lin - S) - L: 2 u (|lin| + |S| + |L|)."""
    y = np.asarray(y, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64).reshape(y.size, -1)
    beta = np.atleast_2d(np.asarray(beta, dtype=np.float64))
    n, K = X.shape
    C = beta.shape[0]
    XL, yL = X.astype(LD), y.astype(LD)
    lf = lfactorial_ref(orc, y).astype(LD)
    L_sum = lf.sum()
    absXty = np.abs(X).T @ np.abs(y)                                     # [K], fp64 is enough for a bound
    stats = XL.T @ yL                                                    # exact X^T y (to the extended precision)
    lf_bound = float(np.sum(_lfactorial_host_bound(y))) + gamma(n) * float(np.sum(np.abs(lf)))
    depth = -(-n // partials) + int(np.log2(partials)) + 2
    value = np.empty(C, dtype=LD)
    bound = np.empty(C)
    med = np.empty(C)
    for c0 in range(0, C, chunk):
        B = beta[c0:c0 + chunk]                                          # [c, K]
        BL = B.astype(LD)
        eta = XL @ BL.T                                                  # [n, c]
        e = np.exp(eta)
        lin = stats @ BL.T                                               # [c]
        S = e.sum(axis=0)
        rows = yL[:, None] * eta - e - lf[:, None]
        value[c0:c0 + chunk] = rows.sum(axis=0)
        a = gamma(K) * (np.abs(X) @ np.abs(B).T)                         # [n, c]: bound on |d eta_i|
        ef = e.astype(np.float64)
        e_err = ef * (np.expm1(a) * (1 + 4 * U) + 4 * U) + 2 * TINY      # eta chain, then the exp of the perturbed eta
        acc = gamma(depth) * (ef + e_err).sum(axis=0)
        xt = np.abs(B) @ (gamma(n) * absXty) + gamma(K) * (np.abs(B) @ np.abs(stats.astype(np.float64)))
        out = 2 * U * (np.abs(lin.astype(np.float64)) + np.abs(S.astype(np.float64)) + abs(float(L_sum)))
        bound[c0:c0 + chunk] = xt + e_err.sum(axis=0) + acc + lf_bound + out
        med[c0:c0 + chunk] = np.median(ef, axis=0)                      # a row changes the result by its exp(eta_i)
    return value, bound, med


# ---- PLATE_NORM_IID / PLATE_NORM_GROUPED ------------------------------------------------------------------------------------
def norm_plate(x, mean, sd, n_groups=1, chunk=64):
    """sum_i ld.norm(x_i, mean_i, sd) per chain -> (value, bound, median (x_i - mean_i)^2 / (2 sd sd)). x: [n]; mean: [C] (NORM_IID) or [C, n] (the group
    mean of each point, NORM_GROUPED); sd: [C].

    The plate computes n (c0 - log sd) - S / (2 sd sd), S = sum_i (x_i - mean_i)^2 (csrc sum_sq_dev, norm_factorised). Its error is
    at most:
      d   x_i - mean_i in fp64: relative u on d_i, so 2u + u^2 on d_i^2;
      S   fma accumulation into four accumulators after a one-point alignment peel, blocks and tail, one partial sum per ring tile or
          per group added in order: gamma_(n/4 + n/2048 + groups + 4) sum_i d_i^2;
      q   S / (2 sd sd): two roundings, and S's error carried through;
      c   n (c0 - log sd): c0 and log sd within 1 ulp each and three roundings: 4 u n (|c0| + |log sd|);
      out the final difference: u |value|."""
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    sd = np.asarray(sd, dtype=np.float64).reshape(-1)
    mean = np.asarray(mean, dtype=np.float64)
    C = sd.size
    per_point = mean.ndim == 2
    xL = x.astype(LD)
    c0 = LD(-0.5) * np.log(LD(2) * LD(JS_PI))
    depth = -(-n // 4) + -(-n // 2048) + n_groups + 4
    value = np.empty(C, dtype=LD)
    bound = np.empty(C)
    med = np.empty(C)
    for a0 in range(0, C, chunk):
        m = mean[a0:a0 + chunk]
        s = sd[a0:a0 + chunk].astype(LD)
        d = xL[:, None] - (m.T if per_point else m[None, :]).astype(LD)           # [n, c]
        d2 = d * d
        S = d2.sum(axis=0)
        ls = np.log(s)
        k = LD(2) * s * s
        A = LD(n) * (c0 - ls)
        v = A - S / k
        value[a0:a0 + chunk] = v
        Sf, kf = S.astype(np.float64), k.astype(np.float64)
        dS = (2 * U + U * U + gamma(depth)) * Sf
        q_err = (dS + 3 * U * Sf) / kf
        c_err = 4 * U * n * (abs(float(c0)) + np.abs(ls.astype(np.float64)))
        bound[a0:a0 + chunk] = q_err + c_err + U * (np.abs(A.astype(np.float64)) + Sf / kf) + U * np.abs(v.astype(np.float64))
        med[a0:a0 + chunk] = np.median((d2 / k[None, :]).astype(np.float64), axis=0)    # a row changes S / (2 sd sd) by this
    return value, bound, med


def group_means(mu, g):
    """[C, J] group means, [n] sorted group ids -> [C, n] the mean of each point"""
    return np.asarray(mu, dtype=np.float64)[:, np.asarray(g, dtype=np.int64)]


# ---- data sets and the oracle's models -----------------------------------------------------------------------------------------
def pois_data(K, n, seed):
    rng = np.random.default_rng(seed)
    X = np.column_stack([np.ones(n), rng.normal(0, 0.4, (n, K - 1))])
    beta = np.concatenate([[0.3], rng.normal(0, 0.25 / np.sqrt(K), K - 1)])
    y = rng.poisson(np.exp(X @ beta)).astype(float)
    return y, X


def edge_data(n, seed, kind):
    """K = 8, last column of X all zero. The initial state beta = (1, 0, ..., 0) puts eta_i = X_i0.
    "mixed": ordinary rows, a run of zero counts, counts near 1e4, and rows with eta = -750 and y > 0 (exp underflows).
    "high": every eta in (690, 694): finite, but beyond the table exp's range (the library exp, out of line). The counts are of the
    order of exp(eta), so the posterior stays there and every row adds exp(eta) ~ 1e300 (sum_i y_i eta_i stays below 1e308)."""
    rng = np.random.default_rng(seed)
    K = 8
    X = np.column_stack([rng.normal(0.5, 0.3, n), rng.normal(0, 0.3, (n, K - 2)), np.zeros(n)])
    if kind == "high":
        X[:, 0] = rng.uniform(690, 694, n)
        X[:, 1:K - 1] *= 1e-3
        y = np.floor(np.exp(X[:, 0]) * rng.uniform(0.5, 1.5, n))
    else:
        y = rng.poisson(np.exp(X[:, 0])).astype(float)
        y[5:40] = 0.0
        X[50:90, 0] = 9.2
        y[50:90] = rng.poisson(1e4, 40)
        X[100:105, 0] = -750.0
        y[100:105] = [1, 2, 3, 1, 7]
    return y, X


def ragged_groups(total, seed):
    """sorted group ids with sizes 1 and 2, an empty group (a gap in g), odd starts, and one large group taking the rest"""
    sizes = [1, 2, 0, 5, 3, 1, 17, 2, 9, 1]
    sizes.append(total - sum(sizes))
    g = np.repeat(np.arange(len(sizes)), sizes)
    rng = np.random.default_rng(seed)
    y = rng.normal(100, 20, len(sizes))[g] + rng.normal(0, 5, total)
    return y, g, len(sizes)


def oracle_logpost(orc, name, data, params, states):
    """orc_model_<name> (the oracle's term-by-term log_post) at each state"""
    import ctypes
    s = orc.OracleSampler(name, data, params)
    fn = getattr(orc.lib(), "orc_model_" + name)
    fn.restype = ctypes.c_double
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    dptr = ctypes.cast(ctypes.pointer(s._keep[-1]), ctypes.c_void_p)
    out = []
    for st in states:
        buf = np.array(list(st) + [0.0] * 4, dtype=np.float64)
        out.append(fn(buf.ctypes.data, dptr, None))
    return np.array(out)
