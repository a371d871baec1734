"""Reference for the posterior covariance of sample_summary(..., covariance=...): the shard record {C, m, B, W} of
amwg_summary_comoments computed with math.fsum from the draws (chain means and the mean of the chain means exact to one
rounding), and a worst-case forward-error bound for what the device computes.

The bound, per element (i, j), follows the operations of the device (csrc/amwg_summary.cuh, K_c1..K_c4), in the manner of
tests/plate_ref.py (gamma_k = k u / (1 - k u), Higham 3.1):
  chain means   xbar_c = fl(fl(sum_r x_rc) / rows) is off the exact mean by at most dlt_c = gamma_{rows+1} mean_r |x_rc|.
  W             the device sums (x - xbar_c)(x - xbar_c)^T with its rounded xbar_c. Because sum_r (x_rc - exact mean) = 0, the
                shift of the centre adds exactly rows * dlt_ic dlt_jc per chain; the rounding of every centred value, of every
                product and of a summation of at most K = rows * chains terms plus G partials adds gamma_{K+G+3} sum_k |d_ik||d_jk|
                with |d| <= |x - exact mean| + dlt.
  m             the sum of C chain means, divided by C: off by at most mean_c dlt_c + gamma_{C+1} mean_c |xbar_c|  (= mu).
  B             with f_c = exact xbar_c - exact m and e_c = dlt_c + mean(dlt) + mu the error of (xbar_c - m): first order
                sum_c (|f_ic| e_jc + e_ic |f_jc|) + sum_c e_ic e_jc, then the roundings gamma_{C+G+3} sum_c (|f_ic| + e_ic)(|f_jc| + e_jc).
Test infrastructure only."""
import math

import numpy as np

U = 2.0 ** -53
G_MAX = 264 * 16                 # amwg_comoments.cuh: kCoCtas x the most reps, the most partial tiles summed per element


def gamma(k) -> float:
    k = float(k)
    return k * U / (1.0 - k * U)


def exact_record(x: np.ndarray, sel) -> tuple:
    """x [rows, entries, chains] -> (C, m [n], B [n, n], W [n, n]) with fsum; every value within one rounding of the exact one."""
    rows, _entries, C = x.shape
    d = np.asarray(x[:, list(sel), :], dtype=np.float64)                     # [rows, n, C]
    n = d.shape[1]
    xbar = np.array([[math.fsum(d[:, s, c]) / rows for c in range(C)] for s in range(n)])        # [n, C]
    m = np.array([math.fsum(xbar[s]) / C for s in range(n)])
    e = d - xbar[None]                                                       # centred by the (correctly rounded) chain means
    f = xbar - m[:, None]
    W = np.empty((n, n))
    B = np.empty((n, n))
    ef = e.transpose(1, 0, 2).reshape(n, -1)
    for i in range(n):
        for j in range(i, n):
            W[i, j] = W[j, i] = math.fsum(ef[i] * ef[j])
            B[i, j] = B[j, i] = math.fsum(f[i] * f[j])
    return float(C), m, B, W


def device_bound(x: np.ndarray, sel) -> tuple:
    """-> (bound of m [n], bound of B [n, n], bound of W [n, n]) for the device record of x's selected entries against
    exact_record, as derived above. The reference's own centres are off by less than the device's (two roundings), so the
    centring terms are doubled, and its rounded products add u times the magnitudes."""
    rows, _entries, C = x.shape
    d = np.asarray(x[:, list(sel), :], dtype=np.float64)
    xbar = d.mean(axis=0)                                                    # [n, C]: magnitudes only
    dlt = gamma(rows + 1) * np.abs(d).mean(axis=0)
    mu = dlt.mean(axis=1) + gamma(C + 1) * np.abs(xbar).mean(axis=1)       # [n]
    ad = (np.abs(d - xbar[None]) + dlt[None]).transpose(1, 0, 2).reshape(d.shape[1], -1)        # [n, K]
    bW = 2 * rows * dlt @ dlt.T + gamma(rows * C + G_MAX + 3) * ad @ ad.T
    f = np.abs(xbar - xbar.mean(axis=1, keepdims=True))
    e = dlt + dlt.mean(axis=1, keepdims=True) + mu[:, None]
    bB = 2 * (f @ e.T + e @ f.T + e @ e.T) + gamma(C + G_MAX + 3) * (f + e) @ (f + e).T
    Wabs = ad @ ad.T
    Babs = (f + e) @ (f + e).T
    return mu + U * np.abs(xbar).mean(axis=1), bB + U * Babs, bW + U * Wabs


def check_record(got, x: np.ndarray, sel, what=""):
    """got: a flat record of the selected entries of x; asserts C, and m, B, W within device_bound of exact_record."""
    n = len(sel)
    C, m, B, W = exact_record(x, sel)
    bm, bB, bW = device_bound(x, sel)
    got = np.asarray(got)
    assert got.size == 1 + n + 2 * n * n
    gm, gB, gW = got[1:1 + n], got[1 + n:1 + n + n * n].reshape(n, n), got[1 + n + n * n:].reshape(n, n)
    assert got[0] == C, what
    assert np.all(np.abs(gm - m) <= bm), (what, "m", float(np.max(np.abs(gm - m) / bm)))
    assert np.all(np.abs(gB - B) <= bB), (what, "B", float(np.max(np.abs(gB - B) / bB)))
    assert np.all(np.abs(gW - W) <= bW), (what, "W", float(np.max(np.abs(gW - W) / bW)))
    assert np.array_equal(gB, gB.T) and np.array_equal(gW, gW.T), what
