"""Reference for the moment record of amwg_summary_moments, [entries, 4] = (chains, mean of the chain means, M2 of the chain
means, sum of the within-chain M2): the chain-level record of tests/nested_ref.py (_superchain over all chains of a block),
exact to a few roundings, with its worst-case bound.

The bound of nested_ref covers this kernel pair, because it follows the same operations (csrc/amwg_summary.cuh):
  - every chain's record comes from chain_record (csrc/amwg_nested.cuh), as in amwg_summary_nested;
  - the records are combined with the same merge, and every merge order is a binary tree: in K_m1 a thread merges its
    ceil(C / (1184 * 256)) chains in sequence, then the CTA's 256 records go through a fixed tree; in K_m2 a thread merges at most
    two of the <= 1184 CTA records, then a fixed 1024-thread tree;
  - so a mean passes through at most ceil(C / (1184 * 256)) + 8 + 2 + 10 steps, far fewer than the n + 20 the bound allows
    by default; record() passes this count as L, which keeps the bound within a few percent of the M2 at 2^20 chains.
Higham's model behind it has no underflow term, so a block of subnormals is held to it only where the absolute rounding error
of a subnormal result (2^-1075) is within 2 u |x|: for values in [2^-1023, 2^-1022).

record() restates _superchain with the per-chain sums vectorised over chains (a compensated sum along the rows, Ogita, Rump &
Oishi's Sum2: off the exact sum by at most u |sum| + gamma_{n-1}^2 sum |x|, far inside the bound) and math.fsum for the sums
over chains; test_summary_host checks that it agrees with _superchain. Test infrastructure only."""
import math

import numpy as np

from nested_ref import _chan_bound, gamma


def _sum2(a: np.ndarray) -> np.ndarray:
    """sum over axis 0, compensated (Sum2): TwoSum of each partial sum, the errors summed apart and added at the end"""
    s = np.zeros(a.shape[1:])
    c = np.zeros(a.shape[1:])
    for v in a:
        t = s + v
        z = t - s
        c += (s - (t - z)) + (v - z)
        s = t
    return s + c


def record(x: np.ndarray):
    """x [rows, entries, chains] -> (exact [entries, 4], bound [entries, 4]): nested_ref._superchain(x, e, 0, chains) per entry,
    its bound taken with the merge steps of amwg_summary_moments"""
    x = np.asarray(x, dtype=np.float64)
    N, entries, C = x.shape
    with np.errstate(invalid="ignore", over="ignore"):
        m = _sum2(x) / N                                           # [entries, C]: the chain means
        dev = x - m[None]
        m2c = _sum2(dev * dev)                                     # the within-chain M2, of the rounded squares as fsum((col - m) ** 2)
        dlt = gamma(N + 1) * np.mean(np.abs(x), axis=0)
        e_m2 = N * dlt * dlt + gamma(N + 2) * np.sum((np.abs(dev) + dlt[None]) ** 2, axis=0)
    exact = np.zeros((entries, 4))
    bound = np.zeros((entries, 4))
    for e in range(entries):
        means = m[e]
        mean = math.fsum(means) / C
        exact[e] = (C, mean, math.fsum((means - mean) ** 2), math.fsum(m2c[e]))
        bm, bm2, bsw = _chan_bound(means, dlt[e], [0.0], [0.0], m2c[e], e_m2[e], steps=-(-C // (1184 * 256)) + 20)
        bound[e] = (0.0, bm, bm2, bsw)
    return exact, bound


def check_record(got, x: np.ndarray, what=""):
    """got [entries, 4] from amwg_summary_moments against record(): the chain count equal, the other fields within the bound"""
    exact, bound = record(x)
    got = np.asarray(got)
    assert np.array_equal(got[:, 0], exact[:, 0]), (what, got[:, 0], exact[:, 0])
    err = np.abs(got - exact)
    ok = err <= bound
    assert np.all(ok), (what, np.argwhere(~ok)[:5], got[~ok][:5], exact[~ok][:5], bound[~ok][:5])
    return exact, bound
