"""The split-chain records of amwg_summary_autocov without a GPU: the kernel's own per-half-chain text (csrc/amwg_autocov.cuh) built
for the host with the kernel's launch (tests/host_shim/autocov_host.cpp) at every small (rows, lag0, n_lags), held to the exact
restatement of tests/autocov_ref.py within its bound; that restatement against a rational-arithmetic loop; Geyer's decisions over
the bound; and the ESS and split R-hat unchanged, bit for bit, when the draws are scaled by a power of two."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import autocov_ref
from ess_ref import NumpyAutocovReducer, ar1, autocov_scale

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("autocov") / "libautocov_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-fPIC", "-shared", "-ffp-contract=off",
           "-I" + os.path.join(ROOT, "tests", "host_shim"), "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"),
           os.path.join(ROOT, "tests", "host_shim", "autocov_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    lib.hs_autocov.restype = C.c_int
    lib.hs_autocov.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    lib.hs_autocov_scale.restype = C.c_double
    lib.hs_autocov_scale.argtypes = [C.c_double, C.c_double]
    return lib


def _host(H, x, thr, lag0, n_lags):
    x = np.ascontiguousarray(x, dtype=np.float64)
    rows, entries, chains = x.shape
    ns = 1 if thr is None else 3
    out = np.full((entries, ns, 4 + n_lags), np.nan)
    t = None if thr is None else np.ascontiguousarray(thr, dtype=np.float64)
    assert H.hs_autocov(x.ctypes.data, rows, entries, chains, None if t is None else t.ctypes.data, lag0, n_lags, out.ctypes.data) == 0
    return out


def _block(rows, chains, seed):
    """[rows, 4, chains]: AR(0.6) far from 0, integers with ties, a constant, and chains each stuck at a value of their own in
    their first half"""
    x = ar1(0.6, rows, chains, 4, seed)
    x[:, 0] = 184.5 + 0.14 * x[:, 0]
    x[:, 1] = np.round(2 * x[:, 1])
    x[:, 2] = 7.25
    x[:rows // 2, 3] = 0.1 * np.arange(chains)[None, :]
    return x


def _thr(x):
    return np.stack([np.quantile(np.moveaxis(x, 1, 0).reshape(x.shape[1], -1), p, axis=1) for p in (0.05, 0.95)], axis=1)


@pytest.mark.parametrize("rows", range(10, 41))
def test_kernel_text_at_every_small_window(H, rows):
    """every (lag0, n_lags) with n_lags in 1..32 inside the half, both kernel passes (windows of more than 16 lags when h >= 17) and
    ring slots past h, for NS = 1 and NS = 3: every record within the bound, and each lag's sum the same bits whichever window
    asks for it"""
    h = rows // 2
    x = _block(rows, 7, rows)
    for thr in (None, _thr(x)):
        exact, bound = autocov_ref.record(x, thr, 0, h)
        full = _host(H, x, thr, 0, h)
        autocov_ref.check_record(full, exact, bound, (rows, thr is None))
        n = 0
        for lag0 in range(h):
            for n_lags in range(1, min(32, h - lag0) + 1):
                got = _host(H, x, thr, lag0, n_lags)
                assert got[:, :, :4].tobytes() == full[:, :, :4].tobytes(), (rows, lag0, n_lags)
                assert got[:, :, 4:].tobytes() == full[:, :, 4 + lag0:4 + lag0 + n_lags].tobytes(), (rows, lag0, n_lags)
                n += 1
        assert n == h * (h + 1) // 2


def test_kernel_text_walks_several_chains_a_thread(H):
    """more chains than 1184 x 256 threads: a thread walks two chains; records within the bound taken for two chains a thread"""
    x = ar1(0.3, 10, 1184 * 256 + 77, 1, 4) * 3.0 - 1.0
    thr = _thr(x)
    exact, bound = autocov_ref.record(x, thr, 0, 5)
    autocov_ref.check_record(_host(H, x, thr, 0, 5), exact, bound)


def test_reference_against_exact_rationals(pkg):
    """record()'s lag sums and sum_w within 3 u sum |d_n d_n+t| of the exact sums of its own centred values (Fractions)"""
    x = _block(13, 5, 2)
    thr = _thr(x)
    h = 6
    exact, _ = autocov_ref.record(x, thr, 0, h)
    for e in range(4):
        for s in range(3):
            d, _m = autocov_ref.centred(x, thr, e, s)
            for t in range(h):
                want = sum(Fraction(float(a)) * Fraction(float(b)) for row in d for a, b in zip(row[:h - t], row[t:]))
                ab = float(np.sum(np.abs(d[:, :h - t] * d[:, t:])))
                assert abs(Fraction(exact[e, s, 4 + t]) - want) <= 3 * autocov_ref.U * ab, (e, s, t)
            assert exact[e, s, 3] == exact[e, s, 4]


def test_means_are_the_devices_bits(H):
    """the restated half-chain means and scale are the host build's bits: a constant entry's record has its value times the scale
    as the mean and exactly zero M2, sum_w and lag sums"""
    x = _block(22, 9, 5)
    thr = _thr(x)
    got = _host(H, x, thr, 0, 3)
    sc = autocov_scale(*thr[2])
    assert sc == H.hs_autocov_scale(*thr[2]) == 1.0                     # q05 == q95: not scaled
    assert got[2, 0, 1] == 7.25 and np.all(got[2, 0, 2:] == 0)
    for q05, q95 in [(-1.0, 1.0), (0.0, 3.0), (1e-310, 2e-310), (-1e308, 1e308), (5.0, 5.0), (0.0, np.inf), (np.nan, 1.0), (1e-320, 1e-300)]:
        assert H.hs_autocov_scale(q05, q95) == autocov_scale(q05, q95), (q05, q95)
    assert autocov_scale(-1.0, 1.0) == 1.0 and autocov_scale(1e-310, 2e-310) == 2.0 ** 1023 and autocov_scale(-1e308, 1e308) == 2.0 ** -1022


def _ess_of(rec, h):
    from bayes_js_b200.summary import GeyerESS
    g = GeyerESS(rec, h)
    g.add(rec[4:])
    return g


@pytest.mark.parametrize("phi", [0.9, 0.6, 0.0, -0.4])
def test_geyer_decisions_over_the_bound(H, pkg, phi):
    """GeyerESS of the host build's record lies in autocov_ref.interval of the exact record, for every series of 40 seeds;
    every case is decided"""
    rows, chains = 60, 24
    decided = total = 0
    for seed in range(40):
        x = ar1(phi, rows, chains, 1, seed)
        thr = _thr(x)
        h = rows // 2
        exact, bound = autocov_ref.record(x, thr, 0, h)
        got = _host(H, x, thr, 0, h)
        for s in range(3):
            total += 1
            iv = autocov_ref.interval(exact[0, s], bound[0, s], h)
            if iv is None:
                continue
            decided += 1
            g = _ess_of(got[0, s], h)
            assert autocov_ref.inside(g.ess, iv[0]), (phi, seed, s, g.ess, iv[0])
            assert autocov_ref.inside(g.varplus / g.W, iv[1]), (phi, seed, s)
    assert decided == total, (decided, total)


SCALES = (-1000, -560, -300, 0, 300, 511, 900)


def _diag(x, red=None):
    import torch
    from bayes_js_b200.summary import summarise_block
    rows, _, chains = x.shape
    *_, (d, _w) = summarise_block(red or NumpyAutocovReducer(), torch.from_numpy(x), rows, chains, (0.5,), False, diagnostics=True)
    return d


def test_ess_and_rhat_do_not_depend_on_the_scale(pkg):
    """AR(0.6) draws times 2^j give the bits of ess_mean, ess_tail and rhat_split of the unscaled draws at every j where the scaled
    draws stay normal (before the scaling, 2^-560 and 2^511 gave ESS 52572, four times the draws)"""
    x = ar1(0.6, 200, 64, 1, 3)
    base = _diag(x)
    assert 3000 < base["ess_mean"][0] < 3500
    for j in SCALES:
        xs = np.ldexp(x, j)
        assert np.all(np.abs(xs) >= 2.0 ** -1022) and np.all(np.isfinite(xs)), j
        d = _diag(xs)
        for k in ("ess_mean", "ess_tail", "rhat_split"):
            assert d[k].tobytes() == base[k].tobytes(), (j, k, d[k], base[k])


def test_what_cannot_be_computed_is_nan(pkg):
    """an entry with q05 == q95 (not scaled) whose squares underflow, and an entry whose scaled outliers overflow: ESS and
    rhat_split NaN, never a finite value; the other entries keep their values"""
    rng = np.random.default_rng(7)
    rows, chains = 40, 32
    x = np.empty((rows, 3, chains))
    x[:, 0] = ar1(0.5, rows, chains, 1, 8)[:, 0]
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.97, 1.0, 1.0 + rng.normal(size=(rows, chains))) * 2.0 ** -600
    x[:, 2] = np.where(rng.uniform(size=(rows, chains)) < 0.97, 1e-300 * rng.normal(size=(rows, chains)), 1e300)
    d = _diag(x)
    assert np.isfinite(d["ess_mean"][0]) and np.isfinite(d["rhat_split"][0])
    for e in (1, 2):
        assert np.isnan(d["ess_mean"][e]) and np.isnan(d["rhat_split"][e]), (e, d)
    assert np.isnan(d["mcse_mean"][2])
