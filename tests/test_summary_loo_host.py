"""Host side of PSIS-LOO and WAIC in sample_summary(..., loo=...): summary.loo_block with a numpy stand-in for the device reductions
(whose Pareto fit is csrc/amwg_loo.cuh compiled for the host) against the numpy restatement of tests/loo_ref.py, on chosen ll
matrices; the header's fit and smoothing against loo_ref, and on synthetic generalised Pareto samples of known k; a gloo world of
two uneven shards against world 1; the traced log_lik program on the CPU evaluator against the oracle's ld.* per point; and every
refusal of the argument, raised before the chains move."""
import ctypes as C
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import loo_ref
from summary_ref import ChanBlockReducer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    out = os.path.join(str(out_dir), "libloo_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "loo_host.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _load(path):
    lib = C.CDLL(path)
    lib.hs_loo_fit.restype = None
    lib.hs_loo_fit.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.hs_loo_smoothed.restype = None
    lib.hs_loo_smoothed.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p]
    lib.hs_loo_fit_m.restype = C.c_int
    lib.hs_loo_fit_m.argtypes = [C.c_int]
    lib.hs_loo_max_tail.restype = C.c_int
    lib.hs_loo_max_m.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    return _load(_build(tmp_path_factory.mktemp("loo_host")))


def host_fit(H, x):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty(2)
    H.hs_loo_fit(x.ctypes.data, len(x), out.ctypes.data)
    return out[0], out[1]


def host_smoothed(H, n, k, sigma, expcut):
    out = np.empty(n)
    H.hs_loo_smoothed(n, k, sigma, expcut, out.ctypes.data)
    return out


class StandInReducer(ChanBlockReducer):
    """The device reductions of loo_block on CPU tensors: finite range, moments and digit counts as the summary tests have them,
    the sums-and-tail pass in numpy, and the fit kernel's steps with the fit and smoothing of the host-compiled amwg_loo.cuh.
    `tails` records every point's tail as the fit saw it (sorted ll, descending)."""

    def __init__(self, H):
        self.H = H
        self.tails = []

    def finite_range(self, block):
        x = block.numpy()
        rows, P, chains = x.shape
        rng = np.empty((P, 2))
        nf = np.zeros((P, 3), dtype=np.int64)
        for p in range(P):
            v = x[:, p, :].ravel()
            f = v[np.isfinite(v)]
            rng[p] = (f.min(), f.max()) if f.size else (np.inf, -np.inf)
            nf[p] = (np.sum(v == -np.inf), np.sum(v == np.inf), np.sum(np.isnan(v)))
        return torch.from_numpy(rng), torch.from_numpy(nf)

    def loo_reduce(self, ll, llmin, llmax, cut, cap):
        x = ll.numpy()
        rows, P, chains = x.shape
        sums = np.empty((P, 3))
        tails = np.zeros((P, cap))
        counts = np.zeros(P, dtype=np.int32)
        with np.errstate(invalid="ignore", over="ignore"):
            for p in range(P):
                v = x[:, p, :].T.ravel()
                lw = llmin[p] - v
                t = lw > cut[p]
                sums[p] = (np.sum(np.exp(v - llmax[p])), np.sum(np.exp(lw[~t])), np.sum(np.exp((lw + v) - llmin[p])[~t]))
                counts[p] = t.sum()
                tails[p, :min(t.sum(), cap)] = v[t][:cap]
        return sums, torch.from_numpy(tails), torch.from_numpy(counts)

    def loo_fit(self, tails, counts, llmin, cut, skip):
        R, P, cap = tails.shape
        out = np.empty((P, 4))
        t, c = tails.numpy(), counts.numpy()
        for p in range(P):
            a = np.concatenate([t[r, p, :min(c[r, p], cap)] for r in range(R)])
            a = -np.sort(-a)
            self.tails.append(a)
            n = len(a)
            if skip[p]:
                out[p] = (np.nan, np.nan, np.nan, n)
                continue
            k, lw = np.inf, llmin[p] - a
            if n > 4:
                expcut = np.exp(cut[p])
                k, sigma = host_fit(self.H, np.exp(llmin[p] - a) - expcut)
                if np.isfinite(k):
                    lw = host_smoothed(self.H, n, k, sigma, expcut)
            out[p] = (k, np.sum(np.exp(lw)), np.sum(np.exp((lw + a) - llmin[p])), n)
        return out


class ArraySource:
    def __init__(self, ll3):
        self.ll3 = np.ascontiguousarray(ll3, dtype=np.float64)           # [rows, points, chains]

    def chunk(self, p0, P):
        return torch.from_numpy(np.ascontiguousarray(self.ll3[:, p0:p0 + P, :]))


def _flat(ll3):
    rows, N, chains = ll3.shape
    return np.moveaxis(ll3, 1, 2).reshape(rows * chains, N)


def run_loo(H, ll3, r_eff=1.0, chunk=None):
    from bayes_js_b200.summary import loo_block
    rows, N, chains = ll3.shape
    red = StandInReducer(H)
    out = loo_block(red, ArraySource(ll3), rows, chains, N, r_eff, chunk or N, False)
    return out, red


def assert_matches(out, ref, red, ll, rtol=1e-12):
    S, N = ll.shape
    for i in range(N):
        if ref["tails"][i] is None:
            continue
        mine = red.tails[i]
        want = -np.sort(-ll[ref["tails"][i], i])
        assert len(mine) == len(want) and np.array_equal(mine, want), i          # the same tail draws
    for key, want in ref["pointwise"].items():
        got = out["pointwise"][key]
        assert np.array_equal(np.isnan(got), np.isnan(want)), key
        ok = ~np.isnan(want)
        scale = np.maximum(1.0, np.abs(ref["pointwise"]["lppd"][ok]))
        if key == "pareto_k":
            assert np.array_equal(np.isinf(got[ok]), np.isinf(want[ok]))
            fin = ok & np.isfinite(want)
            assert np.all(np.abs(got[fin] - want[fin]) <= rtol * np.maximum(1.0, np.abs(want[fin]))), (got, want)
        else:
            assert np.all(np.abs(got[ok] - want[ok]) <= rtol * scale * 8), (key, got[ok] - want[ok])
    for key in ("elpd_loo", "p_loo", "elpd_waic", "p_waic", "se_elpd_loo", "se_elpd_waic", "looic", "waic"):
        if np.isnan(ref[key]):
            assert np.isnan(out[key]), key
        else:
            assert abs(out[key] - ref[key]) <= 1e-10 * max(1.0, abs(ref[key])), (key, out[key], ref[key])
    assert out["n_high_k"] == ref["n_high_k"] and out["pareto_k_threshold"] == ref["pareto_k_threshold"]
    assert out["n_draws"] == S and out["points"] == N


def _normal_ll(rows, chains, y, seed, df=None):
    """ll3 [rows, N, chains] of a normal model's draws of (mu, sigma) at data y."""
    rng = np.random.default_rng(seed)
    mu = rng.normal(np.mean(y), np.std(y) / np.sqrt(len(y)), size=(rows, 1, chains))
    sd = np.std(y) * np.sqrt(rng.chisquare(len(y) - 1, size=(rows, 1, chains)) / (len(y) - 1))
    yy = np.asarray(y, dtype=np.float64)[None, :, None]
    return -0.5 * np.log(2 * np.pi) - np.log(sd) - (yy - mu) ** 2 / (2 * sd * sd)


# ---- the ll matrices of the cases: one list, which tests/test_gpu_summary_loo_reduce.py runs through the device reductions ----
def case_well_behaved():
    return _normal_ll(4, 500, np.random.default_rng(1).normal(3.0, 2.0, 30), 2)


def case_heavy_tailed():
    y = np.random.default_rng(3).normal(0.0, 1.0, 12)
    y[5] = 9.0                                                     # an outlier: its leave-one-out weights have a heavy tail
    return _normal_ll(2, 2000, y, 4)


def case_small_sample():
    return _normal_ll(2, 60, np.random.default_rng(5).normal(0, 1, 7), 6)        # S = 120: 0.2 S = 24 < 3 sqrt(S) = 32.9


def case_tied_discrete():
    rng = np.random.default_rng(7)
    theta = rng.choice([0.2, 0.35, 0.5, 0.65], size=(3, 1, 400))               # few distinct draws: ll ties everywhere
    y = rng.integers(0, 2, 15).astype(float)[None, :, None]
    return np.log(y * theta + (1 - y) * (1 - theta))


def case_tail_of_four():
    return _normal_ll(1, 20, np.random.default_rng(8).normal(0, 1, 5), 9)        # S = 20: M = 4


def case_dbl_min_floor():
    rng = np.random.default_rng(10)
    S, N = 1000, 3
    ll = rng.normal(0.0, 1.0, size=(S, N))
    ll[:50] -= 1000.0                                              # 50 draws far below: the 96th largest lw is under log(DBL_MIN)
    return ll.reshape(1, S, N).transpose(0, 2, 1).copy()


def case_non_finite():
    ll3 = _normal_ll(2, 100, np.random.default_rng(11).normal(0, 1, 6), 12)
    ll3[1, 2, 17] = -np.inf
    ll3[0, 4, 3] = np.nan
    return ll3


def case_forced_chunks():
    return _normal_ll(3, 150, np.random.default_rng(13).normal(1, 2, 11), 14)


def case_r_eff():
    return _normal_ll(2, 300, np.random.default_rng(15).normal(0, 1, 4), 16)


def case_two_valued(rows, chains, c, seed):
    """the ll of a binary observation: log 0.2 at c draws (the rarer state) and log 0.8 at the others, and the mirror point.
    With c <= M the first point's tail is exactly the c tied draws."""
    S = rows * chains
    low = np.zeros(S, dtype=bool)
    low[np.random.default_rng(seed).choice(S, c, replace=False)] = True
    ll = np.stack([np.where(low, np.log(0.2), np.log(0.8)), np.where(low, np.log(0.8), np.log(0.2))], axis=1)
    return ll.reshape(rows, chains, 2).transpose(0, 2, 1).copy()


def case_zero_x_quarter():
    """a tail of M = 269 (S = 8000) whose 100 smallest lw sit within 1e-19 of the cut: exp(lw) - exp(cut) rounds to 0 for them,
    so the fit's first quartile x_q is 0 and every candidate b is infinite"""
    rng = np.random.default_rng(21)
    S, M = 8000, 269
    ll = np.full(S, -1e-5)                                         # the bulk: lw = cut exactly (llmin - ll, exact by Sterbenz)
    ll[:100] = -1e-5 - np.arange(1, 101) * 2e-21                   # a hair below the bulk: lw a hair above the cut
    ll[100:M - 1] = rng.uniform(-2e-5, -1.1e-5, M - 101)
    ll[M - 1] = -2e-5                                              # llmin
    ll = ll[rng.permutation(S)]
    return np.stack([ll, ll[::-1]], axis=1).reshape(2, 4000, 2).transpose(0, 2, 1).copy()


# name -> (builder of ll3 [rows, points, chains], r_eff)
CASES = {
    "well_behaved": (case_well_behaved, 1.0),
    "heavy_tailed": (case_heavy_tailed, 1.0),
    "small_sample": (case_small_sample, 1.0),
    "tied_discrete": (case_tied_discrete, 1.0),
    "tail_of_four": (case_tail_of_four, 1.0),
    "dbl_min_floor": (case_dbl_min_floor, 1.0),
    "non_finite": (case_non_finite, 1.0),
    "forced_chunks": (case_forced_chunks, 1.0),
    "r_eff": (case_r_eff, 0.3),
    "two_valued_c60": (lambda: case_two_valued(2, 4000, 60, 22), 1.0),      # S = 8000, M = 269: a tail of 60 tied draws
    "two_valued_c110": (lambda: case_two_valued(2, 4000, 110, 23), 1.0),    # a tail of 110: candidate 3 of m = 40 has b = 0
    "two_valued_c700": (lambda: case_two_valued(3, 20000, 700, 24), 1.0),   # S = 60000, M = 735: a tail of 700, b_4 of 56 = 0
    "zero_x_quarter": (case_zero_x_quarter, 1.0),
}


def run_case(H, name, chunk=None):
    build, r_eff = CASES[name]
    ll3 = build()
    out, red = run_loo(H, ll3, r_eff, chunk)
    ref = loo_ref.loo(_flat(ll3), r_eff)
    assert_matches(out, ref, red, _flat(ll3))
    return out, ref, ll3


def test_well_behaved_model(H):
    out, _, _ = run_case(H, "well_behaved")
    assert np.all(np.isfinite(out["pointwise"]["pareto_k"]))


def test_heavy_tailed_point(H):
    out, _, _ = run_case(H, "heavy_tailed")
    assert out["pointwise"]["pareto_k"][5] > 0.7 and out["n_high_k"] >= 1


def test_small_sample_where_the_tail_is_a_fifth(H):
    assert 0.2 * 120 < 3 * math.sqrt(120)
    run_case(H, "small_sample")


def test_tied_ll_of_discrete_data(H):
    run_case(H, "tied_discrete")


def test_tail_of_at_most_four_draws(H):
    out, _, _ = run_case(H, "tail_of_four")
    assert np.all(np.isinf(out["pointwise"]["pareto_k"]))


def test_log_dbl_min_floor(H):
    ll = _flat(case_dbl_min_floor())
    assert all(loo_ref.psis_point(ll[:, i])["cut"] == loo_ref.LOG_TINY for i in range(ll.shape[1]))
    run_case(H, "dbl_min_floor")


def test_non_finite_point(H):
    out, _, _ = run_case(H, "non_finite")
    for key, v in out["pointwise"].items():
        assert np.isnan(v[2]) and np.isnan(v[4]) and not np.isnan(v[0]), key
    assert np.isnan(out["elpd_loo"]) and np.isnan(out["waic"])


def test_several_forced_chunks(H):
    ll3 = case_forced_chunks()
    one, _ = run_loo(H, ll3)
    out, _, _ = run_case(H, "forced_chunks", chunk=3)
    for key in one["pointwise"]:
        assert np.array_equal(one["pointwise"][key], out["pointwise"][key]), key


def test_r_eff_moves_the_tail(H):
    out, _, _ = run_case(H, "r_eff")
    assert out["r_eff"] == 0.3


@pytest.mark.parametrize("name, c", [("two_valued_c60", 60), ("two_valued_c110", 110), ("two_valued_c700", 700)])
def test_tied_tail_of_a_binary_observation(H, name, c):
    """the rarer state's c <= M draws are the whole tail, all tied. At c = 110 and 700 one candidate b is 0 and its profile value
    NaN; left out, the fit stays finite, continuous with the tails around it, and so does every value of the point"""
    out, ref, ll3 = run_case(H, name)
    assert len(ref["tails"][0]) == c and ref["tails"][1].size == 0
    k = out["pointwise"]["pareto_k"][0]
    assert np.isfinite(k) and k < -5, k
    assert all(np.isfinite(v[0]) for v in out["pointwise"].values()) and np.isfinite(out["elpd_loo"])
    assert np.isinf(out["pointwise"]["pareto_k"][1])                  # the mirror point: an empty tail


def test_tail_whose_first_quartile_rounds_to_zero(H):
    """x = exp(lw) - exp(cut) is 0 for more than a quarter of the tail: every candidate is infinite, no profile value is finite,
    and the point keeps its raw weights with k = +inf (counted as high k), its other values finite"""
    out, ref, ll3 = run_case(H, "zero_x_quarter")
    ll = _flat(ll3)
    r = loo_ref.psis_point(ll[:, 0])
    x = np.exp(np.sort((ll[:, 0].min() - ll[:, 0])[r["tail"]])) - np.exp(r["cut"])
    assert len(x) == 269 and np.sum(x == 0) >= len(x) / 4 and x[int(len(x) / 4 + 0.5) - 1] == 0
    assert np.all(np.isinf(out["pointwise"]["pareto_k"])) and out["n_high_k"] == 2
    assert np.isfinite(out["elpd_loo"])


# ---- the header's fit and smoothing ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n, k, seed", [(5, 0.2, 1), (17, -0.3, 2), (100, 0.5, 3), (1000, 0.9, 4), (3000, 0.0, 5)])
def test_fit_and_smoothing_equal_the_restatement(H, n, k, seed):
    rng = np.random.default_rng(seed)
    x = np.sort(loo_ref.gpinv(rng.uniform(size=n), k, 1.7))
    got = host_fit(H, x)
    want = loo_ref.gpdfit(x)
    assert abs(got[0] - want[0]) <= 1e-12 * max(1, abs(want[0])) and abs(got[1] - want[1]) <= 1e-12 * abs(want[1])
    expcut = 0.37
    sm = host_smoothed(H, n, got[0], got[1], expcut)
    ref = np.log(loo_ref.gpinv(np.arange(0.5, n) / n, want[0], want[1]) + expcut)
    ref[ref > 0] = 0
    assert np.allclose(sm, ref, rtol=1e-12, atol=1e-14)


def test_fit_of_all_equal_tails_equals_the_restatement(H):
    """every n in 5..4000, an all-equal tail: for n with m = 16 j - 8 (100..120, 676..728, 1764..1848, 3364..3480) candidate j
    is b = 0 with a NaN profile value. Header and restatement leave it out alike and the fit stays finite for every n"""
    ks = []
    for v in (0.37, 1e-3):
        for n in range(5, 4001):
            x = np.full(n, v)
            got, want = host_fit(H, x), loo_ref.gpdfit(x)
            assert np.isfinite(got[0]) and np.isfinite(got[1]), (v, n, got)
            assert abs(got[0] - want[0]) <= 1e-9 * max(1.0, abs(want[0])) and abs(got[1] - want[1]) <= 1e-9 * abs(want[1]), (v, n, got, want)
            if v == 0.37:
                ks.append(got[0])
    d = np.diff(ks)                                                 # k falls with n, in small steps also where a candidate drops out
    assert np.all(d < 0) and np.max(np.abs(d[45:])) < 0.04, (np.argmax(d) + 5, np.max(np.abs(d[45:])))


def test_fit_kernel_arrays_hold_the_largest_tail(H):
    """the fit kernel's candidate arrays (kMaxM) hold the candidates of the largest tail the API accepts (kMaxTail)"""
    assert H.hs_loo_max_tail() == 1 << 20
    assert H.hs_loo_fit_m(H.hs_loo_max_tail()) <= H.hs_loo_max_m()
    assert H.hs_loo_fit_m(H.hs_loo_max_tail()) == 30 + 1024 == 30 + int((1 << 20) ** 0.5)
    from bayes_js_b200.summary import MAX_LOO_TAIL
    assert MAX_LOO_TAIL == H.hs_loo_max_tail()


@pytest.mark.parametrize("n, k, seed", [(5, 0.2, 1), (17, -0.3, 2), (100, 0.5, 3), (1000, 0.9, 4), (3000, 0.0, 5), (20000, 0.7, 6)])
def test_blocked_restatement_equals_the_whole_matrix(n, k, seed):
    """loo_ref.gpdfit forms k(b) over blocks of candidates (for n = 2^20 the whole m x n matrix would be 8.8 GB): the same fit"""
    x = np.sort(loo_ref.gpinv(np.random.default_rng(seed).uniform(size=n), k, 1.7))
    m = 30 + int(n ** 0.5)
    whole = loo_ref.gpdfit(x, block=m)
    for rows in (1, 7, None):
        got = loo_ref.gpdfit(x, block=rows)
        assert abs(got[0] - whole[0]) <= 1e-15 * max(1.0, abs(whole[0])) and abs(got[1] - whole[1]) <= 1e-15 * abs(whole[1]), (rows, got, whole)


@pytest.mark.parametrize("k", [-0.2, 0.3, 0.7])
def test_fit_recovers_a_known_k(H, k):
    rng = np.random.default_rng(42)
    n = 20000
    x = np.sort(loo_ref.gpinv(rng.uniform(size=n), k, 2.0))
    kh, sigma = host_fit(H, x)
    assert abs(kh - k) < 0.05 and abs(sigma / 2.0 - 1) < 0.1, (kh, sigma)


# ---- a gloo world of two uneven shards ---------------------------------------------------------------------------------------------
def _worker(rank, world, port, lib_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.summary import loo_block
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ll3 = _normal_ll(3, 200, np.random.default_rng(17).normal(0, 1.5, 9), 18)
        ll3[0, 6, 150] = 40.0                                    # one heavy point, its tail drawn from the second shard
        cut = 77
        mine = ll3[:, :, :cut] if rank == 0 else ll3[:, :, cut:]
        H = _load(lib_path)
        out = loo_block(StandInReducer(H), ArraySource(mine), 3, 200, 9, 1.0, 4, True)
        one = loo_block(StandInReducer(H), ArraySource(ll3), 3, 200, 9, 1.0, 4, False)
        ok = all(np.allclose(out["pointwise"][k], one["pointwise"][k], rtol=1e-12, atol=1e-12, equal_nan=True) for k in one["pointwise"])
        ok = ok and abs(out["elpd_loo"] - one["elpd_loo"]) <= 1e-10 * abs(one["elpd_loo"])
        q.put((rank, ok, np.concatenate([out["pointwise"][k] for k in sorted(out["pointwise"])]).tobytes()))
    finally:
        dist.destroy_process_group()


def test_loo_over_gloo_world2(tmp_path):
    """two uneven shards: every rank returns the same bytes, equal to one shard holding every chain within rounding"""
    import torch.multiprocessing as mp
    lib = _build(tmp_path)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, lib, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=180) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert all(ok for _, ok, _ in res)
    assert res[0][2] == res[1][2]


# ---- the traced log_lik program against the oracle's ld.* ---------------------------------------------------------------------------
def _eval_points(lik, prog, O, state, points):
    """The body at every point i < points on the CPU evaluator: DATA_I / COMP_I read column[off + stride * i], which the evaluator
    reads at its loop index 0 from the column shifted by stride * i (the strides come from the traced expression)."""
    import prog_eval                                               # needs the package: not at import (the gloo workers import this module)
    consts = prog_eval.fold_constants(prog, O)
    code = prog.code
    strides, stack = {}, [lik.expr]
    while stack:
        n = stack.pop()
        if n.op in ("DATA_I", "COMP_I"):
            strides.setdefault(n.val[0], set()).add(n.val[2])
        stack.extend(n.args)
    out = []
    cols = prog.columns
    for i in range(points):
        shifted = list(cols)
        for c, st in strides.items():
            assert len(st) == 1
            shifted[c] = np.asarray(cols[c])[next(iter(st)) * i:]
        view = type("P", (), {"code": code, "columns": shifted, "plates": prog.plates})
        out.append(prog_eval.run(view, consts, state, prog.logpost_prog, O, want_top=True))
    return np.array(out)


def _lik(pkg, log_lik, params, data, points):
    from bayes_js_b200.mcmc import complete_params
    from bayes_js_b200.tracer import trace_log_lik
    params = complete_params({k: dict(v) for k, v in params.items()}, pkg.mcmc.param_init_fixed)
    offsets, n = {}, 0
    for name, p in params.items():
        offsets[name] = n
        n += int(np.prod(p["dim"]))
    lik = trace_log_lik(log_lik, params, offsets, data, points)
    return lik, lik.lower({name: offsets[name] for name in lik.reads}), offsets


def test_traced_body_equals_the_oracle_per_point(pkg, orc):
    ld, Math = pkg.ld, pkg.mcmc.Math
    O = orc.lib()
    rng = np.random.default_rng(19)
    N, J = 12, 3
    d = {"y": rng.normal(1, 2, N).round(3).tolist(), "b": rng.integers(0, 2, N).astype(float).tolist(), "c": rng.poisson(3, N).astype(float).tolist(),
         "g": np.sort(rng.integers(0, J, N)).astype(float).tolist(), "X": rng.normal(0, 1, (N, 2)).round(3).tolist(), "s": [1.7, 2.3]}
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}, "p": {"type": "real", "lower": 0, "upper": 1},
              "a": {"type": "real", "dim": [J]}, "beta": {"type": "real", "dim": [2]}}
    state = [0.7, 1.9, 0.3, -0.4, 0.25, 1.1, 0.2, -0.6]
    cases = {
        "norm": (lambda s, dd, i: ld.norm(dd.y[i], s.mu, s.sigma), lambda i: O.orc_ld_norm(d["y"][i], state[0], state[1])),
        "bern": (lambda s, dd, i: ld.bern(dd.b[i], s.p), lambda i: O.orc_ld_bern(d["b"][i], state[2])),
        "grouped": (lambda s, dd, i: ld.norm(dd.y[i], s.a[dd.g[i]], s.sigma),
                    lambda i: O.orc_ld_norm(d["y"][i], state[3 + int(d["g"][i])], state[1])),
        "poisson": (lambda s, dd, i: ld.pois(dd.c[i], Math.exp(dd.X[i][0] * s.beta[0] + dd.X[i][1] * s.beta[1])),
                    lambda i: O.orc_ld_pois(d["c"][i], O.orc_exp(d["X"][i][0] * state[6] + d["X"][i][1] * state[7]))),
        "composed": (lambda s, dd, i: ld.norm(dd.y[i], s.mu, s.sigma) + ld.bern(dd.b[i], s.p) - Math.log(s.sigma * 2),
                     lambda i: (O.orc_ld_norm(d["y"][i], state[0], state[1]) + O.orc_ld_bern(d["b"][i], state[2])) - O.orc_log(state[1] * 2)),
        # a data element at a fixed index: its parameter-free terms (-0.5 log(2 pi) - log(sd), 2 sd sd) are folded, reading DATA
        "fixed_index": (lambda s, dd, i: ld.norm(dd.y[i], s.mu, dd.s[0]), lambda i: O.orc_ld_norm(d["y"][i], state[0], d["s"][0])),
    }
    for name, (f, want) in cases.items():
        lik, prog, _ = _lik(pkg, f, params, d, N)
        got = _eval_points(lik, prog, O, state, N)
        ref = np.array([want(i) for i in range(N)])
        assert np.array_equal(got.view(np.int64), ref.view(np.int64)), (name, got, ref)
        if name == "fixed_index":
            assert "DATA" in _fold_ops(prog)


def _fold_ops(prog):
    """the opcodes of the fold programs (instruction words only: inline operands and extra words skipped)"""
    from bayes_js_b200._ffi import OP
    inv = {v: k for k, v in OP.items()}
    extra = {"DATA": 1, "DATA_I": 2, "COMP_I": 3}
    ops = []
    for pc in prog.fold_prog:
        while True:
            w = prog.code[pc] & 0xffffffff
            op = inv[w & 0xff]
            ops.append(op)
            if op == "END":
                break
            inline = sum(1 for k in range(4) if ((w >> (8 + 2 * k)) & 3) in (1, 2))
            pc += 1 + inline + extra.get(op, 0)
    return ops


def test_reads_name_the_parameters_the_body_uses(pkg):
    ld = pkg.ld
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}, "a": {"type": "real", "dim": [3]}}
    lik, prog, offsets = _lik(pkg, lambda s, d, i: ld.norm(d.y[i], s.a[d.g[i]], 1.0), params, {"y": [1.0, 2.0], "g": [0.0, 2.0]}, 2)
    assert lik.reads == ["a"]
    # the block holds a at entries 5..7: COMP_I's base moves with it, and the body reads the same values from there
    prog2 = lik.lower({"a": 5})
    assert prog2.code != prog.code


def test_lowering_reads_the_entries_the_block_holds(pkg, orc):
    """the body lowered for a block laid out as [sigma, junk, a[0..2], mu] reads what the component layout reads"""
    ld, O = pkg.ld, orc.lib()
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}, "a": {"type": "real", "dim": [3]}}
    d = {"y": [1.0, 2.5, -0.5, 0.75], "g": [0.0, 2.0, 1.0, 2.0]}
    f = lambda s, dd, i: ld.norm(dd.y[i], s.a[dd.g[i]] + s.mu, s.sigma)
    lik, prog, offsets = _lik(pkg, f, params, d, 4)
    assert lik.reads == ["mu", "sigma", "a"]
    comps = [0.3, 1.4, -0.2, 0.9, 0.05]                           # mu, sigma, a[0..2]
    block = [1.4, 99.0, -0.2, 0.9, 0.05, 0.3]                    # sigma, an unread entry, a[0..2], mu
    got = _eval_points(lik, lik.lower({"sigma": 0, "a": 2, "mu": 5}), O, block, 4)
    want = _eval_points(lik, prog, O, comps, 4)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    ref = np.array([O.orc_ld_norm(d["y"][i], comps[2 + int(d["g"][i])] + comps[0], comps[1]) for i in range(4)])
    assert np.array_equal(got.view(np.int64), ref.view(np.int64))


# ---- refusals, before the chains move ------------------------------------------------------------------------------------------------
def _model_only(pkg, **extra):
    ld = pkg.ld

    def log_post(state, data):
        lp = ld.norm(state.mu, 0, 100) + ld.unif(state.sigma, 0, 100)
        for i in range(len(data["y"])):
            lp += ld.norm(data["y"][i], state.mu, state.sigma)
        return lp
    opts = {"chains": 8, "_model_only": True}
    opts.update(extra)
    return pkg.mcmc.AmwgSampler({"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}, log_post,
                                {"y": [1.0, 2.0, 3.5, 0.2]}, opts)


def test_refusals_raise_before_the_chains_move(pkg):
    ld, mcmc = pkg.ld, pkg.mcmc
    s = _model_only(pkg)
    good = lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma)
    bad = [
        ("None or a dict", [good, 4]),
        ("unknown", {"log_lik": good, "points": 4, "weights": 1}),
        ("log_lik", {"points": 4}),
        ("points", {"log_lik": good, "points": 0}),
        ("points", {"log_lik": good, "points": 4.0}),
        ("points", {"log_lik": good, "points": True}),
        ("r_eff", {"log_lik": good, "points": 4, "r_eff": 0.0}),
        ("r_eff", {"log_lik": good, "points": 4, "r_eff": float("inf")}),
        ("r_eff", {"log_lik": good, "points": 4, "r_eff": float("nan")}),
        ("branches", {"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma) if st.mu > 0 else 0.0, "points": 4}),
        ("past the end", {"log_lik": good, "points": 5}),
        ("outside its bounds", None),
        ("at least 2 draws", "S1"),
    ]
    for what, spec in bad:
        if spec is None:
            s3 = pkg.mcmc.AmwgSampler({"a": {"type": "real", "dim": [2]}}, lambda st, d: ld.norm(st.a[0], 0, 1) + ld.norm(st.a[1], 0, 1),
                                      {"y": [1.0, 2.0], "g": [0.0, 2.0]}, {"chains": 8, "_model_only": True})
            with pytest.raises(ValueError, match="outside its bounds"):
                s3.sample_summary(4, loo={"log_lik": lambda st, d, i: ld.norm(d.y[i], st.a[d.g[i]], 1.0), "points": 2})
            continue
        if spec == "S1":
            s1 = _model_only(pkg, chains=1)
            with pytest.raises(ValueError, match=what):
                s1.sample_summary(1, loo={"log_lik": good, "points": 4})
            continue
        with pytest.raises(ValueError, match=what):
            s.sample_summary(10, loo=spec)
    def log_post(state, data):
        state.loo = state.mu * 2                                   # a derived quantity named like the result's key
        return ld.norm(state.mu, 0, 100) + ld.norm(data["y"][0], state.mu, 1.0)
    s2 = mcmc.AmwgSampler({"mu": {"type": "real"}}, log_post, {"y": [1.0, 2.0]}, {"chains": 8, "_model_only": True})
    with pytest.raises(ValueError, match="named 'loo'"):
        s2.sample_summary(10, loo={"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, 1.0), "points": 2})
    assert s._handle is None                                       # nothing reached a device
