"""Host side of LOO-PIT in sample_summary(..., ppc={..., "loo_pit": ...}): summary.ppc_block with a numpy stand-in for the device
reductions (whose Pareto fit, smoothing and run-mean step are csrc/amwg_loo.cuh compiled for the host) against the numpy
restatement of tests/loo_pit_ref.py, on continuous and count families, NaN replicated data, a non-finite point, a tail of at most
four draws, the log(DBL_MIN) floor, forced chunks and r_eff != 1; the tie rule, independent of the order of the draws; a
parameter-free likelihood, where LOO-PIT is the in-sample PIT bit for bit; a gloo world of two uneven shards; and every refusal,
raised before the chains move."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import loo_pit_ref
import loo_ref
import test_summary_loo_host as loo_host
import test_summary_ppc_host as ppc_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-12
PROBS = (0.05, 0.5, 0.95)


def _build(out_dir):
    out = os.path.join(str(out_dir), "libloo_pit_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "loo_pit_host.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _load(path):
    lib = C.CDLL(path)
    vp = C.c_void_p
    lib.hs_pit_fit.restype = None
    lib.hs_pit_fit.argtypes = [vp, C.c_int, vp]
    lib.hs_pit_smoothed.restype = None
    lib.hs_pit_smoothed.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, vp]
    lib.hs_pit_runs.restype = None
    lib.hs_pit_runs.argtypes = [vp, vp, vp, C.c_int, vp]
    return lib


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    return _load(_build(tmp_path_factory.mktemp("loo_pit_host")))


@pytest.fixture(scope="module")
def HL(tmp_path_factory):
    """the PSIS-LOO host library of test_summary_loo_host, for loo_block's stand-in"""
    return loo_host._load(loo_host._build(tmp_path_factory.mktemp("loo_host")))


class StandInReducer(ppc_host.StandInReducer):
    """The device reductions of ppc_block with LOO-PIT on CPU tensors: the threshold counts of the ppc stand-in, the finite range of
    the PSIS-LOO stand-in, the sums-and-tail pass in numpy, and the fit kernel's steps with the fit, smoothing and run-mean step of
    the host-compiled amwg_loo.cuh. `shuffle` (a numpy Generator) puts the gathered tail in a random order before the sort, so
    tied ll reach the sort in any order, as the device's atomic slots deliver them."""

    def __init__(self, H, shuffle=None):
        self.H, self.shuffle = H, shuffle

    finite_range = loo_host.StandInReducer.finite_range

    def loo_pit_reduce(self, ll, yrep, llmin, cut, y, cap):
        x, yr = ll.numpy(), yrep.numpy()
        rows, P, chains = x.shape
        sums = np.empty((P, 3))
        tails = np.zeros((P, cap))
        flags = np.zeros((P, cap), dtype=np.uint8)
        counts = np.zeros(P, dtype=np.int32)
        with np.errstate(invalid="ignore", over="ignore"):
            for p in range(P):
                v, r = x[:, p, :].T.ravel(), yr[:, p, :].T.ravel()
                lw = llmin[p] - v
                t = lw > cut[p]
                w = np.exp(lw[~t])
                sums[p] = (np.sum(w), np.sum(w[r[~t] <= y[p]]), np.sum(w[r[~t] == y[p]]))
                counts[p] = t.sum()
                f = (r[t] <= y[p]).astype(np.uint8) | ((r[t] == y[p]).astype(np.uint8) << 1)
                tails[p, :min(t.sum(), cap)] = v[t][:cap]
                flags[p, :min(t.sum(), cap)] = f[:cap]
        return sums, torch.from_numpy(tails), torch.from_numpy(flags), torch.from_numpy(counts)

    def loo_pit_fit(self, tails, flags, counts, llmin, cut, skip):
        R, P, cap = tails.shape
        out = np.empty((P, 5))
        t, fl, c = tails.numpy(), flags.numpy(), counts.numpy()
        for p in range(P):
            a = np.concatenate([t[r, p, :min(c[r, p], cap)] for r in range(R)])
            f = np.concatenate([fl[r, p, :min(c[r, p], cap)] for r in range(R)])
            if self.shuffle is not None:
                perm = self.shuffle.permutation(len(a))
                a, f = a[perm], f[perm]
            order = np.argsort(-a, kind="stable")
            a, f = np.ascontiguousarray(a[order]), np.ascontiguousarray(f[order])
            n = len(a)
            if skip[p]:
                out[p] = (np.nan, np.nan, np.nan, np.nan, n)
                continue
            k, lw = np.inf, llmin[p] - a
            if n > 4:
                expcut = np.exp(cut[p])
                x = np.ascontiguousarray(np.exp(llmin[p] - a) - expcut)
                ks = np.empty(2)
                self.H.hs_pit_fit(x.ctypes.data, n, ks.ctypes.data)
                k, sigma = ks
                if np.isfinite(k):
                    lw = np.empty(n)
                    self.H.hs_pit_smoothed(n, k, sigma, expcut, lw.ctypes.data)
            w = np.ascontiguousarray(np.exp(lw))
            runs = np.zeros(2)
            self.H.hs_pit_runs(a.ctypes.data, w.ctypes.data, f.ctypes.data, n, runs.ctypes.data)
            out[p] = (k, np.sum(w), runs[0], runs[1], n)
        return out


class ArraySource:
    def __init__(self, x3):
        self.x3 = np.ascontiguousarray(x3, dtype=np.float64)           # [rows, points, chains]

    def chunk(self, p0, P):
        return torch.from_numpy(np.ascontiguousarray(self.x3[:, p0:p0 + P, :]))


def _flat(x3):
    rows, N, chains = x3.shape
    return np.moveaxis(x3, 1, 2).reshape(rows * chains, N)


def run_pit(H, ll3, yrep3, y, r_eff=1.0, chunk=None, family="norm", shuffle=None):
    from bayes_js_b200.summary import ppc_block
    rows, N, chains = ll3.shape
    red = StandInReducer(H, shuffle)
    return ppc_block(red, ppc_host.ArraySource(yrep3), rows, chains, N, family, y, PROBS, chunk or N, False,
                     loo_pit=(ArraySource(ll3), r_eff))


def assert_pit_matches(out, ref):
    got = out["loo_pit"]
    for key in ("pit", "pit_equal"):
        g, w = got[key], ref[key]
        assert np.array_equal(np.isnan(g), np.isnan(w)), key
        ok = ~np.isnan(w)
        assert np.all(np.abs(g[ok] - w[ok]) <= TOL), (key, np.max(np.abs(g[ok] - w[ok])))
    g, w = got["pareto_k"], ref["pareto_k"]
    assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(np.isinf(g), np.isinf(w))
    fin = np.isfinite(w)
    assert np.all(np.abs(g[fin] - w[fin]) <= TOL * np.maximum(1.0, np.abs(w[fin]))), (g, w)
    assert got["pareto_k_threshold"] == ref["pareto_k_threshold"] and got["n_high_k"] == ref["n_high_k"]


def assert_k_is_loos(HL, out, ll3, r_eff):
    """pareto_k has the bits of loo_block's (the PSIS-LOO stand-in) over the same ll"""
    from bayes_js_b200.summary import loo_block
    rows, N, chains = ll3.shape
    loo = loo_block(loo_host.StandInReducer(HL), loo_host.ArraySource(ll3), rows, chains, N, r_eff, N, False)
    assert out["loo_pit"]["pareto_k"].tobytes() == loo["pointwise"]["pareto_k"].tobytes()


# ---- the cases: (ll3, yrep3, y) [rows, points, chains] ------------------------------------------------------------------------------
def _sticky(rng, rows, chains, draw):
    """draws [rows, chains] of a chain that repeats its state with probability 1/2 (a rejected step): ties in ll"""
    out = np.empty((rows, chains))
    out[0] = draw(chains)
    for r in range(1, rows):
        keep = rng.uniform(size=chains) < 0.5
        out[r] = np.where(keep, out[r - 1], draw(chains))
    return out


def case_normal(rows=4, chains=300, N=12, seed=1):
    rng = np.random.default_rng(seed)
    y = rng.normal(1.0, 2.0, N)
    mu = rng.normal(y.mean(), 2.0 / np.sqrt(N), (rows, 1, chains))
    sd = 2.0 * np.sqrt(rng.chisquare(N - 1, (rows, 1, chains)) / (N - 1))
    ll3 = -0.5 * np.log(2 * np.pi) - np.log(sd) - (y[None, :, None] - mu) ** 2 / (2 * sd * sd)
    yrep3 = rng.normal(mu, sd, (rows, N, chains))
    return ll3, yrep3, y


def case_pois(rows=6, chains=200, N=9, seed=2):
    rng = np.random.default_rng(seed)
    y = rng.poisson(3.0, N).astype(float)
    lam = _sticky(rng, rows, chains, lambda n: rng.gamma(y.sum() + 1, 1.0 / N, n))[:, None, :]
    from scipy.special import gammaln
    ll3 = y[None, :, None] * np.log(lam) - lam - gammaln(y[None, :, None] + 1)
    yrep3 = rng.poisson(np.broadcast_to(lam, (rows, N, chains))).astype(float)
    return ll3, yrep3, y


def case_bern(rows=5, chains=240, N=10, seed=3):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 2, N).astype(float)
    p = _sticky(rng, rows, chains, lambda n: rng.beta(y.sum() + 1, N - y.sum() + 1, n))[:, None, :]
    ll3 = np.where(y[None, :, None] == 1, np.log(p), np.log1p(-p))
    yrep3 = (rng.uniform(size=(rows, N, chains)) < p).astype(float)
    return ll3, yrep3, y


def test_continuous_family(H, HL):
    ll3, yrep3, y = case_normal()
    out = run_pit(H, ll3, yrep3, y)
    assert_pit_matches(out, loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y))
    assert np.all(out["loo_pit"]["pit_equal"] == 0) and np.all(np.isfinite(out["loo_pit"]["pareto_k"]))
    assert_k_is_loos(HL, out, ll3, 1.0)
    assert out["loo_pit"]["r_eff"] == 1.0


@pytest.mark.parametrize("case, family", [(case_pois, "pois"), (case_bern, "bern")])
def test_count_families_with_many_equal_replicates(H, HL, case, family):
    ll3, yrep3, y = case()
    out = run_pit(H, ll3, yrep3, y, family=family)
    ref = loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y)
    assert_pit_matches(out, ref)
    assert np.all(out["loo_pit"]["pit_equal"] > 0.02)                  # y_rep == y is common
    assert np.all(out["loo_pit"]["pit"] >= out["loo_pit"]["pit_equal"])
    assert_k_is_loos(HL, out, ll3, 1.0)


def test_nan_replicates_count_in_the_normaliser_only(H):
    ll3, yrep3, y = case_normal(seed=4)
    yrep3[:, 3, :] = np.nan                                          # every draw of point 3
    yrep3[1, 5, ::7] = np.nan
    out = run_pit(H, ll3, yrep3, y)
    assert_pit_matches(out, loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y))
    assert out["loo_pit"]["pit"][3] == 0 and out["loo_pit"]["pit_equal"][3] == 0


def test_non_finite_point(H):
    ll3, yrep3, y = case_normal(seed=5)
    ll3[:, 2, :] = np.nan
    ll3[0, 6, 11] = -np.inf
    out = run_pit(H, ll3, yrep3, y)
    assert_pit_matches(out, loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y))
    for key in ("pit", "pit_equal", "pareto_k"):
        assert np.isnan(out["loo_pit"][key][2]) and np.isnan(out["loo_pit"][key][6]) and not np.isnan(out["loo_pit"][key][0]), key


def test_tail_of_at_most_four_draws(H):
    ll3, yrep3, y = case_normal(rows=1, chains=20, N=5, seed=6)          # S = 20: M = 4, raw weights
    out = run_pit(H, ll3, yrep3, y)
    assert_pit_matches(out, loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y))
    assert np.all(np.isinf(out["loo_pit"]["pareto_k"]))


def test_log_dbl_min_floor(H):
    rng = np.random.default_rng(7)
    S, N = 1000, 3
    ll = rng.normal(0.0, 1.0, size=(S, N))
    ll[:50] -= 1000.0                                              # 50 draws far below: the cut is log(DBL_MIN)
    yrep = rng.normal(0.0, 1.0, size=(S, N))
    y = np.array([0.1, -0.4, 1.2])
    ll3, yrep3 = (a.reshape(1, S, N).transpose(0, 2, 1).copy() for a in (ll, yrep))
    assert all(loo_ref.psis_point(ll[:, i])["cut"] == loo_ref.LOG_TINY for i in range(N))
    out = run_pit(H, ll3, yrep3, y)
    assert_pit_matches(out, loo_pit_ref.loo_pit(ll, yrep, y))


def test_forced_chunks_give_the_same_bits(H):
    ll3, yrep3, y = case_pois(N=15, seed=8)
    outs = [run_pit(H, ll3, yrep3, y, chunk=c, family="pois") for c in (15, 1, 7)]
    assert_pit_matches(outs[0], loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y))
    for other in outs[1:]:
        for key in ("pit", "pit_equal", "pareto_k"):
            assert outs[0]["loo_pit"][key].tobytes() == other["loo_pit"][key].tobytes(), key


def test_r_eff_moves_the_tail(H, HL):
    ll3, yrep3, y = case_normal(rows=2, chains=400, N=6, seed=9)
    out = run_pit(H, ll3, yrep3, y, r_eff=0.3)
    ref = loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y, r_eff=0.3)
    assert_pit_matches(out, ref)
    assert out["loo_pit"]["r_eff"] == 0.3
    assert not np.array_equal(ref["pit"], loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y)["pit"])
    assert_k_is_loos(HL, out, ll3, 0.3)


def test_other_keys_keep_their_bits(H):
    ll3, yrep3, y = case_bern(seed=10)
    from bayes_js_b200.summary import ppc_block
    rows, N, chains = ll3.shape
    plain = ppc_block(StandInReducer(H), ppc_host.ArraySource(yrep3), rows, chains, N, "bern", y, PROBS, 4, False)
    with_pit = run_pit(H, ll3, yrep3, y, chunk=4, family="bern")
    assert set(with_pit) == set(plain) | {"loo_pit"}
    for key in plain:
        assert _same(plain[key], with_pit[key]), key


def _same(x, y):
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    a, b = np.asarray(x), np.asarray(y)
    if a.dtype.kind in "fiub":
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


# ---- the tie rule -----------------------------------------------------------------------------------------------------------------
def _tied_tail(seed=11):
    """S = 1000 draws (M = 95) of one point: a run of 10 tied ll inside the Pareto tail (the 21st..30th smallest), the first five
    of them (by draw index) with y_rep <= y and the last five above; every other draw has y_rep > y"""
    rng = np.random.default_rng(seed)
    S = 1000
    ll = np.sort(rng.normal(0.0, 1.0, S))
    ll[20:30] = ll[25]
    yrep = np.full(S, 2.0)
    yrep[20:25] = -1.0
    return ll, yrep, 0.0


def test_tie_rule_is_independent_of_the_order_of_the_draws(H):
    ll, yrep, y = _tied_tail()
    S = len(ll)
    r = loo_ref.psis_point(ll)
    run = np.flatnonzero(ll == ll[20])
    assert len(run) == 10 and np.all(np.isin(run, r["tail"])) and np.isfinite(r["k"])
    want = loo_pit_ref.point(ll, yrep, y)
    index_order = loo_pit_ref.point(ll, yrep, y, tie_mean=False)
    assert abs(want[0] - index_order[0]) > 1e6 * TOL, (want, index_order)     # the rule is not the index-ordered tie-break
    rng = np.random.default_rng(12)
    results = []
    for k in range(12):
        perm = np.arange(S) if k == 0 else (np.arange(S)[::-1] if k == 1 else rng.permutation(S))
        for rows in (1, 4):
            ll3, yrep3 = ll[perm].reshape(rows, 1, S // rows), yrep[perm].reshape(rows, 1, S // rows)
            out = run_pit(H, ll3, yrep3, np.array([y]), shuffle=np.random.default_rng(100 + k))
            got = out["loo_pit"]["pit"][0]
            assert abs(got - want[0]) <= TOL, (k, rows, got, want)
            results.append(got)
            ref_perm = loo_pit_ref.point(ll[perm], yrep[perm], y)
            assert abs(ref_perm[0] - want[0]) <= TOL
    assert max(results) - min(results) <= TOL
    # the index-ordered tie-break moves with the order of the draws: no reference could match it
    flipped = loo_pit_ref.point(ll[::-1], yrep[::-1], y, tie_mean=False)
    assert abs(flipped[0] - index_order[0]) > 1e6 * TOL


def test_run_mean_step_of_the_header(H):
    """hs_pit_runs (amwg_loo.cuh's run_mean_tail_seq over run_mean_sums) against the definition on a tail with runs of 1..7"""
    rng = np.random.default_rng(13)
    vals = np.sort(rng.normal(0, 1, 12))[::-1]
    lens = rng.integers(1, 8, 12)
    a = np.repeat(vals, lens)
    n = len(a)
    w = np.ascontiguousarray(rng.uniform(0.1, 1.0, n))
    f = np.ascontiguousarray(rng.integers(0, 4, n).astype(np.uint8) & np.uint8(3))
    f[(f & 2) > 0] |= 1                                                # == implies <=
    out = np.zeros(2)
    H.hs_pit_runs(np.ascontiguousarray(a).ctypes.data, w.ctypes.data, f.ctypes.data, n, out.ctypes.data)
    le = eq = 0.0
    start = 0
    for L in lens:
        m = w[start:start + L].sum() / L
        le += m * np.sum(f[start:start + L] & 1)
        eq += m * np.sum((f[start:start + L] >> 1) & 1)
        start += L
    assert abs(out[0] - le) <= 1e-13 and abs(out[1] - eq) <= 1e-13


# ---- a parameter-free likelihood: every weight 1, no tail --------------------------------------------------------------------------
def test_parameter_free_likelihood_gives_the_in_sample_pit(H):
    rng = np.random.default_rng(14)
    rows, N, chains = 3, 8, 50
    y = rng.normal(0, 1, N)
    ll3 = np.broadcast_to((-0.5 * np.log(2 * np.pi) - y * y / 2)[None, :, None], (rows, N, chains)).copy()
    yrep3 = rng.normal(0, 1, (rows, N, chains))
    yrep3[0, 2, :9] = y[2]
    out = run_pit(H, ll3, yrep3, y)
    assert out["loo_pit"]["pit"].tobytes() == out["pointwise"]["pit"].tobytes()
    assert np.all(np.isinf(out["loo_pit"]["pareto_k"]))
    assert out["loo_pit"]["pit_equal"][2] == 9 / (rows * chains)


# ---- a gloo world of two uneven shards ---------------------------------------------------------------------------------------------
def _worker(rank, world, port, lib_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.summary import ppc_block
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ll3, yrep3, y = case_pois(rows=3, chains=200, N=9, seed=15)
        ll3[0, 6, 150] = 4.0                                         # one heavy point, its tail drawn from the second shard
        cut = 77
        mine = (lambda a: a[:, :, :cut]) if rank == 0 else (lambda a: a[:, :, cut:])
        H = _load(lib_path)
        out = ppc_block(StandInReducer(H), ppc_host.ArraySource(mine(yrep3)), 3, 200, 9, "pois", y, PROBS, 4, True,
                        loo_pit=(ArraySource(mine(ll3)), 1.0))["loo_pit"]
        one = ppc_block(StandInReducer(H), ppc_host.ArraySource(yrep3), 3, 200, 9, "pois", y, PROBS, 4, False,
                        loo_pit=(ArraySource(ll3), 1.0))["loo_pit"]
        ok = all(np.allclose(out[k], one[k], rtol=0, atol=TOL, equal_nan=True) for k in ("pit", "pit_equal"))
        ok = ok and out["pareto_k"].tobytes() == one["pareto_k"].tobytes() and out["n_high_k"] == one["n_high_k"]
        q.put((rank, ok, np.concatenate([out[k] for k in ("pit", "pit_equal", "pareto_k")]).tobytes()))
    finally:
        dist.destroy_process_group()


def test_loo_pit_over_gloo_world2(tmp_path):
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


# ---- refusals, before the chains move ------------------------------------------------------------------------------------------------
def test_refusals_raise_before_the_chains_move(pkg):
    from bayes_js_b200.summary import resolve_ppc
    ld = pkg.ld
    s = ppc_host._model_only(pkg)
    good = lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma)
    bad = [
        ("loo_pit must be True", None),
        ("loo_pit must be True", False),
        ("loo_pit must be True", 1),
        ("loo_pit must be True", "yes"),
        ("loo_pit must be True", {}),
        ("loo_pit must be True", {"r_eff": 1.0, "k": 2}),
        ("loo_pit must be True", {"reff": 1.0}),
        ("loo_pit r_eff", {"r_eff": 0.0}),
        ("loo_pit r_eff", {"r_eff": -1.0}),
        ("loo_pit r_eff", {"r_eff": float("inf")}),
        ("loo_pit r_eff", {"r_eff": float("nan")}),
        ("loo_pit r_eff", {"r_eff": True}),
        ("loo_pit r_eff", {"r_eff": "1"}),
    ]
    for what, pit in bad:
        with pytest.raises(ValueError, match=what):
            s.sample_summary(10, ppc={"log_lik": good, "points": 4, "loo_pit": pit})
    with pytest.raises(ValueError, match="unknown"):
        s.sample_summary(10, ppc={"log_lik": good, "points": 4, "loo_pit": True, "r_eff": 1.0})
    s1 = ppc_host._model_only(pkg, chains=1)
    with pytest.raises(ValueError, match="at least 2 draws"):
        s1.sample_summary(1, ppc={"log_lik": good, "points": 4, "loo_pit": True})
    with pytest.raises(ValueError, match="exceeds"):
        s.sample_summary(1 << 20, ppc={"log_lik": good, "points": 4, "loo_pit": {"r_eff": 1e-6}})     # M = 0.2 S > 2^20
    assert s._handle is None and s1._handle is None                # nothing reached a device
    assert resolve_ppc({"log_lik": good, "points": 4, "loo_pit": True}, []).loo_pit == 1.0
    assert resolve_ppc({"log_lik": good, "points": 4, "loo_pit": {"r_eff": 2}}, []).loo_pit == 2.0
    assert resolve_ppc({"log_lik": good, "points": 4}, []).loo_pit is None
