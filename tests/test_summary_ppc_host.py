"""Host side of the posterior predictive checks in sample_summary(..., ppc=...): the samplers of csrc/amwg_ppc.cuh compiled for the
host against the independent restatement of tests/ppc_ref.py bit for bit (including the uniforms each draw takes) and against
scipy.stats in distribution; summary.ppc_block with a numpy stand-in for the device reductions against the restatement, in chunks
and over a gloo world of two uneven shards; the tracing of the ld.* call; and every refusal, raised before the chains move."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats as st

import ppc_ref
from summary_ref import ChanBlockReducer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 20261017


def _build(out_dir):
    out = os.path.join(str(out_dir), "libppc_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "ppc_host.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("ppc_host")))
    u64, vp, d = C.c_uint64, C.c_void_p, C.c_double
    lib.hs_ppc_position.restype = u64
    lib.hs_ppc_position.argtypes = [u64, u64, u64]
    lib.hs_ppc_draw.restype = d
    lib.hs_ppc_draw.argtypes = [C.c_int, vp, u64, u64, u64, u64, u64, C.POINTER(u64)]
    lib.hs_ppc_draws.restype = None
    lib.hs_ppc_draws.argtypes = [C.c_int, vp, u64, u64, u64, vp]
    lib.hs_ppc_draw_tape.restype = d
    lib.hs_ppc_draw_tape.argtypes = [C.c_int, vp, vp, u64, C.POINTER(u64)]
    lib.hs_ppc_log_factorial.restype = d
    lib.hs_ppc_log_factorial.argtypes = [d]
    return lib


def _args(p):
    return np.ascontiguousarray(list(p) + [0.0] * (3 - len(p)), dtype=np.float64)


def host_draw(H, fam, p, seed, chain, row, points, i):
    used = C.c_uint64()
    a = _args(p)
    x = H.hs_ppc_draw(ppc_ref.FAMILIES.index(fam), a.ctypes.data, seed, chain, row, points, i, C.byref(used))
    return x, used.value


def host_draws(H, fam, p, n, chain=3):
    out = np.empty(n)
    a = _args(p)
    H.hs_ppc_draws(ppc_ref.FAMILIES.index(fam), a.ctypes.data, SEED, chain, n, out.ctypes.data)
    return out


# (family, parameters) covering every branch: pois below and above 10 up to 1e6, binom by inversion and by BTRS with p on both
# sides of 1/2, gamma shape < 1 and >= 1, t with small and huge df
REGIMES = [("norm", (1.5, 2.0)), ("lnorm", (0.3, 0.5)), ("cauchy", (-1.0, 0.5)), ("laplace", (1.0, 2.0)), ("logis", (0.5, 1.5)),
           ("exp", (2.5,)), ("weibull", (1.5, 2.0)), ("weibull", (0.6, 1.0)), ("pareto", (1.0, 3.0)), ("unif", (-1.0, 2.0)),
           ("gamma", (0.3, 2.0)), ("gamma", (4.5, 1.5)), ("invgamma", (3.0, 2.0)), ("beta", (0.5, 2.0)), ("beta", (3.0, 4.0)),
           ("t", (0.0, 1.0, 3.0)), ("t", (1.0, 2.0, 1e300)), ("bern", (0.3,)), ("pois", (0.0,)), ("pois", (3.2,)), ("pois", (25.0,)),
           ("pois", (1e6,)), ("binom", (20.0, 0.2)), ("binom", (20.0, 0.9)), ("binom", (100.0, 0.3)), ("binom", (100.0, 0.8)),
           ("binom", (7.0, 0.0)), ("binom", (7.0, 1.0)), ("nbinom", (3.0, 0.4)), ("nbinom", (0.7, 0.05)), ("nbinom", (2.0, 1.0))]


def test_samplers_equal_the_restatement_bit_for_bit(H, orc):
    O = orc.lib()
    rng = np.random.default_rng(1)
    for fam, p in REGIMES:
        for _ in range(120):
            g, r, N = int(rng.integers(0, 1 << 22)), int(rng.integers(0, 50)), int(rng.integers(1, 5000))
            i = int(rng.integers(0, N))
            got, used = host_draw(H, fam, p, SEED, g, r, N, i)
            want, wused = ppc_ref.draw_at(O, fam, p, SEED, g, r, N, i)
            assert np.float64(got).tobytes() == np.float64(want).tobytes() and used == wused, (fam, p, g, r, i, got, want, used, wused)


def test_logis_redraws_a_zero_uniform(H, orc):
    tape = np.array([0.0, 0.0, 0.3])
    used = C.c_uint64()
    x = H.hs_ppc_draw_tape(ppc_ref.FAMILIES.index("logis"), _args((1.0, 2.0)).ctypes.data, tape.ctypes.data, 3, C.byref(used))
    s = ppc_ref.Tape(orc.lib(), tape)
    want = ppc_ref.draw("logis", (1.0, 2.0), s)
    assert used.value == 3 == s.used() and np.float64(x).tobytes() == np.float64(want).tobytes() and np.isfinite(x)


def test_log_factorial_table_is_correctly_rounded(H):
    import mpmath
    mpmath.mp.prec = 300
    for k in range(128):
        exact = mpmath.loggamma(k + 1)
        v = H.hs_ppc_log_factorial(float(k))
        assert v == ppc_ref.LOG_FACTORIAL[k]
        for w in (np.nextafter(v, -np.inf), np.nextafter(v, np.inf)):
            assert abs(mpmath.mpf(float(w)) - exact) >= abs(mpmath.mpf(v) - exact)
    for k in (128.0, 1000.0, 1e6, 1e12):                            # Stirling's series: within a few ulp of the exact value
        assert abs(H.hs_ppc_log_factorial(k) - float(mpmath.loggamma(k + 1))) <= 4e-16 * float(mpmath.loggamma(k + 1))


@pytest.mark.parametrize("fam, p", [("norm", (0.0, 0.0)), ("norm", (0.0, -1.0)), ("norm", (np.nan, 1.0)), ("norm", (np.inf, 1.0)),
                                    ("cauchy", (0.0, 0.0)), ("exp", (0.0,)), ("exp", (-1.0,)), ("weibull", (0.0, 1.0)),
                                    ("pareto", (1.0, 0.0)), ("unif", (1.0, 1.0)), ("unif", (2.0, 1.0)), ("gamma", (0.0, 1.0)),
                                    ("gamma", (1.0, -1.0)), ("invgamma", (-1.0, 1.0)), ("beta", (0.0, 1.0)), ("t", (0.0, 1.0, 0.0)),
                                    ("t", (0.0, 1.0, np.inf)), ("bern", (1.5,)), ("bern", (-0.1,)), ("pois", (-1.0,)),
                                    ("pois", (np.inf,)), ("binom", (2.5, 0.5)), ("binom", (-1.0, 0.5)), ("binom", (5.0, 1.1)),
                                    ("nbinom", (0.0, 0.5)), ("nbinom", (2.0, 0.0)), ("lnorm", (0.0, 0.0)), ("laplace", (0.0, -2.0)),
                                    ("logis", (0.0, 0.0))])
def test_out_of_domain_gives_nan_and_takes_no_uniform(H, orc, fam, p):
    x, used = host_draw(H, fam, p, SEED, 5, 0, 10, 3)
    assert np.isnan(x) and used == 0
    assert np.isnan(ppc_ref.draw_at(orc.lib(), fam, p, SEED, 5, 0, 10, 3)[0])


def test_stream_positions(H):
    # below the dispersal region (2^63) for every row x points < 2^46, and 2^16 uniforms apart
    assert H.hs_ppc_position(0, 1, 0) == 1 << 62
    last = H.hs_ppc_position((1 << 46) // 1024 - 1, 1024, 1023)
    assert last + (1 << 16) <= 1 << 63
    seen = set()
    for r in range(6):
        for i in range(7):
            pos = H.hs_ppc_position(r, 7, i)
            assert pos == ppc_ref.position(r, 7, i) and pos not in seen
            seen.add(pos)
    ps = sorted(seen)
    assert all(b - a == 1 << 16 for a, b in zip(ps, ps[1:]))


def _continuous(fam, p):
    a = p
    make = {"norm": lambda: st.norm(a[0], a[1]), "lnorm": lambda: st.lognorm(a[1], scale=np.exp(a[0])),
            "cauchy": lambda: st.cauchy(a[0], a[1]), "laplace": lambda: st.laplace(a[0], a[1]), "logis": lambda: st.logistic(a[0], a[1]),
            "exp": lambda: st.expon(scale=1 / a[0]), "weibull": lambda: st.weibull_min(a[0], scale=a[1]),
            "pareto": lambda: st.pareto(a[1], scale=a[0]), "unif": lambda: st.uniform(a[0], a[1] - a[0]),
            "gamma": lambda: st.gamma(a[0], scale=1 / a[1]), "invgamma": lambda: st.invgamma(a[0], scale=a[1]),
            "beta": lambda: st.beta(a[0], a[1]), "t": lambda: st.t(min(a[2], 1e10), a[0], a[1])}
    return make[fam]() if fam in make else None


def _discrete(fam, p):
    return {"bern": lambda: st.bernoulli(p[0]), "pois": lambda: st.poisson(p[0]), "binom": lambda: st.binom(int(p[0]), p[1]),
            "nbinom": lambda: st.nbinom(p[0], p[1])}[fam]()


def chi_square_p(x, dist):
    """chi-square of the counts against the pmf, cells with expected count < 5 pooled into the tails"""
    lo, hi = int(dist.ppf(1e-7)), int(dist.ppf(1 - 1e-7)) + 1
    ks = np.arange(lo, hi + 1)
    exp = dist.pmf(ks) * len(x)
    obs = np.array([np.sum(x == k) for k in ks], dtype=float)
    exp[0] += dist.cdf(lo - 1) * len(x)
    obs[0] += np.sum(x < lo)
    exp[-1] += dist.sf(hi) * len(x)
    obs[-1] += np.sum(x > hi)
    cells_o, cells_e, ao, ae = [], [], 0.0, 0.0
    for o, e in zip(obs, exp):
        ao, ae = ao + o, ae + e
        if ae >= 5:
            cells_o.append(ao)
            cells_e.append(ae)
            ao = ae = 0.0
    if ae > 0 and cells_e:
        cells_o[-1] += ao
        cells_e[-1] += ae
    cells_o, cells_e = np.array(cells_o), np.array(cells_e)
    if len(cells_o) < 2:
        return 1.0 if np.all(x == x[0]) else 0.0
    return st.chisquare(cells_o, cells_e * cells_o.sum() / cells_e.sum()).pvalue


def distribution_p(x, fam, p):
    if fam == "binom" and p[1] in (0.0, 1.0):
        return 1.0 if np.all(x == p[0] * p[1]) else 0.0
    if fam == "nbinom" and p[1] == 1.0:
        return 1.0 if np.all(x == 0) else 0.0
    if fam == "pois" and p[0] == 0.0:
        return 1.0 if np.all(x == 0) else 0.0
    d = _continuous(fam, p)
    if d is not None:
        return st.kstest(x, d.cdf).pvalue
    return chi_square_p(x, _discrete(fam, p))


@pytest.mark.parametrize("fam, p", REGIMES)
def test_host_draws_follow_the_distribution(H, fam, p):
    x = host_draws(H, fam, p, 100000)
    assert np.all(np.isfinite(x))
    assert distribution_p(x, fam, p) > 1e-3, (fam, p)


# ---- ppc_block with numpy stand-ins -------------------------------------------------------------------------------------------
class StandInReducer(ChanBlockReducer):
    def threshold_counts(self, block, thresholds):
        x = block.numpy()
        out = np.zeros((x.shape[1], 4), dtype=np.int64)
        for e in range(x.shape[1]):
            out[e] = ppc_ref.counts(x[:, e, :].ravel(), thresholds[e])
        return torch.from_numpy(out)


class ArraySource:
    """y_rep [rows, N, chains] in chunks, with the statistics records formed chunk by chunk as the device carries them"""

    def __init__(self, yrep3):
        self.y = np.ascontiguousarray(yrep3, dtype=np.float64)
        self.taken = 0

    def chunk(self, p0, P):
        assert p0 == self.taken
        self.taken += P
        return torch.from_numpy(np.ascontiguousarray(self.y[:, p0:p0 + P, :]))

    def stats(self):
        assert self.taken == self.y.shape[1]
        rows, N, chains = self.y.shape
        T = np.empty((rows, 4, chains))
        for r in range(rows):
            for c in range(chains):
                T[r, :, c] = ppc_ref.dataset_stats(self.y[r, :, c])
        return torch.from_numpy(T)


def _flat(y3):
    rows, N, chains = y3.shape
    return np.moveaxis(y3, 1, 2).reshape(rows * chains, N)


PROBS = (0.05, 0.5, 0.95)


def run_ppc(y3, y, chunk=None, family="norm"):
    from bayes_js_b200.summary import ppc_block
    rows, N, chains = y3.shape
    return ppc_block(StandInReducer(), ArraySource(y3), rows, chains, N, family, y, PROBS, chunk or N, False)


def assert_ppc_matches(out, ref):
    from bayes_js_b200.summary import finalize_moments
    assert out["points"] == ref["points"] and out["n_draws"] == ref["n_draws"] and out["family"] == ref["family"]
    for key in ("n_below", "n_equal", "n_nan"):
        assert np.array_equal(out["pointwise"][key], ref["pointwise"][key]), key
        assert out["pointwise"][key].dtype == np.int64
    assert np.array_equal(out["pointwise"]["pit"], ref["pointwise"]["pit"])
    for key in ("mean", "sd"):
        assert np.allclose(out["pointwise"][key], ref["pointwise"][key], rtol=1e-12, atol=1e-12, equal_nan=True), key
    for name in ppc_ref.STATS:
        got, want = out["stats"][name], ref["stats"][name]
        assert got["observed"] == want["observed"] or (np.isnan(got["observed"]) and np.isnan(want["observed"])), name
        for key in ("n_greater", "n_equal", "n_nan", "p_value"):
            assert got[key] == want[key], (name, key, got[key], want[key])
        for key in ("mean", "sd"):
            assert np.isclose(got[key], want[key], rtol=1e-12, atol=1e-12, equal_nan=True), (name, key)
        assert np.allclose(got["quantiles"], want["quantiles"], rtol=1e-12, atol=1e-12, equal_nan=True), name


def test_ppc_block_equals_the_restatement():
    rng = np.random.default_rng(2)
    y3 = rng.normal(1.0, 2.0, size=(3, 17, 40))
    y = rng.normal(1.0, 2.0, 17)
    y3[0, 4, :5] = y[4]                                          # ties with the observation
    out = run_ppc(y3, y)
    assert_ppc_matches(out, ppc_ref.ppc(_flat(y3), y, PROBS))


def test_ppc_block_pointwise_moments_are_the_base_summary():
    from bayes_js_b200.summary import summarise_block
    rng = np.random.default_rng(3)
    y3 = rng.gamma(2.0, 1.5, size=(2, 9, 33))
    out = run_ppc(y3, rng.gamma(2.0, 1.5, 9))
    mean, sd, _, _ = summarise_block(StandInReducer(), torch.from_numpy(y3), 2, 33, PROBS, False)
    assert np.array_equal(out["pointwise"]["mean"], mean) and np.array_equal(out["pointwise"]["sd"], sd)


def test_discrete_counts_and_nan_draws():
    rng = np.random.default_rng(4)
    y3 = rng.poisson(3.0, size=(2, 11, 25)).astype(float)
    y3[1, 3, 7] = np.nan                                         # a NaN draw: counted in n_nan, its dataset's min / max / mean NaN
    y = rng.poisson(3.0, 11).astype(float)
    out = run_ppc(y3, y, family="pois")
    ref = ppc_ref.ppc(_flat(y3), y, PROBS, family="pois")
    assert_ppc_matches(out, ref)
    assert out["pointwise"]["n_nan"][3] == 1 and out["stats"]["max"]["n_nan"] == 1
    assert out["pointwise"]["n_below"].sum() + out["pointwise"]["n_equal"].sum() > 0


def test_forced_small_chunks_give_the_same_bits():
    rng = np.random.default_rng(5)
    y3 = rng.standard_t(3, size=(3, 13, 21))
    y = rng.standard_t(3, 13)
    one, some = run_ppc(y3, y), run_ppc(y3, y, chunk=4)
    for key in one["pointwise"]:
        assert np.array_equal(one["pointwise"][key], some["pointwise"][key]), key
    for name in one["stats"]:
        for key, v in one["stats"][name].items():
            assert np.array_equal(np.asarray(v), np.asarray(some["stats"][name][key])), (name, key)


def test_dataset_stats_of_numpy_data():
    from bayes_js_b200.summary import dataset_stats
    rng = np.random.default_rng(6)
    for n in (1, 2, 5, 1000):
        y = rng.normal(50.0, 3.0, n)
        m, sd, mn, mx = dataset_stats(y)
        assert abs(m - np.mean(y)) <= 1e-12 * abs(np.mean(y))
        assert (np.isnan(sd) if n == 1 else abs(sd - np.std(y, ddof=1)) <= 1e-12 * np.std(y, ddof=1))
        assert mn == np.min(y) and mx == np.max(y)
        assert np.array_equal(np.array([m, sd, mn, mx]), np.array(ppc_ref.dataset_stats(y)), equal_nan=True)
    y = np.array([1.0, np.nan, 3.0])
    assert np.all(np.isnan(dataset_stats(y)))


# ---- a gloo world of two uneven shards ---------------------------------------------------------------------------------------------
def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.summary import ppc_block
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(7)
        y3 = rng.normal(0.0, 1.5, size=(3, 10, 90))
        y = rng.normal(0.0, 1.5, 10)
        cut = 31
        mine = y3[:, :, :cut] if rank == 0 else y3[:, :, cut:]
        out = ppc_block(StandInReducer(), ArraySource(mine), 3, 90, 10, "norm", y, PROBS, 4, True)
        one = ppc_block(StandInReducer(), ArraySource(y3), 3, 90, 10, "norm", y, PROBS, 4, False)
        ok = all(np.array_equal(out["pointwise"][k], one["pointwise"][k]) for k in ("n_below", "n_equal", "n_nan", "pit"))
        ok = ok and all(np.allclose(out["pointwise"][k], one["pointwise"][k], rtol=1e-12) for k in ("mean", "sd"))
        for name in one["stats"]:
            ok = ok and all(out["stats"][name][k] == one["stats"][name][k] for k in ("n_greater", "n_equal", "n_nan", "p_value", "observed"))
            ok = ok and np.allclose(out["stats"][name]["quantiles"], one["stats"][name]["quantiles"], rtol=1e-12)
        blob = np.concatenate([np.asarray(out["pointwise"][k], dtype=np.float64) for k in sorted(out["pointwise"])]).tobytes()
        q.put((rank, ok, blob))
    finally:
        dist.destroy_process_group()


def test_ppc_over_gloo_world2():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=180) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert all(ok for _, ok, _ in res)
    assert res[0][2] == res[1][2]


# ---- tracing -------------------------------------------------------------------------------------------------------------------------
def _lik(pkg, f, params, data, points):
    from bayes_js_b200.mcmc import complete_params
    from bayes_js_b200.tracer import trace_log_lik
    params = complete_params({k: dict(v) for k, v in params.items()}, pkg.mcmc.param_init_fixed)
    offsets, n = {}, 0
    for name, p in params.items():
        offsets[name] = n
        n += int(np.prod(p["dim"]))
    return trace_log_lik(f, params, offsets, data, points, what="ppc")


def test_tracing_finds_the_family_the_observations_and_the_parameters(pkg):
    ld, Math = pkg.ld, pkg.mcmc.Math
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}, "a": {"type": "real", "dim": [3]},
              "beta": {"type": "real", "dim": [2]}}
    d = {"y": [1.0, 2.5, -0.5, 0.75], "g": [0.0, 2.0, 1.0, 2.0], "c": [3.0, 0.0, 5.0, 1.0], "x": [0.1, 0.2, 0.3, 0.4]}
    lik = _lik(pkg, lambda s, dd, i: ld.norm(dd.y[i], s.a[dd.g[i]], s.sigma), params, d, 4)
    fam, y, args = lik.observed_call(4)
    assert fam == "norm" and np.array_equal(y, d["y"]) and len(args) == 2 and args[0].op == "COMP_I"
    prog, offs = lik.lower_exprs(args, {"sigma": 0, "a": 1})
    assert len(offs) == 2 and offs[0] == 0 and prog.code[offs[1] - 1] & 0xff == pkg._ffi.OP["END"]
    lik = _lik(pkg, lambda s, dd, i: ld.pois(dd.c[i], Math.exp(s.beta[0] + s.beta[1] * dd.x[i])), params, d, 4)
    fam, y, args = lik.observed_call(4)
    assert fam == "pois" and np.array_equal(y, d["c"]) and lik.reads == ["beta"]
    lik = _lik(pkg, lambda s, dd, i: ld.norm(dd[i], s.mu, s.sigma), params, [4.0, 5.0, 6.0], 3)
    fam, y, _ = lik.observed_call(2)
    assert fam == "norm" and np.array_equal(y, [4.0, 5.0])


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
    ld, mcmc, Math = pkg.ld, pkg.mcmc, pkg.mcmc.Math
    s = _model_only(pkg)
    good = lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma)
    bad = [
        ("None or a dict", [good, 4]),
        ("unknown", {"log_lik": good, "points": 4, "r_eff": 1.0}),
        ("log_lik", {"points": 4}),
        ("points", {"log_lik": good, "points": 0}),
        ("points", {"log_lik": good, "points": 4.0}),
        ("points", {"log_lik": good, "points": True}),
        ("one ld", {"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma) + 0.0, "points": 4}),
        ("one ld", {"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma) * 2, "points": 4}),
        ("data value", {"log_lik": lambda st, d, i: ld.norm(st.mu, 0.0, st.sigma), "points": 4}),
        ("data value", {"log_lik": lambda st, d, i: ld.norm(d.y[3], st.mu, st.sigma), "points": 4}),
        ("data value", {"log_lik": lambda st, d, i: ld.lnorm(Math.log(d.y[i]), st.mu, st.sigma), "points": 4}),
        ("no sampler", {"log_lik": lambda st, d, i: ld.hyper(d.y[i], 5, 5, 3), "points": 4}),
        ("one ld", {"log_lik": lambda st, d, i: ld.cat(d.y[i], [0.5, 0.5]), "points": 4}),
        ("branches", {"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, st.sigma) if st.mu > 0 else 0.0, "points": 4}),
        ("past the end", {"log_lik": good, "points": 5}),
    ]
    for what, spec in bad:
        with pytest.raises(ValueError, match=what):
            s.sample_summary(10, ppc=spec)
    with pytest.raises(ValueError, match="2\\^46"):
        s.sample_summary(1 << 44, ppc={"log_lik": good, "points": 4})

    def log_post(state, data):
        state.ppc = state.mu * 2                                   # a derived quantity named like the result's key
        return ld.norm(state.mu, 0, 100) + ld.norm(data["y"][0], state.mu, 1.0)
    s2 = mcmc.AmwgSampler({"mu": {"type": "real"}}, log_post, {"y": [1.0, 2.0]}, {"chains": 8, "_model_only": True})
    with pytest.raises(ValueError, match="named 'ppc'"):
        s2.sample_summary(10, ppc={"log_lik": lambda st, d, i: ld.norm(d.y[i], st.mu, 1.0), "points": 2})
    assert s._handle is None                                       # nothing reached a device
