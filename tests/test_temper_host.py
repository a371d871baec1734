"""Tempered ladders without a GPU (DESIGN.md §2 "Tempered ladders"): option validation in the Python host, ladder-aligned shards,
the device's swap decision (csrc/amwg_temper.cuh compiled with g++) against the reference's, and the reference ladder itself
(tests/temper_ref.py) against the oracle."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import temper_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("temper") / "libtemper_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "temper_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    lib.hs_swap_uniform.restype, lib.hs_swap_uniform.argtypes = C.c_double, [C.c_uint64, C.c_uint64, C.c_uint64]
    lib.hs_swap_accept.restype, lib.hs_swap_accept.argtypes = C.c_int, [C.c_double] * 5
    lib.hs_swap_pairs.restype, lib.hs_swap_pairs.argtypes = C.c_int, [C.c_int, C.c_uint64]
    lib.hs_max_rungs.restype = C.c_int
    return lib


def _model(pkg, chains, **opts):
    ld = pkg.ld

    def lp(par, data):
        l = 0
        l += ld.norm(par.mu, 0, 10)
        l += ld.unif(par.sigma, 0, 10)
        return l
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0, "init": 1}}
    return pkg.mcmc.AmwgSampler(params, lp, None, dict({"chains": chains, "_model_only": True}, **opts))


# ---- options.temperatures ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("temps,msg", [
    ("1,2", "options.temperatures must be a list of numbers"),
    (2.0, "options.temperatures must be a list of numbers"),
    ([1, "2"], "options.temperatures must be a list of numbers"),
    ([1, True], "options.temperatures must be a list of numbers"),
    ([1], "options.temperatures must have between 2 and 256 entries"),
    ([], "options.temperatures must have between 2 and 256 entries"),
    (list(range(1, 258)), "options.temperatures must have between 2 and 256 entries"),
    ([1, math.inf], "options.temperatures must be finite"),
    ([1, math.nan], "options.temperatures must be finite"),
    ([2, 4], "options.temperatures must start at 1"),
    ([1, 1], "options.temperatures must be strictly increasing"),
    ([1, 3, 2, 4], "options.temperatures must be strictly increasing"),
    ([1, 2, 4], "options.temperatures: their number must divide options.chains"),
])
def test_temperatures_refusals(pkg, temps, msg):
    with pytest.raises(pkg.mcmc.JsThrow) as e:
        _model(pkg, 8, temperatures=temps)
    assert str(e.value) == msg


def test_temperatures_accepted_and_betas(pkg, H):
    temps = [1, 1.5, 2.0 ** 0.5 * 3, 7.25]
    s = _model(pkg, 12, temperatures=temps)
    assert s.betas == [1.0 / float(t) for t in temps] and s.temperatures == [float(t) for t in temps]
    assert (s.cold_chains, s.local_cold) == (3, 3)
    s = _model(pkg, 256 * 2, temperatures=list(range(1, 257)))
    assert len(s.betas) == H.hs_max_rungs() == pkg.mcmc.MAX_RUNGS
    s = _model(pkg, 6, temperatures=np.array([1.0, 2.0, 3.0]))
    assert s.cold_chains == 2
    u = _model(pkg, 5)                                 # untempered: every chain is recorded
    assert u.betas is None and (u.cold_chains, u.local_cold) == (5, 5)


def test_temperatures_refused_combinations(pkg):
    with pytest.raises(pkg.mcmc.JsThrow) as e:
        _model(pkg, 8, temperatures=[1, 2], superchain_size=4)
    assert "superchain_size cannot be combined with options.temperatures" in str(e.value)
    with pytest.raises(pkg.mcmc.JsThrow) as e:
        _model(pkg, 8, temperatures=[1, 2], first_chain=3)
    assert str(e.value) == "options.first_chain must be a multiple of the number of temperatures"
    assert _model(pkg, 8, temperatures=[1, 2], first_chain=6).first_chain == 6


@pytest.mark.parametrize("rank", [0, 1])
def test_ladders_do_not_straddle_ranks(pkg, monkeypatch, rank):
    """A world of two ranks: 12 chains in ladders of 3 shard as [0, 6) and [6, 12); 10 chains in ladders of 2 as [0, 5) and [5, 10),
    which splits ladder 2, and 12 chains in ladders of 4 as [0, 6), [6, 12): both refused on every rank."""
    from bayes_js_b200.parallel import ladder_shard_error
    monkeypatch.setenv("RANK", str(rank))
    monkeypatch.setenv("WORLD_SIZE", "2")
    s = _model(pkg, 12, temperatures=[1, 2, 3], distributed=True)
    assert (s.first_chain, s.local_chains, s.cold_chains, s.local_cold) == (6 * rank, 6, 4, 2)
    for chains, temps in ((10, [1, 2]), (12, [1, 2, 3, 4])):
        with pytest.raises(pkg.mcmc.JsThrow) as e:
            _model(pkg, chains, temperatures=temps, distributed=True)
        assert "every GPU must hold whole ladders" in str(e.value)
    assert ladder_shard_error(16, 2, 4) is None and ladder_shard_error(16, 3, 4) is not None
    assert ladder_shard_error(24, 3, 4) is None and ladder_shard_error(7, 1, 7) is None


# ---- the swap decision -----------------------------------------------------------------------------------------------------------
def test_swap_pairs(H):
    for K in range(2, 12):
        for k in range(4):
            assert H.hs_swap_pairs(K, k) == len(range(k & 1, K - 1, 2)), (K, k)


def test_swap_uniform_is_the_reserved_stream_position(H, orc):
    O = orc.lib()
    rng = np.random.default_rng(7)
    for _ in range(200):
        seed, chain, k = (int(v) for v in rng.integers(0, 2 ** 63, 3, dtype=np.uint64))
        k %= 1 << 40
        u = H.hs_swap_uniform(seed, chain, k)
        assert u == O.orc_stream_uniform(seed, chain, temper_ref.SWAP_STREAM_BASE + k) == temper_ref.swap_uniform(O, seed, chain, k)


def _decision_cases():
    rng = np.random.default_rng(11)
    inf, nan = math.inf, math.nan
    cases = []
    for _ in range(4000):
        b = np.sort(rng.uniform(0.001, 1.0, 2))[::-1]
        cases.append((1.0 if rng.random() < 0.3 else float(b[0]), float(b[1]), float(rng.normal(0, 50)), float(rng.normal(0, 50)), float(rng.random())))
    specials = [inf, -inf, nan, 0.0, -0.0, 1e308, -1e308, 5e-324, 700.0, -745.2]
    for la in specials:
        for lb in specials:
            for u in (0.0, 0.5, 1.0 - 2.0 ** -53):
                cases.append((1.0, 0.5, la, lb, u))
    one_ulp_less = float(np.nextafter(1.0, 0.0))
    for k in range(1, 6):                              # beta gaps of a few ulps
        bb = 1.0
        for _ in range(k):
            bb = float(np.nextafter(bb, 0.0))
        for d in (1e300, 1e308, -1e308, 1.0, 1e-300, 7e306):
            for u in (0.0, 0.3, 0.999999):
                cases.append((1.0, bb, 0.0, d, u))
                cases.append((one_ulp_less, bb, d, -d, u))
    for lp in (0.0, 12.5, -3e5, inf, -inf):            # equal log_post
        cases.append((1.0, 0.25, lp, lp, 0.5))
    return cases


def test_swap_decision_matches_the_reference(H, orc):
    O = orc.lib()
    n_acc = 0
    for ba, bb, la, lb, u in _decision_cases():
        ref = temper_ref.swap_accept(O, ba, bb, la, lb, u)
        got = bool(H.hs_swap_accept(ba, bb, la, lb, u))
        assert got == ref, (ba, bb, la, lb, u)
        n_acc += got
    assert n_acc > 100                                 # both outcomes are exercised
    assert not H.hs_swap_accept(1.0, 0.5, math.nan, 0.0, 0.0) and not H.hs_swap_accept(1.0, 0.5, math.inf, math.inf, 0.0)
    assert H.hs_swap_accept(1.0, 0.5, 0.0, 0.0, 0.999)              # equal log_post: the ratio is 1 > u


# ---- the reference ladder ------------------------------------------------------------------------------------------------------
PARAMS_MIX = {"mu": {"type": "real"}, "s": {"type": "real", "lower": 0, "init": 1.5}, "k": {"type": "int", "lower": -20, "upper": 20},
              "v": {"type": "real", "dim": [3]}, "m": {"type": "binary"}}


def _f_mix(O, y):
    def f(x):
        mu, s, k, v, m = x[0], x[1], x[2], x[3:6], x[6]
        lp = O.orc_ld_norm(mu, 0, 5) + O.orc_ld_gamma(s, 2, 1) + O.orc_ld_norm(k, 2, 3) + O.orc_ld_bern(m, 0.3)
        for j in range(3):
            lp += O.orc_ld_norm(v[j], mu, s)
        for yi in y:
            lp += O.orc_ld_norm(yi, mu + 0.5 * m, s)
        x[7] = s * s
        return lp
    return f


def test_reference_chain_at_beta_one_is_the_oracle(orc):
    """beta = 1 without swaps: every chain equals the oracle's chain of the same id -- state, derived slot, draws, info"""
    O = orc.lib()
    y = [0.3, 1.7, -0.4, 2.2]
    f = _f_mix(O, y)
    for g in (0, 5):
        ref = temper_ref.RefChain(orc, f, PARAMS_MIX, 17, g, 1.0, n_derived=1, comp_options={"mu": {"batch_size": 7}})
        o = orc.OracleSampler(f, None, PARAMS_MIX, seed=17, chain=g, n_derived=1, derived_names=["var"], comp_options={"mu": {"batch_size": 7}})
        for _ in range(40):
            ref.step()
            o.step()
            assert np.array_equal(ref.x, o.state())
        assert ref.n.value == o.rng_position()
        inf = o.info()
        real = [c for c in range(7) if c != 6]
        assert np.array_equal(ref.pls[real], inf[real, 0]) and np.array_equal(ref.acc[real], inf[real, 2])


def test_ladder_without_accepted_swaps_is_untempered_on_rung_zero(orc):
    """T_1 huge and log_post differences that make every swap ratio underflow: rung 0 is the untempered oracle chain"""
    O = orc.lib()

    def f(x):                                          # a narrow Normal: hot chains wander far, cold ones stay near 0
        return O.orc_ld_norm(x[0], 0, 0.01) * 1e6
    params = {"x": {"type": "real", "init": 0.0}}
    lad = temper_ref.RefLadder(orc, f, params, 23, [1.0, 1.0 / 1e300], ladders=3)
    for _ in range(60):
        lad.step()
    assert lad.rounds == 60 and lad.accepts.sum() == 0
    for ell in range(3):
        o = orc.OracleSampler(f, None, params, seed=23, chain=2 * ell)
        o.burn(60)
        assert np.array_equal(lad.chains[2 * ell].x, o.state())


def test_accepted_swaps_conserve_the_states(orc):
    """A swap round only permutes states inside ladders: the multiset of (state, log_post) pairs of every ladder is unchanged"""
    O = orc.lib()
    f = _f_mix(O, [0.5, -1.0])
    lad = temper_ref.RefLadder(orc, f, PARAMS_MIX, 31, [1.0, 0.7, 0.4, 0.1], ladders=2, first_chain=8, n_derived=1)
    total = 0
    for _ in range(30):
        for ch in lad.chains:
            ch.step()
        before = [sorted(map(tuple, lad.states()[l * 4:(l + 1) * 4])) for l in range(2)]
        lad.swap_round()
        after = [sorted(map(tuple, lad.states()[l * 4:(l + 1) * 4])) for l in range(2)]
        assert before == after
        total = int(lad.accepts.sum())
    assert total > 5
    assert lad.accepts[:, 0].sum() + lad.accepts[:, 2].sum() > 0 and lad.accepts[:, 1].sum() > 0
