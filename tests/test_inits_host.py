"""Per-chain starting points without a GPU: the dispersal transform of amwg_disperse_state (csrc/amwg_init.cuh compiled for the host)
against its restatement over the oracle (tests/init_ref.py), the host-side shaping of set_state, options.init_radius checks, and the
all-reduced failure decision of a distributed dispersal over a world-2 gloo group."""
import ctypes as C
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import init_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = math.inf


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("inits") / "libinit_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "init_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    lib.hs_disperse_uniform.restype, lib.hs_disperse_uniform.argtypes = C.c_double, [C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int]
    lib.hs_disperse_component.restype = C.c_int
    lib.hs_disperse_component.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_double)]
    lib.hs_disperse_attempts.restype = C.c_int
    return lib


def _bits(x):
    return np.float64(x).view(np.uint64)


# every bound combination, with inits inside, on a bound and outside it
BOUNDS = [(-INF, INF, (0.5, -3.0, 1e6)), (0.0, INF, (0.5, 0.0, -1.0, 7.0)), (-INF, 5.0, (4.5, 5.0, 9.0)), (-2.0, 3.0, (0.5, -2.0, 3.0, 10.0)),
          (0.2, 3.7, (1.0, 0.2)), (-INF, 2.5, (1.0,)), (1.0, INF, (1.0, 2.0))]


def test_dispersal_transform_is_the_restatement_bit_for_bit(H, orc):
    O = orc.lib()
    assert H.hs_disperse_attempts() == init_ref.ATTEMPTS
    out = C.c_double()
    us = [0.0, 1e-17, 0.25, 0.4999999999999999, 0.5, 0.75, 0.9999999999999999]
    for seed, chain in ((7, 0), (12345, 77), (2**40 + 3, 2**32 + 5), (2**64 - 1, 2**35 + 1)):       # chain ids beyond 2^32
        for attempt in (0, 1, 57, 99):
            for n_comp, c in ((1, 0), (3, 2), (300, 299)):
                U = H.hs_disperse_uniform(seed, chain, attempt, n_comp, c)
                assert _bits(U) == _bits(init_ref.uniform(O, seed, chain, attempt, n_comp, c))
                us.append(U)
    n_checked, int_out_of_range = 0, 0
    for U in us:
        for radius in (1e-3, 2.0, 50.0):
            for typ in (init_ref.REAL, init_ref.INT, init_ref.BINARY):
                for lower, upper, inits in BOUNDS:
                    lo, hi = (0.0, 1.0) if typ == init_ref.BINARY else (lower, upper)
                    for init in inits:
                        ok = H.hs_disperse_component(typ, lo, hi, init, radius, U, C.byref(out))
                        want, want_ok = init_ref.component(O, typ, lo, hi, init, radius, U)
                        assert _bits(out.value) == _bits(want) and bool(ok) == want_ok, (typ, lo, hi, init, radius, U)
                        n_checked += 1
                        int_out_of_range += typ == init_ref.INT and not ok
    assert n_checked > 9000
    assert int_out_of_range > 0            # [0.2, 3.7] and (-inf, 2.5] round out of range at some attempts


def test_dispersal_edge_cases(H, orc):
    O = orc.lib()
    out = C.c_double()

    def comp(typ, lo, hi, init, radius, U):
        ok = H.hs_disperse_component(typ, lo, hi, init, radius, U, C.byref(out))
        assert (_bits(out.value), bool(ok)) == (_bits(init_ref.component(O, typ, lo, hi, init, radius, U)[0]),
                                                init_ref.component(O, typ, lo, hi, init, radius, U)[1])
        return out.value, bool(ok)
    # a centre on the bound is replaced by 0: init = lower gives the same value as an init whose centre is 0
    assert comp(0, 0.0, INF, 0.0, 2.0, 0.75) == comp(0, 0.0, INF, 1.0, 2.0, 0.75)             # log(1 - 0) = 0
    assert comp(0, -2.0, 3.0, 3.0, 2.0, 0.25) == comp(0, -2.0, 3.0, 0.5, 2.0, 0.25)            # log(2.5) - log(2.5) = 0
    # U = 0.5 is the centre itself; an unbounded component moves by at most radius
    assert comp(0, -INF, INF, 1.25, 50.0, 0.5)[0] == 1.25
    assert abs(comp(0, -INF, INF, 1.25, 1e-3, 0.9999)[0] - 1.25) <= 1e-3
    # binary: U < 0.5 -> 0, else 1, whatever the bounds, init and radius
    assert comp(2, 0.0, 1.0, 1.0, 2.0, 0.4999) == (0.0, True) and comp(2, 0.0, 1.0, 0.0, 2.0, 0.5) == (1.0, True)
    # int: rounding past a non-integral bound fails; far outside the support the exponential saturates onto the bound
    assert comp(1, 0.2, 3.7, 1.0, 50.0, 0.0)[1] is False                                      # x -> 0.2, round(0.2) = 0 < 0.2
    assert comp(1, -INF, 2.5, 1.0, 50.0, 0.0)[1] is False                                     # x -> 2.5, round(2.5) = 3 > 2.5
    assert comp(1, 1.0, INF, 2.0, 50.0, 0.0) == (1.0, True)                                  # 1 + exp(-50) rounds to 1


# ---- set_state: host-side shaping ------------------------------------------------------------------------------------------------
def _model(pkg, chains, **opts):
    ld = pkg.ld

    def lp(par, data):
        l = 0
        l += ld.norm(par.mu, 0, 10)
        l += ld.unif(par.sigma, 0, 10)
        for i in range(2):
            for j in range(3):
                l += ld.norm(par.b[i][j], 0, 1)
        par.var = par.sigma * par.sigma
        return l
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0, "init": 1}, "b": {"type": "real", "dim": [2, 3]}}
    return pkg.mcmc.AmwgSampler(params, lp, None, dict({"chains": chains, "_model_only": True}, **opts))


def test_set_state_block_broadcast_and_per_chain(pkg):
    Cn = 5
    s = _model(pkg, Cn)
    assert s.n_comp == 8 and s._derived_names == ["var"]
    cur = np.arange(8 * Cn, dtype=np.float64).reshape(8, Cn)
    blk = s._set_state_block({}, cur)
    assert np.array_equal(blk, cur) and blk is not cur
    blk = s._set_state_block({"mu": 3.5}, cur)                               # a number: every chain
    assert np.all(blk[0] == 3.5) and np.array_equal(blk[1:], cur[1:])
    assert np.array_equal(s._set_state_block({"mu": [3.5]}, cur), blk)       # shaped like dim [1]
    sig = np.linspace(1, 2, Cn)
    blk = s._set_state_block({"sigma": sig}, cur)                            # [chains]: per chain
    assert np.array_equal(blk[1], sig) and np.array_equal(np.delete(blk, 1, 0), np.delete(cur, 1, 0))
    one = np.arange(6.0).reshape(2, 3) + 0.25
    blk = s._set_state_block({"b": one.tolist()}, cur)                       # dim [2, 3]: every chain
    assert np.array_equal(blk[2:], np.repeat(one.reshape(6, 1), Cn, axis=1))
    per = np.random.default_rng(0).normal(size=(Cn, 2, 3))
    blk = s._set_state_block({"b": per, "mu": -1.0}, cur)                    # [chains, 2, 3]: per chain, row-major components
    assert np.array_equal(blk[2:], per.reshape(Cn, 6).T) and np.all(blk[0] == -1.0) and np.array_equal(blk[1], cur[1])
    # one chain: the reference's shapes (state of a one-chain sampler) are taken as they are
    s1 = _model(pkg, 1)
    cur1 = np.zeros((8, 1))
    blk = s1._set_state_block({"mu": 2.0, "sigma": [3.0], "b": one}, cur1)
    assert blk[0, 0] == 2.0 and blk[1, 0] == 3.0 and np.array_equal(blk[2:, 0], one.reshape(-1))


def test_set_state_errors(pkg):
    Cn = 4
    s = _model(pkg, Cn)
    cur = np.zeros((8, Cn))
    JsThrow = pkg.mcmc.JsThrow
    cases = [({"var": 1.0}, "set_state: var is a derived quantity, not a parameter"),
             ({"nu": 1.0}, "set_state: nu is not a parameter of this sampler"),
             ({"mu": np.zeros(Cn + 1)}, "set_state: mu is of dimension [5] but should be [1] or [4]"),
             ({"b": np.zeros((2, 2))}, "set_state: b is of dimension [2,2] but should be [2,3] or [4,2,3]"),
             ({"b": np.zeros((Cn, 3, 2))}, "set_state: b is of dimension [4,3,2] but should be [2,3] or [4,2,3]"),
             ({"b": 1.0}, "set_state: b is of dimension [] but should be [2,3] or [4,2,3]"),
             ({"mu": "a"}, "set_state: the value of mu is not numeric")]
    for values, msg in cases:
        with pytest.raises(JsThrow) as e:
            s._set_state_block(values, cur)
        assert str(e.value) == msg, str(e.value)
    with pytest.raises(JsThrow) as e:
        s.set_state([1.0])
    assert str(e.value) == "set_state expects an object keyed by parameter name"


@pytest.mark.parametrize("rank", [0, 1])
def test_set_state_takes_this_ranks_slice_of_uneven_shards(pkg, monkeypatch, rank):
    from bayes_js_b200.parallel import local_chain_rows, shard_bounds
    monkeypatch.setenv("RANK", str(rank))
    monkeypatch.setenv("WORLD_SIZE", "2")
    Cn = 7
    s = _model(pkg, Cn, distributed=True)
    first, count = shard_bounds(Cn, rank, 2)
    assert (s.first_chain, s.local_chains) == (first, count) == ((0, 4) if rank == 0 else (4, 3))
    glob = np.arange(Cn, dtype=np.float64) * 10 + 1
    per = np.random.default_rng(1).normal(size=(Cn, 2, 3))
    blk = s._set_state_block({"sigma": glob, "b": per, "mu": 0.5}, np.zeros((8, count)))
    assert np.array_equal(blk[1], glob[first:first + count])
    assert np.array_equal(blk[2:], per.reshape(Cn, 6)[first:first + count].T) and np.all(blk[0] == 0.5)
    with pytest.raises(pkg.mcmc.JsThrow):                                     # arrays cover the GLOBAL chains
        s._set_state_block({"sigma": glob[:count]}, np.zeros((8, count)))
    with pytest.raises(ValueError):
        local_chain_rows(glob[:5], 4, 3)


def test_init_radius_must_be_finite_and_positive(pkg):
    for bad in (0, -1.0, math.inf, math.nan, "2", True):
        with pytest.raises(pkg.mcmc.JsThrow) as e:
            _model(pkg, 3, init_radius=bad)
        assert str(e.value) == "options.init_radius must be a finite number > 0"
    assert _model(pkg, 3, init_radius=2).init_radius == 2.0 and _model(pkg, 3).init_radius is None
    assert pkg.mcmc.dispersal_failure_message(0, 10) is None
    assert pkg.mcmc.dispersal_failure_message(3, 10) == "options.init_radius: 3 of 10 chains found no starting point with a finite log_post in 100 attempts"


def test_init_radius_checked_by_the_javascript_host(pkg):
    from js_host import JsHost, RecordingNative
    rec = RecordingNative()
    h = JsHost(native=rec)
    h.it.set_global("amwg_trace", h.load("amwg_trace"))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.run('var lp = function (state, data) { var log_post = 0; log_post += ld.norm(state.mu, 0, 1); return log_post; };')
    for bad in ("0", "-1", "Infinity", "NaN", '"2"'):
        with pytest.raises(Exception) as e:
            h.run('new mcmc.AmwgSampler({mu: {type: "real"}}, lp, null, {chains: 2, init_radius: %s});' % bad)
        assert "options.init_radius must be a finite number > 0" in str(e.value)
    assert not rec.created


# ---- the failure decision of a distributed dispersal: every rank raises the same message, or none does ------------------------------
def _worker(rank, world, port, failed, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import __graft_entry__ as graft
    pkg = graft.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, [pkg.mcmc.dispersal_failure_message(f[rank], 11, True, 0) for f in failed]))
    finally:
        dist.destroy_process_group()


def test_dispersal_failure_decision_over_gloo_world2():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    failed = [(0, 0), (0, 3), (2, 0), (1, 4)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, failed, q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=120) for _ in procs)
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    msg = "options.init_radius: %d of 11 chains found no starting point with a finite log_post in 100 attempts"
    want = [None, msg % 3, msg % 2, msg % 5]
    assert res[0] == want and res[1] == want
