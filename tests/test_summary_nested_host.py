"""Host side of the nested R-hat of sample_summary(..., nested=M) and of superchain starting points: csrc/amwg_nested.cuh compiled
for the host with the kernels' grids against the fsum restatement and derived bound of tests/nested_ref.py; the leader rule of
csrc/amwg_init.cuh against the restated dispersal (tests/init_ref.py); the checks of the argument and of
options.superchain_size in the Python and JavaScript hosts; summary.finalize_nested's edge cases; and a gloo world of two uneven
shards whose boundary cuts a superchain."""
import ctypes as C
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import init_ref
import nested_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path_factory, name, src):
    out = tmp_path_factory.mktemp(name) / ("lib%s.so" % name)
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), src, "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(str(out))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    lib = _build(tmp_path_factory, "nested_host", os.path.join(ROOT, "tests", "host_shim", "nested_host.cpp"))
    lib.hs_nested.restype = C.c_longlong
    lib.hs_nested.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_void_p]
    return lib


def host_nested(H, x, first_chain, M):
    x = np.ascontiguousarray(x, dtype=np.float64)
    rows, entries, chains = x.shape
    out = np.empty((entries, 14))
    bad = H.hs_nested(x.ctypes.data, rows, entries, chains, first_chain, M, out.ctypes.data)
    assert bad == 0
    return out


def _draws(rows, entries, chains, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    scale = rng.uniform(0.5, 3.0, size=(1, entries, 1))
    shift = rng.normal(size=(1, 1, chains)) * 0.3                   # chains that disagree a little
    return offset + scale * rng.normal(size=(rows, entries, chains)) + shift


# (M, rows, chains, first_chain): every M, ragged K, cuts at both ends, one superchain cut at both ends, N = 1 and N = 2
CASES = [(1, 1, 37, 0), (1, 2, 37, 5), (2, 1, 38, 0), (2, 2, 41, 3), (7, 2, 70, 0), (7, 9, 71, 4), (7, 1, 5, 15), (64, 2, 640, 0),
         (64, 1, 700, 61), (64, 13, 129, 64), (3, 300, 3 * 1100, 0)]


@pytest.mark.parametrize("M, rows, chains, first", CASES)
@pytest.mark.parametrize("offset", [0.0, 1e6])
def test_nested_header_equals_the_definition_within_the_bound(H, M, rows, chains, first, offset):
    x = _draws(rows, 3, chains, M * 1000 + rows + chains, offset)
    got = host_nested(H, x, first, M)
    exact, bound = nested_ref.check_record(got, x, first, M, (M, rows, chains, first, offset))
    k0, k1 = first // M, (first + chains - 1) // M
    n_cut = (first % M != 0) + ((first + chains) % M != 0 and (k1 > k0 or first % M == 0))
    assert int(np.sum(got[0, [4, 9]] >= 0)) == n_cut
    assert got[0, 0] == (k1 - k0 + 1) - n_cut


@pytest.mark.parametrize("M, rows, chains", [(1, 2, 37), (2, 1, 38), (7, 3, 70), (64, 1, 640), (64, 2, 1024)])
def test_rhat_of_whole_superchains_within_the_bound(H, pkg, M, rows, chains):
    from bayes_js_b200.summary import finalize_nested, merge_nested_records
    x = _draws(rows, 3, chains, 7 * M + rows)
    got = host_nested(H, x, 0, M)
    rh = finalize_nested(merge_nested_records([got], M, rows))
    want = nested_ref.rhat_nested(x, M)
    exact, bound = nested_ref.record(x, 0, M)
    lo, hi = nested_ref.rhat_interval(exact[:, :4], bound[:, :4])
    assert np.all((lo <= rh) & (rh <= hi)), (rh, lo, hi)
    assert np.all((lo <= want) & (want <= hi))


def test_shards_that_cut_superchains_merge_to_one_shard(H, pkg):
    """three uneven host shards, the boundaries inside superchains: the merged record equals one shard's within the bound"""
    from bayes_js_b200.summary import finalize_nested, merge_nested_records
    M, rows, chains = 7, 4, 70
    x = _draws(rows, 2, chains, 11)
    cuts = [0, 10, 12, 70]                                           # [10, 12) lies inside superchain 1
    recs = [host_nested(H, x[:, :, a:b], a, M) for a, b in zip(cuts[:-1], cuts[1:])]
    assert recs[1][0, 4] == 1 and recs[1][0, 9] == -1 and recs[1][0, 0] == 0
    merged = merge_nested_records(recs, M, rows)
    exact, bound = nested_ref.record(x, 0, M)
    # the cut superchain's chain records merge in another order than one shard's: within twice the bound of the exact record
    assert np.all(np.abs(merged - exact[:, :4]) <= 2 * bound[:, :4] + 4 * nested_ref.gamma(8) * np.abs(exact[:, :4]))
    lo, hi = nested_ref.rhat_interval(exact[:, :4], 2 * bound[:, :4] + 4 * nested_ref.gamma(8) * np.abs(exact[:, :4]))
    rh = finalize_nested(merged)
    assert np.all((lo <= rh) & (rh <= hi))
    with pytest.raises(RuntimeError, match="superchain 1 has 2 of its 7 chains"):
        merge_nested_records([recs[1]], M, rows)


def test_finalize_nested_edge_cases(pkg):
    from bayes_js_b200.summary import finalize_nested, merge_nested_records, nested_unit
    inf, nan = math.inf, math.nan
    rec = np.array([[4, 1.0, 3.0, 8.0],           # B^ = 1, W^ = 2: sqrt(1.5)
                    [1, 1.0, 0.0, 2.0],           # K = 1
                    [5, 1.0, 2.0, 0.0],           # W^ = 0 (M = 1 with N = 1, or a constant entry)
                    [5, nan, 2.0, 1.0],
                    [5, inf, 2.0, 1.0],
                    [5, 1.0, inf, 1.0],
                    [5, 1.0, 2.0, -inf],
                    [5, 1.0, 0.0, 3.0]])          # superchains that agree: exactly 1
    got = finalize_nested(rec)
    assert got[0] == math.sqrt(1.5) and got[7] == 1.0
    assert np.all(np.isnan(got[1:7]))
    # M = 1: B~ = 0; N = 1: W- = 0
    sc = np.array([[3.0, 2.0, 4.0, 6.0]])
    assert np.array_equal(nested_unit(sc, 3, 4), [[1.0, 2.0, 0.0, 4.0 / 2 + 6.0 / 9]])
    assert np.array_equal(nested_unit(sc, 1, 4), [[1.0, 2.0, 0.0, 6.0 / 3]])
    assert np.array_equal(nested_unit(sc, 3, 1), [[1.0, 2.0, 0.0, 2.0]])
    assert np.array_equal(nested_unit(sc, 1, 1), [[1.0, 2.0, 0.0, 0.0]])
    # draws through the whole host path: a NaN or +-inf draw, M = 1 with N = 1, a constant entry
    x = _draws(1, 4, 12, 3)
    x[0, 1, 5] = nan
    x[0, 2, 7] = inf
    x[0, 3, :] = 2.5
    for M in (1, 3):
        rec = np.zeros((4, 14))
        rec[:, [4, 9]] = -1
        for e in range(4):
            ch = x[0, e]
            sk = ch.reshape(-1, M).mean(axis=1)
            units = np.stack([np.ones(len(sk)), sk, np.zeros(len(sk)),
                              ch.reshape(-1, M).var(axis=1, ddof=1) if M > 1 else np.zeros(len(sk))], axis=1)
            rec[e, :4] = merge_nested_records([np.concatenate([u[None], np.tile([-1.0, 0, 0, 0, 0], (1, 2))], axis=1) for u in units], M, 1)[0]
        got = finalize_nested(rec[:, :4])
        assert np.all(np.isnan(got[1:])), (M, got)
        assert np.isnan(got[0]) == (M == 1)


def test_resolve_nested_refusals_and_ranges(pkg):
    from bayes_js_b200.summary import resolve_nested
    assert resolve_nested(None, 4, 0, 16) is None and resolve_nested(False, 4, 0, 16) is None
    assert resolve_nested(True, 4, 0, 16) == 4 and resolve_nested(8, None, 0, 16) == 8 and resolve_nested(np.int64(2), None, 4, 6) == 2
    assert resolve_nested(1, None, 3, 5) == 1
    refusals = [((True, None, 0, 16), "nested=True needs options.superchain_size"),
                ((2.0, None, 0, 16), "nested must be None, False, True or an int superchain size >= 1, not 2.0"),
                ((0, None, 0, 16), "nested must be None, False, True or an int superchain size >= 1, not 0"),
                (("4", None, 0, 16), "nested must be None, False, True or an int superchain size >= 1, not '4'"),
                ((5, None, 0, 16), "nested: the chains summarised, [0, 16), are not whole superchains of 5 chains"),
                ((4, None, 2, 16), "nested: the chains summarised, [2, 18), are not whole superchains of 4 chains"),
                ((True, 3, 3, 4), "nested: the chains summarised, [3, 7), are not whole superchains of 3 chains")]
    for args, msg in refusals:
        with pytest.raises(ValueError) as e:
            resolve_nested(*args)
        assert str(e.value) == msg


def _model(pkg, chains, **opts):
    ld = pkg.ld

    def lp(par, data):
        l = 0
        l += ld.norm(par.mu, 0, 10)
        return l
    return pkg.mcmc.AmwgSampler({"mu": {"type": "real"}}, lp, None, dict({"chains": chains, "_model_only": True}, **opts))


SIZE_REFUSALS = [("0", "options.superchain_size must be an integer >= 1"), ("-2", "options.superchain_size must be an integer >= 1"),
                 ("2.5", "options.superchain_size must be an integer >= 1"), ("Infinity", "options.superchain_size must be an integer >= 1"),
                 ("NaN", "options.superchain_size must be an integer >= 1"), ('"4"', "options.superchain_size must be an integer >= 1"),
                 ("true", "options.superchain_size must be an integer >= 1"), ("5", "options.superchain_size must divide options.chains"),
                 ("24", "options.superchain_size must divide options.chains")]


def test_superchain_size_checked_by_the_python_host(pkg):
    py = {"0": 0, "-2": -2, "2.5": 2.5, "Infinity": math.inf, "NaN": math.nan, '"4"': "4", "true": True, "5": 5, "24": 24}
    for js, msg in SIZE_REFUSALS:
        with pytest.raises(pkg.mcmc.JsThrow) as e:
            _model(pkg, 12, superchain_size=py[js])
        assert str(e.value) == msg
    assert _model(pkg, 12, superchain_size=4).superchain_size == 4 and _model(pkg, 12, superchain_size=12.0).superchain_size == 12
    assert _model(pkg, 12).superchain_size is None


def test_superchain_size_checked_by_the_javascript_host(pkg):
    from js_host import JsHost, RecordingNative
    rec = RecordingNative()
    h = JsHost(native=rec)
    h.it.set_global("amwg_trace", h.load("amwg_trace"))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.run('var lp = function (state, data) { var log_post = 0; log_post += ld.norm(state.mu, 0, 1); return log_post; };')
    for bad, msg in SIZE_REFUSALS:
        with pytest.raises(Exception) as e:
            h.run('new mcmc.AmwgSampler({mu: {type: "real"}}, lp, null, {chains: 12, superchain_size: %s});' % bad)
        assert msg in str(e.value)
    assert not rec.created


# ---- the leader rule of csrc/amwg_init.cuh ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L(tmp_path_factory):
    src = tmp_path_factory.mktemp("leader_src") / "leader_host.cpp"
    src.write_text('#include "amwg_init.cuh"\nusing namespace amwg;\nextern "C" {\n'
                   'unsigned long long hs_leader(unsigned long long g, unsigned long long m) { return superchain_leader(g, m); }\n'
                   'double hs_uniform(unsigned long long seed, unsigned long long g, unsigned long long m, int a, int n, int c) {\n'
                   '  return disperse_uniform(seed, superchain_leader(g, m), a, n, c); }\n}\n')
    lib = _build(tmp_path_factory, "leader_host", str(src))
    lib.hs_leader.restype, lib.hs_leader.argtypes = C.c_uint64, [C.c_uint64, C.c_uint64]
    lib.hs_uniform.restype = C.c_double
    lib.hs_uniform.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int]
    return lib


def test_leader_rule_is_todays_dispersal_at_one_and_the_leaders_beyond(L, orc):
    O = orc.lib()
    bits = lambda v: np.float64(v).view(np.uint64)
    for g in (0, 1, 5, 63, 64, 65, 2**32 + 5, 2**40 + 3):
        assert L.hs_leader(g, 1) == g
        for M in (2, 3, 7, 64, 2**20):
            assert L.hs_leader(g, M) == M * (g // M)
    for seed, g in ((7, 0), (12345, 77), (2**40 + 3, 2**32 + 5)):
        for attempt, n_comp, c in ((0, 1, 0), (57, 3, 2), (99, 300, 299)):
            assert bits(L.hs_uniform(seed, g, 1, attempt, n_comp, c)) == bits(init_ref.uniform(O, seed, g, attempt, n_comp, c))
            for M in (2, 7, 64):
                lead = M * (g // M)
                want = bits(init_ref.uniform(O, seed, lead, attempt, n_comp, c))
                assert all(bits(L.hs_uniform(seed, h, M, attempt, n_comp, c)) == want for h in range(lead, lead + M, max(1, M // 5)))
    # every chain of a superchain keeps its leader's point, with the restated dispersal, and superchains differ
    comps = [(init_ref.REAL, -math.inf, math.inf, 0.0), (init_ref.REAL, 0.0, math.inf, 1.0), (init_ref.INT, 0.2, 3.7, 1.0)]
    pts = {}
    for g in range(24):
        pts[g], _ = init_ref.disperse_chain(O, 9, 8 * (g // 8), comps, 2.0, lambda xs: True)
    for g in range(24):
        assert pts[g] == pts[8 * (g // 8)]
    assert pts[0] != pts[8] and pts[8] != pts[16]


# ---- gloo world of two uneven shards whose boundary cuts a superchain -------------------------------------------------------------
class HostNestedReducer:
    """amwg_summary_nested's host build as the reducer of summary.nested_block, on a CPU block."""

    def __init__(self, lib):
        self.lib = lib

    def nested(self, block, first_chain, M):
        return host_nested(self.lib, block.numpy(), first_chain, M)


def _worker(rank, world, port, lib_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.summary import nested_block
    lib = C.CDLL(lib_path)
    lib.hs_nested.restype = C.c_longlong
    lib.hs_nested.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_void_p]
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        M, rows = 8, 5
        x = _draws(rows, 3, 64, 21)
        cut = 36                                                 # uneven shards, 36 + 28 chains: superchain 4 is cut
        mine = x[:, :, :cut] if rank == 0 else x[:, :, cut:]
        first = 0 if rank == 0 else cut
        out = nested_block(HostNestedReducer(lib), torch.from_numpy(np.ascontiguousarray(mine)), rows, first, M, True)
        one = nested_block(HostNestedReducer(lib), torch.from_numpy(x), rows, 0, M, False)
        exact, bound = nested_ref.record(x, 0, M)
        b2 = 2 * bound[:, :4] + 4 * nested_ref.gamma(8) * np.abs(exact[:, :4])
        lo, hi = nested_ref.rhat_interval(exact[:, :4], b2)
        ok = bool(np.all((lo <= out) & (out <= hi)) and np.all((lo <= one) & (one <= hi)))
        q.put((rank, ok, np.ascontiguousarray(out).tobytes()))
    finally:
        dist.destroy_process_group()


def test_nested_over_gloo_world2(H):
    """every rank reduces its shard; one all-gather of the records, the cut superchain merged by id in rank order: both ranks
    return the same bytes, within the bound of one shard holding every chain"""
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, H._name, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert all(ok for _, ok, _ in res)
    assert res[0][2] == res[1][2]
