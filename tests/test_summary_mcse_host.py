"""sample_summary(..., mcse=True) without a GPU: the indicator walk of amwg_summary_indicator_autocov (csrc/amwg_indicator.cuh,
built for the host by tests/host_shim/indicator_host.cpp) equal to direct counting at word boundaries, windows and adversarial
values; the exact-integer ESS against the FFT estimator; mcse_block with a numpy stand-in reducer against tests/mcse_ref.py,
in one process and in a gloo world of two uneven shards; chain-permutation and power-of-two invariances, the edge cases, the
refusals, and RadixSelect at per-entry ranks."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch

import mcse_ref
from ess_ref import ar1, ess_fft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)


def _build(out_dir):
    import subprocess
    out = os.path.join(str(out_dir), "libindicator_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-fPIC", "-shared", "-ffp-contract=off",
           "-I" + os.path.join(ROOT, "tests", "host_shim"), "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"),
           os.path.join(ROOT, "tests", "host_shim", "indicator_host.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _load(path):
    lib = C.CDLL(path)
    lib.hs_indicator.restype = C.c_int
    lib.hs_indicator.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    return _load(_build(tmp_path_factory.mktemp("indicator")))


def _host(H, x, thr, lag0, n_lags):
    x = np.ascontiguousarray(x, dtype=np.float64)
    rows, entries, chains = x.shape
    t = np.ascontiguousarray(thr, dtype=np.float64).reshape(entries, -1)
    out = np.full((entries, t.shape[1], 2 + 2 * n_lags), -1, dtype=np.int64)
    assert H.hs_indicator(x.ctypes.data, rows, entries, chains, t.ctypes.data, t.shape[1], lag0, n_lags, out.ctypes.data) == 0
    return out


class HostIndicatorReducer(mcse_ref.NumpyMcseReducer):
    """the numpy stand-in, with the indicator sums from the host-compiled kernel text"""

    def __init__(self, H):
        super().__init__()
        self.H = H

    def indicator_autocov(self, block, thresholds, lag0, n_lags):
        got = _host(self.H, block.numpy(), thresholds, lag0, n_lags)
        assert np.array_equal(got, super().indicator_autocov(block, thresholds, lag0, n_lags))
        return got


def _adversarial(rows, chains, seed):
    """[rows, 5, chains]: ties on a half grid, +-0, +-inf among normals, a constant, AR(0.8)"""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, 5, chains))
    x[:, 0] = np.round(2 * rng.normal(size=(rows, chains))) / 2
    x[:, 1] = np.where(rng.uniform(size=(rows, chains)) < 0.5, -0.0, 0.0)
    x[:, 2] = rng.normal(size=(rows, chains))
    x[1, 2, 0], x[rows - 1, 2, chains - 1], x[rows // 2, 2, 1] = np.inf, -np.inf, np.inf
    x[:, 3] = 7.25
    x[:, 4] = ar1(0.8, rows, chains, 1, seed)[:, 0]
    return x


def _thresholds(x, K, rng):
    """K thresholds per entry: the minimum, below it, the maximum, 0.0 and -0.0, then draws themselves (ties)"""
    entries = x.shape[1]
    thr = np.empty((entries, K))
    for e in range(entries):
        v = x[:, e, :].ravel()
        pool = [v.min(), np.nextafter(v.min(), -np.inf), v.max(), 0.0, -0.0]
        pool += list(rng.choice(v, size=max(K - len(pool), 0)))
        thr[e] = pool[:K] if K <= len(pool) else pool
    return thr


@pytest.mark.parametrize("rows", [10, 11, 126, 127, 128, 129, 130, 258, 259, 600])      # h = 5, 63, 64, 65, 129, 300, odd rows
@pytest.mark.parametrize("K", [1, 5, 16])
def test_integer_sums_equal_direct_counting(H, rows, K):
    h = rows // 2
    x = _adversarial(rows, 6, rows + K)
    thr = _thresholds(x, K, np.random.default_rng(rows * K))
    windows = {(0, min(64, h)), (0, 1)}
    for lag0 in (1, 5, 63, 64, 65, h - 64, h - 1):
        if 0 <= lag0 < h:
            windows |= {(lag0, min(64, h - lag0)), (lag0, 1)}
    for lag0, n_lags in sorted(windows):
        got = _host(H, x, thr, lag0, n_lags)
        ref = mcse_ref.indicator_sums(x, thr, lag0, n_lags)
        assert np.array_equal(got, ref), (rows, K, lag0, n_lags, np.argwhere(got != ref)[:4])


def test_windows_agree_with_the_whole_range(H):
    """every lag's counters have the same value whichever window asks for it"""
    rows = 300
    h = rows // 2
    x = _adversarial(rows, 4, 3)
    thr = _thresholds(x, 5, np.random.default_rng(3))
    whole = mcse_ref.indicator_sums(x, thr, 0, h)
    for lag0 in range(0, h, 37):
        n = min(64, h - lag0)
        got = _host(H, x, thr, lag0, n)
        assert np.array_equal(got[:, :, :2], whole[:, :, :2])
        assert np.array_equal(got[:, :, 2:2 + n], whole[:, :, 2 + lag0:2 + lag0 + n])
        assert np.array_equal(got[:, :, 2 + n:], whole[:, :, 2 + h + lag0:2 + h + lag0 + n])


@pytest.mark.parametrize("phi, p", [(0.0, 0.5), (0.6, 0.05), (0.9, 0.5), (0.9, 0.975)])
def test_exact_integer_ess_against_the_fft_estimator(phi, p):
    rows, chains = 200, 16
    x = ar1(phi, rows, chains, 1, 7)
    q = np.quantile(x.ravel(), [p])[:, None]
    got = mcse_ref.ess_quantile(x, q)[0, 0]
    ref = ess_fft((x[:, 0, :] <= q[0, 0]).astype(float))
    assert abs(got - ref) <= 1e-12 * ref, (got, ref)


def _summary(reducer, x, probs, distributed=False, total_chains=None):
    from bayes_js_b200.summary import mcse_block, summarise_block
    rows, _, chains = x.shape
    total = chains if total_chains is None else total_chains
    mean, sd, _rhat, q = summarise_block(reducer, torch.from_numpy(x), rows, total, probs, distributed)
    return mcse_block(reducer, torch.from_numpy(x), rows, total, probs, mean, sd, q, distributed), (mean, sd, q)


def _reference(x, probs, mean, sd, q):
    ess = mcse_ref.ess_quantile(x, q)
    for e in range(x.shape[1]):
        if np.isnan(x[:, e, :]).any():
            ess[:, e] = np.nan
    return ess, mcse_ref.mcse_quantile(x, probs, ess), mcse_ref.mcse_sd(x, mean, sd)


def _mixed(rows, chains, seed):
    """[rows, 6, chains]: AR(0.5) far from 0, integers with ties, a constant, +-inf among normals, a NaN, AR(0.95)"""
    x = ar1(0.5, rows, chains, 6, seed)
    x[:, 0] = 184.5 + 0.14 * x[:, 0]
    x[:, 1] = np.round(2 * x[:, 1])
    x[:, 2] = -3.5
    x[2, 3, 1], x[5, 3, 0] = np.inf, -np.inf
    x[3, 4, 2] = np.nan
    x[:, 5] = ar1(0.95, rows, chains, 1, seed + 1)[:, 0]
    return x


@pytest.mark.parametrize("rows", [10, 41, 140])
def test_mcse_block_equals_the_restatement(H, rows):
    x = _mixed(rows, 9, rows)
    red = HostIndicatorReducer(H)
    got, (mean, sd, q) = _summary(red, x, PROBS)
    ess, mq, msd = _reference(x, PROBS, mean, sd, q)
    assert got["ess_quantile"].tobytes() == ess.tobytes()
    assert got["mcse_quantile"].tobytes() == mq.tobytes()
    np.testing.assert_allclose(got["mcse_sd"], msd, rtol=1e-12, atol=0, equal_nan=True)
    # edge cases: the constant entry, +-inf, NaN
    h, M = rows // 2, 18
    assert np.all(got["ess_quantile"][:, 2] == M * h) and np.all(got["mcse_quantile"][:, 2] == 0) and got["mcse_sd"][2] == 0
    assert np.all(np.isfinite(got["ess_quantile"][:, 3])) and np.isnan(got["mcse_sd"][3])
    assert np.all(np.isnan(got["ess_quantile"][:, 4])) and np.all(np.isnan(got["mcse_quantile"][:, 4])) and np.isnan(got["mcse_sd"][4])
    assert np.all(np.isfinite(got["mcse_sd"][[0, 1, 5]])) and np.all(got["mcse_sd"][[0, 1, 5]] > 0)


def test_windows_asked_only_while_geyer_needs_a_lag(H):
    """AR(0.99) over 2000 rows: Geyer's loop runs past the first 64-lag window, and stops long before h"""
    x = ar1(0.99, 2000, 8, 1, 5)
    red = HostIndicatorReducer(H)
    got, (mean, sd, q) = _summary(red, x, (0.5,))
    ess, mq, _ = _reference(x, (0.5,), mean, sd, q)
    assert got["ess_quantile"].tobytes() == ess.tobytes() and got["mcse_quantile"].tobytes() == mq.tobytes()
    lags = [w for w in red.indicator_windows]
    assert len(lags) >= 2 and lags[0] == (0, 64) and lags[-1][0] + lags[-1][1] < 1000, lags


def test_fewer_than_ten_rows_is_nan(H):
    x = ar1(0.3, 9, 20, 2, 1)
    got, _ = _summary(HostIndicatorReducer(H), x, PROBS)
    assert all(np.all(np.isnan(v)) for v in got.values())


def test_chain_permutation_and_scale_invariance(H):
    x = _mixed(60, 11, 4)[:, [0, 1, 5]]
    base, _ = _summary(HostIndicatorReducer(H), x, PROBS)
    perm = np.random.default_rng(2).permutation(x.shape[2])
    got, _ = _summary(HostIndicatorReducer(H), np.ascontiguousarray(x[:, :, perm]), PROBS)
    assert got["ess_quantile"].tobytes() == base["ess_quantile"].tobytes()
    for j in (-300, -20, 7, 300):
        s = np.ldexp(1.0, j)
        got, _ = _summary(HostIndicatorReducer(H), x * s, PROBS)
        assert got["ess_quantile"].tobytes() == base["ess_quantile"].tobytes(), j
        assert got["mcse_quantile"].tobytes() == (base["mcse_quantile"] * s).tobytes(), j
        assert got["mcse_sd"].tobytes() == (base["mcse_sd"] * s).tobytes(), j


def test_refusals_before_any_work(monkeypatch):
    from bayes_js_b200.summary import check_mcse, check_mcse_size
    for bad in (1, 0, None, "yes", np.bool_(True), 1.0):
        with pytest.raises(ValueError, match="mcse must be True or False"):
            check_mcse(bad)
    check_mcse(True)
    check_mcse(False)
    check_mcse_size(100, 1 << 22)
    h = 1 << 20                                                       # 2 M h^2 = 2^63 exactly with M = 2^22
    with pytest.raises(ValueError, match="2 M h\\^2 >= 2\\^63"):
        check_mcse_size(2 * h, 1 << 21)
    check_mcse_size(2 * h, (1 << 21) - 1)
    monkeypatch.setitem(sys.modules, "scipy.special", None)
    with pytest.raises(ValueError, match="needs scipy"):
        check_mcse_size(100, 64)


def test_sample_summary_refuses_before_the_chains_move(monkeypatch, pkg):
    """mcse is checked before anything touches the device: a refused call leaves no trace (no GPU is needed to see the error)"""
    s = object.__new__(pkg.mcmc.AmwgSampler)
    for bad in (1, None, "rank"):
        with pytest.raises(ValueError, match="mcse must be True or False"):
            pkg.mcmc.AmwgSampler.sample_summary(s, 10, mcse=bad)


def test_radix_select_at_per_entry_ranks():
    from bayes_js_b200.summary import RadixSelect
    from summary_ref import NumpyBlockReducer
    from bayes_js_b200.summary import _select
    rng = np.random.default_rng(9)
    x = np.round(rng.normal(size=(30, 4, 7)) * 3) / 3
    x[:, 3] = -0.0
    x[0, 2, 0] = -np.inf
    blk = torch.from_numpy(x)
    red = NumpyBlockReducer()
    S = 30 * 7
    ranks = np.stack([rng.integers(0, S, size=12) for _ in range(4)])
    got = _select(red, blk, ranks, False).values()
    srt = np.sort(np.moveaxis(x, 1, 0).reshape(4, -1), axis=1)
    assert np.array_equal(got, np.take_along_axis(srt, ranks, axis=1))          # np.sort leaves -0 and +0 in either order
    shared = np.array([0, 5, 100, S - 1])
    a = _select(red, blk, shared, False)
    b = _select(red, blk, np.tile(shared, (4, 1)), False)
    assert a.values().tobytes() == b.values().tobytes() and a.prefix.tobytes() == b.prefix.tobytes()
    assert isinstance(a, RadixSelect)


# ---- a gloo world of two uneven shards ---------------------------------------------------------------------------------------------
def _worker(rank, world, port, lib_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        x = _mixed(40, 13, 8)
        cut = 4
        mine = np.ascontiguousarray(x[:, :, :cut] if rank == 0 else x[:, :, cut:])
        H = _load(lib_path)
        out, _ = _summary(HostIndicatorReducer(H), mine, PROBS, True, 13)
        one, _ = _summary(HostIndicatorReducer(H), x, PROBS)
        ok = out["ess_quantile"].tobytes() == one["ess_quantile"].tobytes()
        ok = ok and out["mcse_quantile"].tobytes() == one["mcse_quantile"].tobytes()
        ok = ok and np.allclose(out["mcse_sd"], one["mcse_sd"], rtol=1e-12, atol=0, equal_nan=True)
        q.put((rank, ok, np.concatenate([out[k].ravel() for k in ("ess_quantile", "mcse_quantile", "mcse_sd")]).tobytes()))
    finally:
        dist.destroy_process_group()


def test_mcse_over_gloo_world2(tmp_path):
    """two uneven shards: every rank returns the same bytes; ess_quantile and mcse_quantile equal one shard's bit for bit"""
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
