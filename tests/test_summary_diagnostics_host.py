"""Host side of the split-chain diagnostics (ESS, MCSE, split R-hat) of the on-device summary: the windowed Geyer driver and
the record merging, on CPU tensors with a numpy stand-in for amwg_summary_autocov (tests/ess_ref.py), against an FFT
restatement of the estimator and against known answers of AR(1) chains."""
import os
import socket
import sys

import numpy as np
import pytest

from ess_ref import (NumpyAutocovReducer, ar1, autocov_records, autocov_scale, ess_fft, fft_diagnostics, geyer_tau, halves, rho_fft)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)
KEYS = ("ess_mean", "ess_tail", "mcse_mean", "rhat_split")


def _mixed(rows, chains, seed):
    """[rows, 4, chains]: AR(0.6) draws far from 0, an integer AR entry with many ties, AR(-0.3), and iid draws."""
    x = ar1(0.6, rows, chains, 4, seed)
    x[:, 0] = 184.5 + 0.14 * x[:, 0]
    x[:, 1] = np.round(2 * x[:, 1])
    x[:, 2] = ar1(-0.3, rows, chains, 1, seed + 1)[:, 0]
    x[:, 3] = np.random.default_rng(seed + 2).normal(size=(rows, chains))
    return x


def _run(x, distributed=False, max_lags=None):
    import torch
    from bayes_js_b200 import summary
    red = NumpyAutocovReducer()
    rows, _, chains = x.shape
    if max_lags is None:
        res = summary.summarise_block(red, torch.from_numpy(x), rows, chains, PROBS, distributed, diagnostics=True)
        return res, red
    mean, sd, rhat, q = summary.summarise_block(red, torch.from_numpy(x), rows, chains, PROBS + summary.DIAGNOSTIC_PROBS, distributed)
    q = q[len(PROBS):]
    return summary.split_chain_diagnostics(red, torch.from_numpy(x), rows, sd, q[1], q[2], q[0], q[3], distributed, max_lags), red


def _assert_close(got, want, rtol=1e-10):
    for k in KEYS:
        assert np.allclose(got[k], want[k], rtol=rtol, atol=0, equal_nan=True), (k, got[k], want[k])


@pytest.mark.parametrize("max_lags", [1, 2, 5, 32])
def test_windowed_driver_equals_the_fft_restatement(pkg, max_lags):
    """lag windows of 1, 2, 5 and 32 lags: the Geyer loop crosses window boundaries at every parity"""
    x = _mixed(60, 37, 1)
    (diag, windows), red = _run(x, max_lags=max_lags)
    _assert_close(diag, fft_diagnostics(x))
    assert windows == len(red.windows) and windows >= 1
    assert [w[0] for w in red.windows] == [max_lags * i for i in range(windows)]         # consecutive windows, only as needed
    assert all(n == max_lags for _, n in red.windows[:-1])
    if max_lags == 1:
        assert windows > 4                                    # AR(0.6) needs several lags


def test_autocorrelations_match_the_fft_restatement(pkg):
    from bayes_js_b200.summary import GeyerESS
    x = _mixed(41, 23, 2)
    h = 20
    thr = np.quantile(np.moveaxis(x, 1, 0).reshape(4, -1), [0.05, 0.95], axis=1).T
    rec = autocov_records(x, thr, 0, h)
    for e in range(4):
        series = [x[:, e], (x[:, e] <= thr[e, 0]).astype(float), (x[:, e] <= thr[e, 1]).astype(float)]
        for s, ys in enumerate(series):
            g = GeyerESS(rec[e, s], h)
            want, varplus, W = rho_fft(halves(ys))
            assert np.allclose(g._rho(rec[e, s, 4:]), want, rtol=0, atol=1e-12), (e, s)
            sc2 = autocov_scale(*thr[e]) ** 2 if s == 0 else 1.0      # the draws series is recorded scaled by a power of two
            assert np.isclose(g.varplus, varplus * sc2, rtol=1e-12) and np.isclose(g.W, W * sc2, rtol=1e-12)


@pytest.mark.parametrize("rows,chains", [(10, 30), (11, 30), (12, 1), (33, 1), (57, 19), (100, 64)])
def test_odd_and_even_rows_single_and_ragged_chains(pkg, rows, chains):
    x = _mixed(rows, chains, rows + chains)
    (mean, sd, rhat, q, (diag, _)), _ = _run(x)
    want = fft_diagnostics(x)
    _assert_close(diag, want)
    assert np.all(np.isfinite(diag["ess_mean"])) and np.all(diag["ess_mean"] > 0)


@pytest.mark.parametrize("rows", [1, 2, 5, 9])
def test_fewer_than_ten_rows_give_nan(pkg, rows):
    x = _mixed(rows, 8, 3)
    (_, _, _, _, (diag, windows)), red = _run(x)
    assert windows == 0 and not red.windows
    for k in KEYS:
        assert np.all(np.isnan(diag[k]))


def test_diagnostics_leave_the_summary_bit_identical(pkg):
    import torch
    from bayes_js_b200.summary import summarise_block
    from summary_ref import NumpyBlockReducer
    x = _mixed(30, 21, 4)
    plain = summarise_block(NumpyBlockReducer(), torch.from_numpy(x), 30, 21, PROBS, False)
    (res, _) = _run(x)
    for a, b in zip(plain, res[:4]):
        assert np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def test_constant_ties_and_infinite_entries(pkg):
    rows, chains = 24, 15
    x = _mixed(rows, chains, 5)
    x[:, 0] = 7.25                                            # constant: ESS = M h, MCSE = 0
    x[:, 1] = np.clip(x[:, 1], -1, 1)                          # integers with ties at both thresholds
    x[3, 2, 4] = np.inf                                       # non-finite draws: all four NaN
    x[5, 3, 0] = -np.inf
    (_, sd, _, q, (diag, _)), _ = _run(x)
    want = fft_diagnostics(x)
    _assert_close(diag, want)
    Mh = 2 * chains * (rows // 2)
    assert diag["ess_mean"][0] == Mh and diag["ess_tail"][0] == Mh and diag["mcse_mean"][0] == 0
    flat = x[:, 1].ravel()
    lo, hi = np.quantile(flat, [0.05, 0.95])
    assert lo == -1 and hi == 1 and np.any(flat == lo) and np.any(flat == hi)           # ties sit on both thresholds
    # 1[x <= q95] = 1[x <= max] is all ones (ESS M h), so the tail ESS is the lower indicator's
    assert np.isclose(diag["ess_tail"][1], ess_fft((x[:, 1] <= lo).astype(float)), rtol=1e-10, atol=0)
    assert np.isfinite(diag["ess_mean"][1])
    for k in KEYS:
        assert np.isnan(diag[k][2]) and np.isnan(diag[k][3])


def test_shards_merge_in_rank_order(pkg):
    import torch
    from bayes_js_b200.summary import merge_autocov_records
    x = _mixed(26, 50, 6)
    thr = np.quantile(np.moveaxis(x, 1, 0).reshape(4, -1), [0.05, 0.95], axis=1).T
    cuts = [0, 17, 18, 50]                                  # ragged shards, one of a single chain
    red = NumpyAutocovReducer()
    parts = [red.autocov(torch.from_numpy(np.ascontiguousarray(x[:, :, a:b])), thr, 3, 7) for a, b in zip(cuts, cuts[1:])]
    got = merge_autocov_records(parts)
    want = autocov_records(x, thr, 3, 7)
    assert np.array_equal(got[:, :, 0], want[:, :, 0])
    assert np.allclose(got[:, :, 1:], want[:, :, 1:], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("phi,tau", [(0.9, 19.0), (0.0, 1.0), (-0.5, 1.0 / 3.0)])
def test_fft_restatement_on_known_autocorrelations(pkg, phi, tau):
    """exact autocorrelations phi^t: Geyer's sum gives tau = (1 + phi) / (1 - phi), including negative lag pairs for phi < 0"""
    h = 400
    rho = phi ** np.arange(h)
    assert np.isclose(geyer_tau(rho, 1e6, h), tau, rtol=1e-9)


@pytest.mark.parametrize("phi,rows", [(0.9, 1000), (0.0, 1000), (-0.5, 4000)])
def test_ess_of_ar1_chains_is_near_the_known_answer(pkg, phi, rows):
    """ess_mean / (M h) within 6 % of 1/tau at 2000 chains (tau = 19, 1, 1/3); the windowed driver against the FFT restatement"""
    chains = 2000
    x = ar1(phi, rows, chains, 1, seed=10 + rows)
    (_, _, _, _, (diag, windows)), _ = _run(x)
    h = rows // 2
    tau = (1 + phi) / (1 - phi)
    got = diag["ess_mean"][0] / (2 * chains * h)
    assert abs(got * tau - 1) < 0.06, (phi, got * tau)
    assert np.isclose(diag["ess_mean"][0], fft_diagnostics(x)["ess_mean"][0], rtol=1e-10)
    assert 0.99 < diag["rhat_split"][0] < 1 + 2 * tau / h     # stationary chains: only the finite-h upward bias


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.parallel import shard_bounds
    from bayes_js_b200.summary import summarise_block
    from ess_ref import NumpyAutocovReducer, fft_diagnostics
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows, chains = 40, 37                                 # ragged: 19 + 18 chains
        x = _mixed(rows, chains, 11)
        first, count = shard_bounds(chains, rank, world)
        mine = torch.from_numpy(np.ascontiguousarray(x[:, :, first:first + count]))
        *_, (diag, windows) = summarise_block(NumpyAutocovReducer(), mine, rows, chains, PROBS, True, diagnostics=True)
        want = fft_diagnostics(x)
        ok = all(np.allclose(diag[k], want[k], rtol=1e-10, equal_nan=True) for k in KEYS)
        q.put((rank, bool(ok), b"".join(diag[k].tobytes() for k in KEYS) + bytes([windows])))
    finally:
        dist.destroy_process_group()


def test_diagnostics_over_gloo_world2():
    """every rank sends its shard's records; both ranks end with the single-process numbers, the same bytes on both"""
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert all(ok for _, ok, _ in res)
    assert res[0][2] == res[1][2]
