"""Host side of the rank-normalised diagnostics of the on-device summary (diagnostics="rank": ess_bulk, rhat_rank): the
driver in summary.rank_diagnostics on CPU tensors with a numpy stand-in for the sort / count / z entries (tests/rank_ref.py),
against a scipy restatement of the estimator, on Vehtari et al.'s motivating cases, and over a two-rank gloo ring."""
import os
import socket
import sys

import numpy as np
import pytest

from ess_ref import ar1
from rank_ref import NumpyRankReducer, rank_diagnostics_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBS = (0.025, 0.25, 0.5, 0.75, 0.975)
KEYS = ("ess_bulk", "rhat_rank")
TRUE_KEYS = ("ess_mean", "ess_tail", "mcse_mean", "rhat_split")


def _mixed(rows, chains, seed):
    """[rows, 4, chains]: AR(0.6) draws far from 0, an integer AR entry with big tie groups, AR(-0.3), and iid draws."""
    x = ar1(0.6, rows, chains, 4, seed)
    x[:, 0] = 184.5 + 0.14 * x[:, 0]
    x[:, 1] = np.round(2 * x[:, 1])
    x[:, 2] = ar1(-0.3, rows, chains, 1, seed + 1)[:, 0]
    x[:, 3] = np.random.default_rng(seed + 2).normal(size=(rows, chains))
    return x


def _run(x, distributed=False, diagnostics="rank", total_chains=None):
    import torch
    from bayes_js_b200.summary import summarise_block
    red = NumpyRankReducer()
    rows, _, chains = x.shape
    res = summarise_block(red, torch.from_numpy(np.ascontiguousarray(x)), rows, total_chains or chains, PROBS, distributed, diagnostics)
    return res, red


def _assert_close(got, want, rtol=1e-10):
    for k in KEYS:
        assert np.allclose(got[k], want[k], rtol=rtol, atol=0, equal_nan=True), (k, got[k], want[k])


@pytest.mark.parametrize("rows,chains", [(10, 30), (11, 30), (12, 1), (33, 1), (57, 19), (100, 64)])
def test_odd_and_even_rows_single_and_ragged_chains(pkg, rows, chains):
    x = _mixed(rows, chains, rows + chains)
    (*_, (diag, _)), _ = _run(x)
    _assert_close(diag, rank_diagnostics_ref(x))
    assert np.all(np.isfinite(diag["ess_bulk"])) and np.all(np.isfinite(diag["rhat_rank"]))


@pytest.mark.parametrize("rows", [1, 2, 5, 9])
def test_fewer_than_ten_rows_give_nan(pkg, rows):
    x = _mixed(rows, 8, 3)
    (*_, (diag, _)), red = _run(x)
    assert not red.sorts
    for k in KEYS:
        assert np.all(np.isnan(diag[k]))


def test_rank_keeps_every_other_key_bit_identical(pkg):
    x = _mixed(30, 21, 4)
    x[3, 2, 4] = np.inf
    plain, _ = _run(x, diagnostics=False)
    true, _ = _run(x, diagnostics=True)
    rank, _ = _run(x)
    for a, b in zip(plain, rank[:4]):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    assert set(rank[4][0]) == set(TRUE_KEYS) | set(KEYS) and set(true[4][0]) == set(TRUE_KEYS)
    for k in TRUE_KEYS:
        assert true[4][0][k].tobytes() == rank[4][0][k].tobytes(), k
    assert true[4][1] == rank[4][1]


@pytest.mark.parametrize("bad", [None, 1, 0, "Rank", "bulk", 1.0])
def test_other_diagnostics_values_raise(pkg, bad):
    with pytest.raises(ValueError, match="diagnostics"):
        _run(_mixed(12, 4, 1), diagnostics=bad)


def test_ties_zeros_infinities_nan_and_constants(pkg):
    rows, chains = 24, 15
    x = _mixed(rows, chains, 5)
    x = np.concatenate([x, x[:, :3]], axis=1)                 # 7 entries
    x[:, 0] = 7.25                                            # constant: ess_bulk = M h, rhat_rank NaN
    x[:, 1] = np.clip(x[:, 1], -1, 1)                          # integers: three huge tie groups
    x[3, 2, 4] = np.inf                                       # +-inf are ranked: both finite
    x[5, 2, 0] = -np.inf
    x[7, 3, 1] = np.nan                                       # a NaN draw: both NaN
    rng = np.random.default_rng(9)
    x[:, 4] = rng.choice([-1.0, 1.0], size=(rows, chains))    # median 0, |x - 0| = 1: a constant folded series
    x[:, 5] = rng.choice([-0.0, 0.0, 1.0], size=(rows, chains))  # -0 ties +0
    x[:, 6] = np.where(rng.random((rows, chains)) < 0.6, np.inf, x[:, 6])  # median inf: the folded series is NaN
    (_, _, _, q, (diag, _)), red = _run(x)
    want = rank_diagnostics_ref(x)
    _assert_close(diag, want)
    Mh = 2 * chains * (rows // 2)
    assert diag["ess_bulk"][0] == Mh and np.isnan(diag["rhat_rank"][0])
    assert np.isfinite(diag["ess_bulk"][1]) and np.isfinite(diag["rhat_rank"][1])
    assert np.isfinite(diag["ess_bulk"][2]) and np.isfinite(diag["rhat_rank"][2])
    assert np.isnan(diag["ess_mean"][2])                      # the non-rank ESS cannot handle the infinite draw
    assert np.isnan(diag["ess_bulk"][3]) and np.isnan(diag["rhat_rank"][3])
    assert np.isfinite(diag["rhat_rank"][4])
    assert np.isfinite(diag["rhat_rank"][5])
    assert np.isfinite(diag["ess_bulk"][6]) and np.isnan(diag["rhat_rank"][6])
    assert [np.isnan(c) for e, c, _ in red.sorts if e == 6] == [True]          # no folded sort around an infinite median


def test_constant_folded_series_gives_the_bulk_rhat(pkg):
    """draws +-1 with median 0: every |x - 0| is 1, so only the bulk R-hat counts"""
    import torch
    from bayes_js_b200 import summary
    from rank_ref import _rhat, half_draws, z_scores
    rows, chains = 20, 9
    x = np.random.default_rng(3).choice([-1.0, 1.0], size=(rows, 1, chains))
    red = NumpyRankReducer()
    out = summary.rank_diagnostics(red, torch.from_numpy(x), rows, np.array([0.0]), np.array([-1.0]), np.array([1.0]), False)
    assert out["rhat_rank"][0] == pytest.approx(_rhat(z_scores(half_draws(x[:, 0]))), rel=1e-12)
    assert len(red.sorts) == 2 and np.isnan(red.sorts[0][1]) and red.sorts[1][1] == 0.0


def test_vehtari_scale_and_location_cases(pkg):
    """equal means, sd 1 vs 3: the split R-hat misses it and the folded rank R-hat catches it; shifted chains: both are large"""
    rows, chains = 400, 8
    rng = np.random.default_rng(12)
    scale = rng.normal(size=(rows, 1, chains)) * np.where(np.arange(chains) < chains // 2, 1.0, 3.0)
    (*_, (diag, _)), _ = _run(scale)
    assert diag["rhat_split"][0] < 1.01 and diag["rhat_rank"][0] > 1.1, (diag["rhat_split"], diag["rhat_rank"])
    _assert_close(diag, rank_diagnostics_ref(scale))
    shift = rng.normal(size=(rows, 1, chains)) + np.where(np.arange(chains) < chains // 2, 0.0, 2.0)
    (*_, (diag, _)), _ = _run(shift)
    assert diag["rhat_split"][0] > 1.1 and diag["rhat_rank"][0] > 1.1
    _assert_close(diag, rank_diagnostics_ref(shift))


def test_heavy_tails_with_an_infinite_draw(pkg):
    """Cauchy draws with one +inf: ess_mean is NaN, ess_bulk is finite and near the iid value"""
    rows, chains = 200, 40
    x = np.random.default_rng(4).standard_cauchy(size=(rows, 1, chains))
    x[17, 0, 3] = np.inf
    (*_, (diag, _)), _ = _run(x)
    assert np.isnan(diag["ess_mean"][0])
    assert np.isfinite(diag["ess_bulk"][0]) and 0.8 < diag["ess_bulk"][0] / (rows * chains) < 1.25
    _assert_close(diag, rank_diagnostics_ref(x))


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
    from rank_ref import NumpyRankReducer
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows, chains = 41, 37                                 # ragged: 19 + 18 chains, odd rows
        x = _mixed(rows, chains, 11)
        x[2, 1, 30] = -np.inf
        first, count = shard_bounds(chains, rank, world)
        mine = torch.from_numpy(np.ascontiguousarray(x[:, :, first:first + count]))
        *_, (diag, _) = summarise_block(NumpyRankReducer(), mine, rows, chains, PROBS, True, diagnostics="rank")
        single = summarise_block(NumpyRankReducer(), torch.from_numpy(x), rows, chains, PROBS, False, diagnostics="rank")[4][0]
        ok = all(np.allclose(diag[k], single[k], rtol=1e-10, atol=0, equal_nan=True) for k in KEYS)
        q.put((rank, bool(ok), b"".join(diag[k].tobytes() for k in KEYS)))
    finally:
        dist.destroy_process_group()


def test_rank_diagnostics_over_gloo_world2():
    """the sorted keys go round the ring; both ranks end with the single-process numbers, the same bytes on both"""
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
