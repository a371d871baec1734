"""Host side of the on-device posterior summaries (SURVEY 8(f).3): exact radix-select bookkeeping, moment merging and the
collectives, on CPU tensors with a numpy stand-in for the two device reductions (tests/summary_ref.py)."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBS = (0.0, 0.025, 0.25, 0.5, 0.75, 0.975, 1.0)


def _block(rows, entries, chains, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, (rows, entries, chains))
    x[:, 0] = 184.5 + 0.14 * x[:, 0]                       # a config-2-like mu: narrow and far from 0
    if entries > 1:
        x[:, 1] = np.round(x[:, 1] * 3)                     # an integer parameter: many ties, both signs, -0/+0
    if entries > 2:
        x[:, 2] = np.exp(5 * x[:, 2]) * np.sign(rng.normal(size=(rows, chains)))     # 20 orders of magnitude, both signs
    return x


def test_ordered_key_is_monotone_and_invertible(pkg):
    from bayes_js_b200.summary import double_to_key, key_to_double
    x = np.array([-np.inf, -1e300, -2.5, -1e-310, -0.0, 0.0, 5e-324, 1.0, 184.5, 1e300, np.inf])
    k = double_to_key(x)
    assert np.all(k[1:] > k[:-1])
    assert np.array_equal(key_to_double(k).view(np.uint64), x.view(np.uint64))


@pytest.mark.parametrize("rows,entries,chains", [(7, 3, 41), (1, 2, 64), (40, 1, 3), (2, 3, 1)])
def test_summary_of_one_shard_matches_numpy(pkg, rows, entries, chains):
    import torch
    from bayes_js_b200.summary import summarise_block
    from summary_ref import NumpyBlockReducer, numpy_summary
    x = _block(rows, entries, chains, rows * 100 + chains)
    mean, sd, rhat, q = summarise_block(NumpyBlockReducer(), torch.from_numpy(x), rows, chains, PROBS, False)
    m0, s0, r0, q0 = numpy_summary(x, PROBS)
    assert np.allclose(mean, m0, rtol=1e-13, atol=0)
    if rows * chains > 1:
        assert np.allclose(sd, s0, rtol=1e-11, atol=0)
    assert np.allclose(rhat, r0, rtol=1e-9, atol=0, equal_nan=True)
    assert np.array_equal(q, q0)                            # exact order statistics, numpy's interpolation rule


def test_long_probability_grids_run_as_several_selects(pkg):
    """more than 16 probabilities (an equal-mass histogram): split into selects of at most 32 order statistics each"""
    import torch
    from bayes_js_b200.summary import summarise_block
    from summary_ref import NumpyBlockReducer, numpy_summary
    x = _block(11, 2, 97, 8)
    probs = tuple(np.linspace(0, 1, 41))
    _, _, _, q = summarise_block(NumpyBlockReducer(), torch.from_numpy(x), 11, 97, probs, False)
    assert q.shape == (41, 2) and np.array_equal(q, numpy_summary(x, probs)[3])


def test_shards_merge_exactly(pkg):
    import torch
    from bayes_js_b200.summary import RadixSelect, finalize_moments, merge_moment_records, quantile_targets
    from summary_ref import NumpyBlockReducer, numpy_summary
    rows, entries, chains = 9, 3, 50
    x = _block(rows, entries, chains, 5)
    cuts = [0, 17, 18, 50]                                  # ragged shards, one of a single chain
    red = NumpyBlockReducer()
    shards = [torch.from_numpy(np.ascontiguousarray(x[:, :, a:b])) for a, b in zip(cuts, cuts[1:])]
    rec = merge_moment_records([red.moments(s) for s in shards])
    mean, sd, rhat = finalize_moments(rec, rows)
    m0, s0, r0, q0 = numpy_summary(x, PROBS)
    assert np.allclose(mean, m0, rtol=1e-13) and np.allclose(sd, s0, rtol=1e-11) and np.allclose(rhat, r0, rtol=1e-9)
    ranks, plan = quantile_targets(rows * chains, PROBS)
    sel = RadixSelect(entries, ranks)
    for p in range(8):
        table, which = sel.prefixes()
        sel.advance(sum(red.digit_counts(s, p, table).numpy() for s in shards), which)
    vals = sel.values()
    flat = np.sort(np.moveaxis(x, 1, 0).reshape(entries, -1), axis=1)
    assert np.array_equal(vals.view(np.uint64), flat[:, ranks].view(np.uint64))


def test_quantile_targets_and_limits(pkg):
    from bayes_js_b200.summary import MAX_PREFIXES, RadixSelect, quantile_targets
    ranks, plan = quantile_targets(11, [0.0, 0.5, 1.0, 0.33])
    assert list(ranks) == [0, 1, 3, 4, 5, 6, 10]
    assert plan[1] == (4, 5, 0.0) and plan[2][0] == 6 and plan[2][1] == 6
    with pytest.raises(ValueError):
        quantile_targets(10, [1.5])
    sel = RadixSelect(1, np.arange(MAX_PREFIXES + 1))
    sel.prefix[0] = np.arange(MAX_PREFIXES + 1, dtype=np.uint64)
    with pytest.raises(ValueError):
        sel.prefixes()


def _by_class(got, want, rtol=1e-13):
    """NaN where numpy has NaN, the same infinities, and the finite values within rtol"""
    got, want = np.asarray(got), np.asarray(want)
    fin = np.isfinite(want)
    return (np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[np.isinf(want)], want[np.isinf(want)])
            and np.all(np.isfinite(got[fin])) and np.allclose(got[fin], want[fin], rtol=rtol, atol=0))


def _nonfinite_block(rows, chains, seed):
    """[rows, 8, chains]: one entry per row of the table in summary.nonfinite_as_numpy, and two finite ones"""
    x = _block(rows, 3, chains, seed)[:, [0, 1, 2, 0, 0, 0, 0, 0]].copy()
    x[:, 7] = 1.5e308                                       # finite draws whose sum overflows: the mean is not finite
    x[0, 3, 0] = np.nan                                     # a NaN
    x[-1, 4, -1] = np.uint64(0xFFF8000000000001).view(np.float64)     # a NaN with the sign bit set, and a +inf
    x[0, 4, 0] = np.inf
    x[0, 5, 0], x[-1, 5, -1] = np.inf, -np.inf             # +inf and -inf
    x[0, 6, :] = np.inf                                     # +inf only, in every chain
    x[-1, 1, -1] = -np.inf                                  # -inf only, in one chain of the integer entry
    return x


@pytest.mark.parametrize("rows,chains", [(5, 9), (1, 4), (3, 1), (7, 41)])
def test_nonfinite_draws_are_summarised_as_numpy(pkg, rows, chains):
    """NaN and +-inf draws: mean, sd, rhat and the quantiles equal numpy's (non-finite values by class), with the device's Chan
    merge (ChanBlockReducer, whose merged mean of +inf and finite chains is NaN) as with numpy's mean; every entry without a
    non-finite draw keeps its bits, including one whose sum overflows (the Chan merge makes its mean NaN, numpy.mean +inf)"""
    import torch
    from bayes_js_b200.summary import finalize_moments, summarise_block
    from summary_ref import ChanBlockReducer, NumpyBlockReducer, numpy_summary
    x = _nonfinite_block(rows, chains, rows + chains)
    probs = PROBS + (0.1, 0.9)
    m0, s0, r0, q0 = numpy_summary(x, probs)
    for red in (ChanBlockReducer(), NumpyBlockReducer()):
        with np.errstate(invalid="ignore", over="ignore"):
            mean, sd, rhat, q = summarise_block(red, torch.from_numpy(x), rows, chains, probs, False)
            raw = red.moments(torch.from_numpy(x))
        assert _by_class(mean[:7], m0[:7]), (type(red).__name__, mean, m0)
        assert np.array_equal(q, q0, equal_nan=True)
        assert np.isnan(q[:, 3]).all() and np.isnan(q[:, 4]).all()          # a NaN draw: NaN at every probability
        assert mean[5] != mean[5] and mean[6] == np.inf and mean[1] == -np.inf
        assert np.isnan(sd[[1, 3, 4, 5, 6]]).all() and np.isnan(rhat[[1, 3, 4, 5, 6]]).all()
        fin = [0, 2]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            want = finalize_moments(raw, rows)
        assert mean[fin].tobytes() == raw[fin, 1].tobytes() and sd.tobytes() == want[1].tobytes() and rhat.tobytes() == want[2].tobytes()
        assert mean[7:].tobytes() == raw[7:, 1].tobytes()                  # no non-finite draw: the merged mean as it is
        if rows * chains > 1:
            assert np.allclose(sd[fin], s0[fin], rtol=1e-11)
    # the stand-in shows the defect this corrects: its merged mean of an entry with +inf draws alone is NaN
    assert np.isnan(ChanBlockReducer().moments(torch.from_numpy(np.array([[[0.5, np.inf, 1.5, 2.0]]])))[0, 1])


def test_the_extremes_are_selected_only_when_a_mean_is_not_finite(pkg):
    """finite means: the one select of the quantiles (8 passes) and nothing more, the same bits as numpy's quantiles; a single
    non-finite draw: one more select of the extremes (8 passes)"""
    import torch
    from bayes_js_b200.summary import summarise_block
    from summary_ref import ChanBlockReducer, numpy_summary

    class Passes(ChanBlockReducer):
        n = 0

        def digit_counts(self, block, npass, prefix_table):
            Passes.n += 1
            return super().digit_counts(block, npass, prefix_table)

    x = _block(7, 3, 41, 2)
    x[0, 2, 0] = 1e300                                      # finite extremes change nothing
    mean, _sd, _rhat, q = summarise_block(Passes(), torch.from_numpy(x), 7, 41, PROBS, False)
    assert Passes.n == 8 and np.array_equal(q, numpy_summary(x, PROBS)[3]) and np.all(np.isfinite(mean))
    x[3, 1, 7] = -np.inf
    Passes.n = 0
    with np.errstate(invalid="ignore"):
        mean, _sd, _rhat, q = summarise_block(Passes(), torch.from_numpy(x), 7, 41, PROBS, False)
    assert Passes.n == 16 and mean[1] == -np.inf and np.isfinite(mean[[0, 2]]).all()


def test_moments_reference_restates_the_nested_one(pkg):
    """tests/moments_ref.py vectorises nested_ref._superchain over chains: the same exact record and the same bound (at the
    nested reference's L = n + 20 the two bounds are equal; moments_ref passes the moments kernels' shorter merge path)"""
    import moments_ref
    import nested_ref
    rng = np.random.default_rng(9)
    x = rng.normal(size=(13, 5, 301))
    x[:, 0] = 1e6 + 1e-3 * x[:, 0]
    x[:, 1] = np.round(3 * x[:, 1])
    x[:, 2] = 1e150 * (1 + 0.01 * x[:, 2])
    x[:, 3] = 2.0 ** -1023 * (1 + rng.random((13, 301)))
    x[:, 4] = -7.25
    exact, bound = moments_ref.record(x)
    for e in range(5):
        rec, bnd = nested_ref._superchain(x, e, 0, 301)
        assert np.array_equal(exact[e], rec), e
        assert np.all(bound[e] <= bnd) and np.all(bound[e] >= 0), e
    assert exact[4, 2] == exact[4, 3] == 0


def _worker(rank, world, port, q, nonfinite=False):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.parallel import shard_bounds
    from bayes_js_b200.summary import summarise_block
    from summary_ref import ChanBlockReducer, NumpyBlockReducer, numpy_summary
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows, entries, chains = 6, 3, 37                       # ragged: 19 + 18 chains
        x = _block(rows, entries, chains, 11)
        if nonfinite:
            # entry 0: a NaN in rank 0's chains only; entry 1: +inf in rank 1's only; entry 2: -inf in rank 0's, +inf in rank 1's
            x[2, 0, 3] = np.nan
            x[4, 1, 30] = x[0, 1, 33] = np.inf
            x[1, 2, 5], x[5, 2, 20] = -np.inf, np.inf
        first, count = shard_bounds(chains, rank, world)
        mine = torch.from_numpy(np.ascontiguousarray(x[:, :, first:first + count]))
        red = ChanBlockReducer() if nonfinite else NumpyBlockReducer()
        mean, sd, rhat, qq = summarise_block(red, mine, rows, chains, PROBS, True)
        m0, s0, r0, q0 = numpy_summary(x, PROBS)
        if nonfinite:
            ok = (_by_class(mean, m0) and np.isnan(sd).all() and np.isnan(rhat).all()
                  and np.array_equal(qq, q0, equal_nan=True))
        else:
            ok = (np.allclose(mean, m0, rtol=1e-13) and np.allclose(sd, s0, rtol=1e-11) and np.allclose(rhat, r0, rtol=1e-9)
                  and np.array_equal(qq, q0))
        q.put((rank, bool(ok), mean.tobytes() + sd.tobytes() + qq.tobytes()))
    finally:
        dist.destroy_process_group()


def test_summary_over_gloo_world2():
    """the N>1 path: every rank reduces its shard, the records are all-gathered and the digit counts all-reduced; both ranks end
    with the single-process numbers, bit for bit the same on both."""
    _world2(False)


def test_nonfinite_draws_over_gloo_world2():
    """a NaN that only rank 0 holds and a +inf that only rank 1 holds: both ranks count the non-finite draws (the merged mean is
    not finite on both) and return numpy's mean and quantiles, the same bits on both"""
    _world2(True)


def _world2(nonfinite):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, nonfinite)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert all(ok for _, ok, _ in res)
    assert res[0][2] == res[1][2]
