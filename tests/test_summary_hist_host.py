"""Host side of the posterior histograms of sample_summary(..., histogram=...): the checks of the argument, the driver
(summary.histogram_block) on CPU tensors with a numpy stand-in for the three device reductions, the collectives of a gloo
world of two uneven shards, and the kernels' two bin rules (csrc/amwg_hist.cuh) compiled for the host against numpy."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from summary_ref import NumpyBlockReducer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class NumpyHistReducer(NumpyBlockReducer):
    """numpy stand-in for amwg_summary_finite_range / _histogram / _histogram2d on a CPU block [rows, entries, chains]."""

    def finite_range(self, block):
        import torch
        x = block.numpy()
        entries = x.shape[1]
        rng = np.empty((entries, 2))
        nonfinite = np.empty((entries, 3), dtype=np.int64)
        for e in range(entries):
            v = x[:, e].ravel()
            f = v[np.isfinite(v)]
            rng[e] = (f.min(), f.max()) if f.size else (np.inf, -np.inf)
            nonfinite[e] = ((v == -np.inf).sum(), (v == np.inf).sum(), np.isnan(v).sum())
        return torch.from_numpy(rng), torch.from_numpy(nonfinite)

    def histogram(self, block, edges, bins):
        import torch
        x = block.numpy()
        out = np.zeros((x.shape[1], bins + 3), dtype=np.int64)
        for e in range(x.shape[1]):
            v = x[:, e].ravel()
            lo, hi = edges[e, 0], edges[e, -1]
            out[e, :bins] = np.histogram(v[~np.isnan(v)], bins=bins, range=(lo, hi))[0]
            out[e, bins:] = ((v < lo).sum(), (v > hi).sum(), np.isnan(v).sum())
        return torch.from_numpy(out)

    def histogram2d(self, block, pairs, edges, bins):
        import torch
        x = block.numpy()
        out = np.zeros((len(pairs), bins, bins), dtype=np.int64)
        for i, (a, b) in enumerate(pairs):
            out[i] = np.histogram2d(x[:, a].ravel(), x[:, b].ravel(), bins=[edges[a], edges[b]])[0].astype(np.int64)
        return torch.from_numpy(out)


NAMES = ["mu", "x", "var"]
DIMS = {"mu": [1], "x": [2, 3], "var": [1]}


def _block(rows, chains, seed):
    """[rows, 8, chains]: mu (narrow, far from 0), x (2 x 3 ints, one component constant, one with no finite draw), var."""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, 8, chains))
    x[:, 0] = 184.5 + 0.14 * rng.normal(size=(rows, chains))
    x[:, 1:7] = np.round(3 * rng.normal(size=(rows, 6, chains)))
    x[:, 2] = 4.0                                             # x[0, 1]: constant
    x[:, 3] = np.where(rng.random((rows, chains)) < 0.5, np.nan, np.inf)     # x[0, 2]: no finite draw
    x[0, 4, :3] = (-np.inf, np.inf, np.nan)
    x[:, 7] = np.exp(rng.normal(size=(rows, chains)))
    x[-1, 7, 0] = -0.0
    return x


def test_resolve_histogram_refuses_bad_arguments(pkg):
    from bayes_js_b200.summary import resolve_histogram
    bad = [2.5, True, "10", [10], {"bins": 0}, {"bins": 4097}, {"bins": 2.5}, {"bins": True}, {"bins": np.float64(3)},
           {"bins": 10, "pair_bins": 129}, {"pairs": [("mu", "var")], "pair_bins": 0}, {"bins": 10, "pair_bins": False},
           {"bins": 10, "range": {"mu": (1.0, 1.0)}}, {"bins": 10, "range": {"mu": (2.0, 1.0)}},
           {"bins": 10, "range": {"mu": (0.0, np.inf)}}, {"bins": 10, "range": {"mu": (np.nan, 1.0)}},
           {"bins": 10, "range": {"mu": (0.0,)}}, {"bins": 10, "range": {"mu": (True, 2)}}, {"bins": 10, "range": {"sigma": (0, 1)}},
           {"bins": 10, "range": [("mu", 0, 1)]}, {"pairs": [("mu", "sigma")]}, {"pairs": [("x", "mu")]}, {"pairs": [(("x", 6), "mu")]},
           {"pairs": [(("x", -1), "mu")]}, {"pairs": [(("x", 1.0), "mu")]}, {"pairs": [("mu",)]}, {"pairs": [("mu", "var", "mu")]},
           {"pairs": [("mu", "var")] * 65}, {"pairs": "mu"}, {}, {"pairs": []}, {"bins": 10, "bin": 3}]
    for spec in bad:
        with pytest.raises(ValueError, match="histogram"):
            resolve_histogram(spec, NAMES, DIMS)


def test_resolve_histogram_accepts_and_plans(pkg):
    from bayes_js_b200.summary import PAIR_BINS, resolve_histogram
    assert resolve_histogram(None, NAMES, DIMS) is None
    p = resolve_histogram(40, NAMES, DIMS)
    assert p.bins == 40 and p.pairs == [] and p.fixed.shape == (8, 2) and np.isnan(p.fixed).all()
    assert resolve_histogram(np.int64(4096), NAMES, DIMS).bins == 4096
    p = resolve_histogram({"range": {"x": (-0.5, 4.5)}, "pairs": [(("x", 3), "var"), ["mu", ["x", 0]], (("x", 3), "var")],
                           "pair_bins": 1}, NAMES, DIMS)
    assert p.bins is None and p.pair_bins == 1
    assert p.pairs == [((("x", 3), "var"), 4, 7), (("mu", ("x", 0)), 0, 1)]
    assert np.array_equal(p.fixed[1:7], np.tile([-0.5, 4.5], (6, 1))) and np.isnan(p.fixed[[0, 7]]).all()
    p = resolve_histogram({"bins": 1, "pairs": [("mu", "mu")]}, NAMES, DIMS)
    assert p.pair_bins == PAIR_BINS and p.pairs == [(("mu", "mu"), 0, 0)]
    # a name monitored twice: its last block, as sample_summary reads it
    p = resolve_histogram({"bins": 3, "range": {"mu": (0, 1)}, "pairs": [("mu", "var")]}, ["mu", "var", "mu"], DIMS)
    assert np.isnan(p.fixed[0, 0]) and p.fixed[2, 0] == 0 and p.pairs == [(("mu", "var"), 2, 1)]


def _numpy_hist(v, k, rng=None):
    """numpy.histogram of the finite draws (range: given, or autodetected) and the counts below / above / NaN."""
    f = v[np.isfinite(v)]
    if rng is None and f.size == 0:
        rng = (0.0, 1.0)
    h, ed = np.histogram(f, bins=k, range=rng)
    lo, hi = ed[0], ed[-1]
    return h, ed, np.array([(v < lo).sum(), (v > hi).sum(), np.isnan(v).sum()])


@pytest.mark.parametrize("rows,chains,bins", [(7, 41, 40), (1, 64, 1), (13, 3, 4096)])
def test_histogram_block_matches_numpy(pkg, rows, chains, bins):
    import torch
    from bayes_js_b200.summary import histogram_block, resolve_histogram
    x = _block(rows, chains, rows * 100 + chains)
    plan = resolve_histogram({"bins": bins, "range": {"var": (0.5, 2.0)}, "pairs": [("mu", "var"), (("x", 3), ("x", 0))],
                              "pair_bins": 32}, NAMES, DIMS)
    out = histogram_block(NumpyHistReducer(), torch.from_numpy(x), rows, plan, False)
    for e in range(8):
        v = x[:, e].ravel()
        h, ed, outside = _numpy_hist(v, bins, (0.5, 2.0) if e == 7 else None)
        assert np.array_equal(out["hist"][e], h), e
        assert np.array_equal(out["hist_edges"][e], ed), e       # by value: -0.0 == +0.0
        assert np.array_equal(out["hist_outside"][e], outside), e
        assert out["hist"][e].sum() + out["hist_outside"][e].sum() == rows * chains
    assert np.array_equal(out["hist_edges"][2], np.linspace(3.5, 4.5, bins + 1))     # constant entry: (c - 0.5, c + 0.5)
    assert np.array_equal(out["hist_edges"][3], np.linspace(0.0, 1.0, bins + 1))     # no finite draw: (0, 1)
    assert out["hist"][3].sum() == 0

    def auto(v):
        f = v[np.isfinite(v)]
        return (f.min() - 0.5, f.max() + 0.5) if f.min() == f.max() else (f.min(), f.max())

    for key, a, b in [(("mu", "var"), 0, 7), ((("x", 3), ("x", 0)), 4, 1)]:
        ra = auto(x[:, a].ravel())
        rb = (0.5, 2.0) if b == 7 else auto(x[:, b].ravel())
        want, xe, ye = np.histogram2d(x[:, a].ravel(), x[:, b].ravel(), bins=32, range=[ra, rb])
        got = out["pairs"][key]
        assert np.array_equal(got["hist"], want.astype(np.int64)), key
        assert np.array_equal(got["xedges"], xe) and np.array_equal(got["yedges"], ye)


def test_histogram_block_pairs_only_skips_the_1d_counts(pkg):
    import torch
    from bayes_js_b200.summary import histogram_block, resolve_histogram
    x = _block(5, 20, 9)
    plan = resolve_histogram({"pairs": [("mu", "var")], "range": {"mu": (184.0, 185.0), "var": (0.0, 3.0)}, "pair_bins": 7}, NAMES, DIMS)

    class NoRange(NumpyHistReducer):
        def finite_range(self, block):
            raise AssertionError("every range used is given: the extremes are not needed")

    out = histogram_block(NoRange(), torch.from_numpy(x), 5, plan, False)
    assert set(out) == {"pairs"}
    want = np.histogram2d(x[:, 0].ravel(), x[:, 7].ravel(), bins=7, range=[(184.0, 185.0), (0.0, 3.0)])[0]
    assert np.array_equal(out["pairs"][("mu", "var")]["hist"], want.astype(np.int64))


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    from bayes_js_b200.summary import histogram_block, resolve_histogram
    from test_summary_hist_host import NAMES, DIMS, NumpyHistReducer, _block
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows, chains = 6, 37
        x = _block(rows, chains, 11)
        cut = 30                                                 # uneven shards: 30 + 7 chains; the extremes lie in either
        mine = x[:, :, :cut] if rank == 0 else x[:, :, cut:]
        plan = resolve_histogram({"bins": 17, "pairs": [("mu", "var"), (("x", 0), ("x", 4))], "pair_bins": 9}, NAMES, DIMS)
        out = histogram_block(NumpyHistReducer(), torch.from_numpy(np.ascontiguousarray(mine)), rows, plan, True)
        one = histogram_block(NumpyHistReducer(), torch.from_numpy(x), rows, plan, False)

        def image(o):
            parts = [o["hist"], o["hist_edges"], o["hist_outside"]]
            for key in sorted(o["pairs"], key=repr):
                parts += [o["pairs"][key]["hist"], o["pairs"][key]["xedges"], o["pairs"][key]["yedges"]]
            return b"".join(np.ascontiguousarray(p).tobytes() for p in parts)
        q.put((rank, image(out) == image(one), image(out)))
    finally:
        dist.destroy_process_group()


def test_histograms_over_gloo_world2():
    """every rank counts its shard; one all-reduce of the extremes and one of the counts give both ranks the single-shard bytes"""
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


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("hist") / "libhist_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "hist_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    vp = C.c_void_p
    for f in (lib.hs_hist_bin, lib.hs_hist2d_axis):
        f.restype, f.argtypes = None, [vp, C.c_int64, vp, C.c_int, vp]
    return lib


# bins a few ulps wide, subnormal and near-overflow ranges, one bin, unit bins; numpy refuses edges that repeat, so none do here
RANGES = [(0.0, 1.0, 10), (-1.0, 1.0, 7), (184.2, 185.1, 50), (-3e-310, 2e-310, 13), (1e15, 1e15 + 4096, 4096), (1.0, 2.0, 1),
          (-5.5, 5.5, 11), (0.1, 0.7, 3), (-1e300, 1e300, 4096), (-0.0, 1e-323, 2), (1 - 2 ** -50, 1 + 2 ** -50, 4), (3.0, 3.0 + 1e-11, 4096),
          (-7.25, 1e-3, 128), (184.49, 184.51, 128)]


def _adversarial(lo, hi, k, rng):
    """every edge and 1-3 ulps to each side, both zeros, subnormals, the ends of the double range, random draws inside."""
    ed = np.linspace(lo, hi, k + 1)
    v = [ed]
    up, dn = ed.copy(), ed.copy()
    for _ in range(3):
        up, dn = np.nextafter(up, np.inf), np.nextafter(dn, -np.inf)
        v += [up, dn]
    v.append(np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -1e-310, np.inf, -np.inf, np.nan, 1.7976931348623157e308,
                       -1.7976931348623157e308, lo, hi]))
    v.append(rng.uniform(lo, hi, 80000) if np.isfinite(hi - lo) else rng.uniform(-1, 1, 80000) * 1e300)
    return np.concatenate(v)


def _axis_ref(v, ed):
    """numpy.histogramdd's per-axis rule, with its own operations"""
    k = len(ed) - 1
    i = np.searchsorted(ed, v, side="right")
    i[v == ed[-1]] -= 1
    return np.where((i >= 1) & (i <= k), i - 1, -1)


def test_bin_rules_compiled_for_the_host_agree_with_numpy(H):
    rng = np.random.default_rng(4)
    total = 0
    for lo, hi, k in RANGES:
        ed = np.linspace(lo, hi, k + 1)
        assert np.all(ed[1:] > ed[:-1])
        v = _adversarial(lo, hi, k, rng)
        total += v.size
        got = np.empty(v.size, dtype=np.int32)
        H.hs_hist_bin(v.ctypes.data, v.size, ed.ctypes.data, k, got.ctypes.data)
        inside = (v >= lo) & (v <= hi)
        assert np.array_equal(got[v < lo], np.full((v < lo).sum(), -1)) and np.array_equal(got[v > hi], np.full((v > hi).sum(), -2))
        assert np.all(got[np.isnan(v)] == -3)
        # index for index: on the sorted values the bins never decrease and reproduce numpy's counts, which fixes every index
        order = np.argsort(v[inside], kind="stable")
        s, gi = v[inside][order], got[inside][order]
        assert np.all(np.diff(gi) >= 0) and gi.min() >= 0 and gi.max() < k, (lo, hi, k)
        assert np.array_equal(np.bincount(gi, minlength=k), np.histogram(s, bins=k, range=(lo, hi))[0]), (lo, hi, k)
        # and value by value for the edges and their neighbours
        for x, b in list(zip(v[inside], got[inside]))[:8 * (k + 1):max(1, k // 64)]:
            assert np.histogram([x], bins=k, range=(lo, hi))[0][b] == 1, (lo, hi, k, x)
        if k <= 128:
            got2 = np.empty(v.size, dtype=np.int32)
            H.hs_hist2d_axis(v.ctypes.data, v.size, ed.ctypes.data, k, got2.ctypes.data)
            assert np.array_equal(got2, _axis_ref(v, ed)), (lo, hi, k)
            w = rng.permutation(v)
            both = (got2 >= 0) & (_axis_ref(w, ed) >= 0)
            cnt = np.zeros((k, k), dtype=np.int64)
            np.add.at(cnt, (got2[both], _axis_ref(w, ed)[both]), 1)
            assert np.array_equal(cnt, np.histogram2d(v, w, bins=k, range=[(lo, hi), (lo, hi)])[0].astype(np.int64)), (lo, hi, k)
    assert total > 10 ** 6
