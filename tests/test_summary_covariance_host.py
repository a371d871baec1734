"""Host side of the posterior covariance of sample_summary(..., covariance=...): the checks of the argument, the driver
(summary.covariance_block, finalize_comoments) on CPU tensors with a numpy stand-in for amwg_summary_comoments against numpy.cov,
numpy.corrcoef and scipy's generalized eigenproblem, the rank-order merge of a gloo world of two uneven shards, and the Gram
kernel's addressing (csrc/amwg_comoments.cuh) compiled for the host, driving an emulated mma.sync.m8n8k4.f64, against an fsum
reference within the bound of tests/cov_ref.py."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import cov_ref
from summary_ref import NumpyBlockReducer, run_means

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class NumpyCovReducer(NumpyBlockReducer):
    """numpy stand-in for amwg_summary_comoments on a CPU block [rows, entries, chains]."""

    def comoments(self, block, sel):
        x = block.numpy()[:, np.asarray(sel), :]                 # [rows, n, chains]
        rows, n, chains = x.shape
        xbar = run_means(x)                                     # [n, chains]
        m = run_means(xbar.T)
        f = xbar - m[:, None]
        d = (x - xbar[None]).transpose(1, 0, 2).reshape(n, -1)
        return np.concatenate([[chains], m, (f @ f.T).ravel(), (d @ d.T).ravel()])


NAMES = ["mu", "x", "var"]
DIMS = {"mu": [1], "x": [2, 3], "var": [1]}


def test_resolve_covariance_refuses_bad_arguments(pkg):
    from bayes_js_b200.summary import resolve_covariance
    bad = [["sigma"], [("nope", 0)], [("x", 6)], [("x", -1)], [("x", 1.0)], ["x"], [("x",)], [("x", 1, 2)], [3], [True],
           ["mu", "mu"], ["mu", ("mu", 0)], [], "mu", 1, {"mu": 1}, ("mu",) * 0, np.array([0])]
    for spec in bad:
        with pytest.raises(ValueError, match="covariance"):
            resolve_covariance(spec, NAMES, DIMS)
    many = ["p%d" % i for i in range(129)]
    with pytest.raises(ValueError, match="129 entries"):
        resolve_covariance(True, many, {p: [1] for p in many})
    with pytest.raises(ValueError, match="129 entries"):
        resolve_covariance(["mu"] + [("x", i) for i in range(6)] + [("w", i) for i in range(122)], ["mu", "x", "w"],
                           {"mu": [1], "x": [2, 3], "w": [122]})
    big = {"w": [16, 8]}
    assert len(resolve_covariance(True, ["w"], big).entries) == 128
    with pytest.raises(ValueError, match="named 'covariance'"):
        resolve_covariance(True, ["mu", "covariance"], {"mu": [1], "covariance": [1]})
    with pytest.raises(ValueError, match="named 'covariance'"):
        resolve_covariance(["mu"], ["mu", "covariance"], {"mu": [1], "covariance": [1]})


def test_resolve_covariance_accepts_and_orders(pkg):
    from bayes_js_b200.summary import resolve_covariance
    assert resolve_covariance(None, NAMES, DIMS) is None and resolve_covariance(False, NAMES, DIMS) is None
    p = resolve_covariance(True, NAMES, DIMS)
    assert p.labels == ["mu"] + [("x", i) for i in range(6)] + ["var"] and list(p.entries) == list(range(8))
    p = resolve_covariance(["var", ("x", 5), ["x", 0], ("mu", 0)], NAMES, DIMS)
    assert p.labels == ["var", ("x", 5), ("x", 0), ("mu", 0)] and list(p.entries) == [7, 6, 1, 0]
    assert p.entries.dtype == np.int32
    # a name monitored twice: its last block, as sample_summary reads it
    p = resolve_covariance(True, ["mu", "var", "mu"], DIMS)
    assert p.labels == ["mu", "var"] and list(p.entries) == [2, 1]


def _draws(rows, chains, E, seed):
    """[rows, E, chains] correlated draws offset by 1e6 (centring), chains with distinct means (a between part)"""
    rng = np.random.default_rng(seed)
    L = np.eye(E) + 0.5 * rng.normal(size=(E, E)) / np.sqrt(E)        # well conditioned
    z = rng.normal(size=(rows, chains, E)) @ L.T + rng.normal(size=(1, chains, E))
    return 1e6 + np.ascontiguousarray(z.transpose(0, 2, 1))


def _numpy_check(out, x):
    import scipy.linalg
    rows, E, chains = x.shape
    flat = np.moveaxis(x, 1, 0).reshape(E, -1)
    M = rows * chains
    scale = np.outer(flat.std(axis=1), flat.std(axis=1)) + 1e-300
    if M > 1:
        assert np.all(np.abs(out["cov"] - np.cov(flat).reshape(E, E)) <= 1e-9 * scale)
        with np.errstate(invalid="ignore", divide="ignore"):
            want_corr = np.corrcoef(flat).reshape(E, E)
        assert np.allclose(out["corr"], want_corr, rtol=0, atol=1e-9, equal_nan=True)
    else:
        assert np.all(np.isnan(out["cov"]))
    assert np.all(np.abs(out["mean"] - flat.mean(axis=1)) <= 1e-15 * np.abs(flat).max())
    assert out["n_draws"] == M
    if rows < 2 or chains < 2 or chains * (rows - 1) < E:       # the last: within has rank C (rows - 1) < E, not positive definite
        assert np.isnan(out["rhat_multivariate"])
        return
    within = np.mean([np.cov(x[:, :, c].T).reshape(E, E) for c in range(chains)], axis=0)
    between = np.cov(x.mean(axis=0)).reshape(E, E)
    assert np.all(np.abs(out["within"] - within) <= 1e-9 * scale)
    assert np.all(np.abs(out["between"] - between) <= 1e-9 * scale)
    lam = scipy.linalg.eigh(between, within, eigvals_only=True).max()
    want = (rows - 1) / rows + (chains + 1) / chains * lam
    assert abs(out["rhat_multivariate"] - want) <= 1e-7 * want, (out["rhat_multivariate"], want)


@pytest.mark.parametrize("rows", [1, 2, 7, 100])
@pytest.mark.parametrize("chains", [1, 3, 41])
@pytest.mark.parametrize("E", [1, 2, 9, 65])
def test_covariance_block_matches_numpy(pkg, rows, chains, E):
    import torch
    from bayes_js_b200.summary import covariance_block, resolve_covariance
    x = _draws(rows, chains, E, rows * 1000 + chains * 10 + E)
    names = ["p%d" % i for i in range(E)]
    plan = resolve_covariance(True, names, {p: [1] for p in names})
    out = covariance_block(NumpyCovReducer(), torch.from_numpy(x), rows, plan, False)
    assert out["labels"] == names
    _numpy_check(out, x)
    if E == 1 and rows >= 2 and chains >= 2:
        # the closed form from amwg_summary_moments' record: (n-1)/n + (C+1)/C (B/(C-1)) / (W/(C(n-1)))
        G, _m, b2, sw = NumpyCovReducer().moments(torch.from_numpy(x))[0]
        want = (rows - 1) / rows + (G + 1) / G * (b2 / (G - 1)) / (sw / (G * (rows - 1)))
        assert abs(out["rhat_multivariate"] - want) <= 1e-13 * want


def test_non_finite_entries_give_nan_rows_and_columns(pkg):
    import torch
    from bayes_js_b200.summary import covariance_block, resolve_covariance
    x = _draws(7, 41, 5, 3)
    x[3, 1, 7] = np.nan
    x[0, 3, 40] = np.inf
    names = ["a", "b", "c", "d", "e"]
    out = covariance_block(NumpyCovReducer(), torch.from_numpy(x), 7, resolve_covariance(True, names, {p: [1] for p in names}), False)
    flat = np.moveaxis(x, 1, 0).reshape(5, -1)
    with np.errstate(invalid="ignore"):
        want = np.cov(flat)
    assert np.array_equal(np.isnan(out["cov"]), np.isnan(want))
    bad = np.array([False, True, False, True, False])
    for key in ("cov", "corr", "within", "between"):
        assert np.all(np.isnan(out[key][bad])) and np.all(np.isnan(out[key][:, bad])), key
        assert np.all(np.isfinite(out[key][np.ix_(~bad, ~bad)])), key
    assert np.isnan(out["rhat_multivariate"])


def test_rhat_is_nan_when_within_is_singular(pkg):
    import torch
    from bayes_js_b200.summary import covariance_block, resolve_covariance
    x = _draws(9, 5, 3, 4)
    x[:, 2] = 2 * x[:, 0] - x[:, 1]                             # linear in the others
    names = ["a", "b", "c"]
    out = covariance_block(NumpyCovReducer(), torch.from_numpy(x), 9, resolve_covariance(True, names, {p: [1] for p in names}), False)
    assert np.isnan(out["rhat_multivariate"])
    x[:, 2] = 4.0                                                # constant
    out = covariance_block(NumpyCovReducer(), torch.from_numpy(x), 9, resolve_covariance(True, names, {p: [1] for p in names}), False)
    assert np.isnan(out["rhat_multivariate"]) and np.isnan(out["corr"][2]).all()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import __graft_entry__ as graft
    graft.load_package()
    import cov_ref
    from bayes_js_b200.summary import covariance_block, resolve_covariance
    from test_summary_covariance_host import NumpyCovReducer, _draws
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows = 6
        x = _draws(rows, 37, 4, 11)
        cut = 30                                                 # uneven shards: 30 + 7 chains
        mine = x[:, :, :cut] if rank == 0 else x[:, :, cut:]
        names = ["a", "b", "c", "d"]
        plan = resolve_covariance(["d", "a", "c"], names, {p: [1] for p in names})
        out = covariance_block(NumpyCovReducer(), torch.from_numpy(np.ascontiguousarray(mine)), rows, plan, True)
        one = covariance_block(NumpyCovReducer(), torch.from_numpy(x), rows, plan, False)
        keys = ("mean", "cov", "corr", "within", "between")
        image = b"".join(np.ascontiguousarray(out[k]).tobytes() for k in keys) + np.float64(out["rhat_multivariate"]).tobytes()
        # both records lie within the device bound of the exact one (cov_ref), so they differ by at most twice that bound
        bm, bB, bW = cov_ref.device_bound(x, plan.entries)
        Cn, M = 37, rows * 37
        tol = {"mean": 2 * bm, "within": 2 * bW / (Cn * (rows - 1)), "between": 2 * bB / (Cn - 1), "cov": (2 * bW + rows * 2 * bB) / (M - 1),
               "corr": 1e-9}
        close = all(np.all(np.abs(out[k] - one[k]) <= tol[k]) for k in keys)
        close = close and abs(out["rhat_multivariate"] - one["rhat_multivariate"]) <= 1e-9 * one["rhat_multivariate"]
        q.put((rank, close and out["labels"] == ["d", "a", "c"] and out["n_draws"] == rows * 37, image))
    finally:
        dist.destroy_process_group()


def test_covariance_over_gloo_world2():
    """every rank reduces its shard; one all-gather of the records, merged in rank order, gives both ranks the same bytes"""
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


def test_merge_matches_one_record(pkg):
    import torch
    from bayes_js_b200.summary import merge_comoment_records, split_comoment_record
    x = _draws(5, 40, 3, 8)
    red = NumpyCovReducer()
    sel = [2, 0, 1]
    parts = [red.comoments(torch.from_numpy(np.ascontiguousarray(x[:, :, a:b])), sel) for a, b in ((0, 13), (13, 14), (14, 40))]
    G, m, B, W = split_comoment_record(merge_comoment_records(parts))
    G1, m1, B1, W1 = split_comoment_record(red.comoments(torch.from_numpy(x), sel))
    assert G == G1 == 40
    assert np.allclose(m, m1, rtol=1e-15) and np.allclose(B, B1, rtol=1e-9) and np.allclose(W, W1, rtol=1e-12)


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("cov") / "libcomoments_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "comoments_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    lib.hs_comoments.restype = C.c_int64
    lib.hs_comoments.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
    return lib


@pytest.mark.parametrize("E", [1, 7, 8, 9, 65, 128])
@pytest.mark.parametrize("chains", [1, 3, 4, 1001])
def test_tile_schedule_on_the_host(H, E, chains):
    """the kernel's grid, stages, warps, tiles and partials with an emulated DMMA: no index leaves its buffer, every fragment read
    was staged, every partial is written once, and B and W lie within the stated bound of the fsum reference"""
    rows = 3 if E >= 65 else 17                                  # 17: two stages of 16 rows at E <= 8, ragged
    rng = np.random.default_rng(E * 7919 + chains)
    entries = E + 2
    x = 1e6 + rng.normal(size=(rows, entries, chains)) * rng.uniform(0.5, 3, size=(1, entries, 1)) + rng.normal(size=(1, entries, chains))
    sel = rng.permutation(entries)[:E].astype(np.int32)
    out = np.empty(1 + E + 2 * E * E)
    bad = H.hs_comoments(x.ctypes.data, rows, entries, chains, sel.ctypes.data, E, out.ctypes.data)
    assert bad == 0
    cov_ref.check_record(out, x, sel, (E, chains))


def _co_stage_rows(nb):
    return max(16 // nb, 1)                                      # amwg_comoments.cuh: co_stage_rows


@pytest.mark.parametrize("nb", range(1, 17))
@pytest.mark.parametrize("chains", [8449, 2 * 8448 + 37])
def test_tile_schedule_every_block_count_over_the_grid_walk(H, nb, chains):
    """every block count nb = 1..16, full (8 nb entries) at 8449 chains and ragged (8 nb - 5) at 2 * 8448 + 37, two staged passes
    plus a ragged row, where each of the 264 CTAs walks two or three 32-chain groups and the last group is ragged: every value
    loaded once, every (tile, row, quad) step issued once across the reps, and B and W within the bound of the reference"""
    rows = 2 * _co_stage_rows(nb) + 1
    for E in [8 * nb if chains == 8449 else max(8 * nb - 5, 1)]:
        rng = np.random.default_rng(nb * 7919 + chains + E)
        entries = E + 1
        x = 184.5 + rng.normal(size=(rows, entries, chains)) * rng.uniform(0.1, 3, size=(1, entries, 1))
        x += 0.3 * rng.normal(size=(1, entries, chains))
        sel = rng.permutation(entries)[:E].astype(np.int32)
        out = np.empty(1 + E + 2 * E * E)
        assert H.hs_comoments(x.ctypes.data, rows, entries, chains, sel.ctypes.data, E, out.ctypes.data) == 0
        cov_ref.check_record(out, x, sel, (nb, E, chains), exact=cov_ref.record(x, sel))


@pytest.mark.parametrize("rows, chains, n", [(1, 1, 1), (3, 5, 2), (17, 41, 9), (2, 1001, 3), (20, 300, 65)])
def test_vectorised_reference_agrees_with_its_loop_form(rows, chains, n):
    rng = np.random.default_rng(rows * 100 + chains + n)
    x = 1e6 + rng.normal(size=(rows, n + 1, chains)) + rng.normal(size=(1, n + 1, chains))
    x[:, 0] = 0.1                                               # a constant entry: exact zeros in both forms
    sel = list(rng.permutation(n + 1)[:n])
    C0, m0, B0, W0 = cov_ref.exact_record(x, sel)
    C1, m1, B1, W1 = cov_ref.record(x, sel)
    bm, bB, bW = cov_ref.device_bound(x, sel)
    assert C0 == C1
    assert np.all(np.abs(m1 - m0) <= 2 * cov_ref.U * np.abs(m0))
    # far inside the device bound: the two forms differ by less than 1 / 100 of it
    assert np.all(np.abs(W1 - W0) <= bW / 100) and np.all(np.abs(B1 - B0) <= bB / 100)


def _constant_block(value, rows, chains, seed):
    """[rows, 4, chains]: two correlated normal entries, `value` everywhere in entry 2, entry 3 constant within each chain"""
    rng = np.random.default_rng(seed)
    z = rng.normal(size=(rows, chains))
    x = np.empty((rows, 4, chains))
    x[:, 0] = 10.0 + z
    x[:, 1] = -3.0 + 0.6 * z + 0.8 * rng.normal(size=(rows, chains))
    x[:, 2] = value
    x[:, 3] = value + (abs(value) + 1.0) * 1e-3 * rng.normal(size=(1, chains))
    return x


@pytest.mark.parametrize("value", [0.1, 184.3, 7.25, -1e150, 5e-324])
@pytest.mark.parametrize("rows, chains", [(3, 1000), (50, 1001)])
def test_constant_entry_has_exact_zero_rows_on_the_host_build(H, pkg, value, rows, chains):
    """The kernels' text: an entry whose draws all equal one value has that value as its mean and exactly zero rows and
    columns of B and W, so corr is NaN there (as numpy.corrcoef gives) and rhat_multivariate is NaN; an entry constant within
    each chain has zero rows of W and a between part."""
    from bayes_js_b200.summary import finalize_comoments
    x = _constant_block(value, rows, chains, 5)
    sel = np.arange(4, dtype=np.int32)
    out = np.empty(1 + 4 + 2 * 16)
    assert H.hs_comoments(x.ctypes.data, rows, 4, chains, sel.ctypes.data, 4, out.ctypes.data) == 0
    m, B, W = out[1:5], out[5:21].reshape(4, 4), out[21:].reshape(4, 4)
    assert m[2] == value
    assert np.all(B[2] == 0) and np.all(B[:, 2] == 0) and np.all(W[2] == 0) and np.all(W[:, 2] == 0)
    assert np.all(W[3] == 0) and np.all(W[:, 3] == 0) and B[3, 3] > 0
    fin = finalize_comoments(out, rows)
    assert np.all(fin["cov"][2] == 0) and np.all(fin["within"][:, 2] == 0) and np.all(fin["between"][2] == 0)
    assert np.all(np.isnan(fin["corr"][2])) and np.all(np.isnan(fin["corr"][:, 2]))
    assert np.isnan(fin["rhat_multivariate"])
    assert np.all(np.isfinite(fin["corr"][np.ix_([0, 1, 3], [0, 1, 3])]))
    # the two normal entries alone keep their bound and a finite R-hat
    keep = np.array([0, 1], dtype=np.int32)
    out2 = np.empty(1 + 2 + 8)
    assert H.hs_comoments(x.ctypes.data, rows, 4, chains, keep.ctypes.data, 2, out2.ctypes.data) == 0
    cov_ref.check_record(out2, x, keep, value)
    assert np.isfinite(finalize_comoments(out2, rows)["rhat_multivariate"])


def test_mixed_signed_zeros_keep_the_summed_mean(H):
    """a run of -0 and +0 is not bitwise constant: the mean is fl(sum) / n = +0, as before the rule"""
    x = np.zeros((4, 1, 3))
    x[0, 0, :] = -0.0
    x[:, 0, 1] = -0.0                                            # chain 1 all -0: its mean is -0
    sel = np.zeros(1, dtype=np.int32)
    out = np.empty(1 + 1 + 2)
    assert H.hs_comoments(x.ctypes.data, 4, 1, 3, sel.ctypes.data, 1, out.ctypes.data) == 0
    assert out[1] == 0 and out[2] == 0 and out[3] == 0
    assert not np.signbit(out[1])                                # the chain means -0, +0, +0 differ in bits: summed, +0
