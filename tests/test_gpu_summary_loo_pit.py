"""LOO-PIT in sample_summary(..., ppc={..., "loo_pit": ...}) on the GPU: the device reductions (amwg_loo_pit_reduce,
amwg_loo_pit_fit) through summary.ppc_block against the numpy restatement of tests/loo_pit_ref.py on the CPU tier's cases, at one
chain and past the reduce kernel's grid stride; their sums and k bit-equal to PSIS-LOO's kernels; the fit over uneven chain ranges
byte-equal to one range; the device-index refusal; the config-2 model end to end (against the restatement on a twin's draws, over
chunks, every other key and the chains unchanged, pareto_k equal to loo='s); ties of a Poisson model's repeated states, in either
chain order; calibration on a conjugate Normal model against the closed-form leave-one-out predictive; and config 2 at 2^20 chains
in forced chunks of 100 points."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy import stats as st

import loo_pit_ref
import loo_ref
import models
import ppc_ref
from conftest import config2_data
from test_summary_loo_pit_host import _flat, case_bern, case_normal, case_pois

pytestmark = pytest.mark.gpu
TOL = 1e-10


class CudaSource:
    """a block [rows, points, chains] held on the device, handed out in chunks of points"""

    def __init__(self, x3):
        self.x = x3 if torch.is_tensor(x3) else torch.from_numpy(np.ascontiguousarray(x3, dtype=np.float64)).to("cuda:0")

    def chunk(self, p0, P):
        return self.x[:, p0:p0 + P, :].contiguous()


class CudaReplicates(CudaSource):
    """y_rep [rows, points, chains] on the device, with each draw's dataset statistics as amwg_ppc_pointwise leaves them"""

    def stats(self):
        y = self.x.cpu().numpy()
        rows, N, chains = y.shape
        T = ppc_ref.dataset_stats_many(np.moveaxis(y, 1, 2).reshape(-1, N)).reshape(rows, chains, 4)
        return torch.from_numpy(np.ascontiguousarray(np.moveaxis(T, 2, 1))).to("cuda:0")


def _device_pit(ll3, yrep3, y, r_eff=1.0, chunk=None, family="norm"):
    from bayes_js_b200.summary import CudaBlockReducer, ppc_block
    rows, N, chains = tuple(ll3.shape)
    return ppc_block(CudaBlockReducer(0), CudaReplicates(yrep3), rows, chains, N, family, y, (0.5,), chunk or N, False,
                     loo_pit=(CudaSource(ll3), r_eff))


def _same(x, y):
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    a, b = np.asarray(x), np.asarray(y)
    if a.dtype.kind in "fiub":
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


def assert_pit_matches(got, ref, tol=TOL):
    for key in ("pit", "pit_equal"):
        g, w = got[key], ref[key]
        assert np.array_equal(np.isnan(g), np.isnan(w)), key
        ok = ~np.isnan(w)
        assert np.all(np.abs(g[ok] - w[ok]) <= tol), (key, np.max(np.abs(g[ok] - w[ok])))
    g, w = got["pareto_k"], ref["pareto_k"]
    assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(np.isinf(g), np.isinf(w))
    fin = np.isfinite(w)
    assert np.all(np.abs(g[fin] - w[fin]) <= tol * np.maximum(1.0, np.abs(w[fin]))), (g, w)
    assert got["n_high_k"] == ref["n_high_k"]


# ---- the reductions on the CPU tier's cases -----------------------------------------------------------------------------------------
def _nan_yrep():
    ll3, yrep3, y = case_normal(seed=4)
    yrep3[:, 3, :] = np.nan
    yrep3[1, 5, ::7] = np.nan
    return ll3, yrep3, y


def _non_finite():
    ll3, yrep3, y = case_normal(seed=5)
    ll3[:, 2, :] = np.nan
    ll3[0, 6, 11] = -np.inf
    return ll3, yrep3, y


def _dbl_min_floor():
    rng = np.random.default_rng(7)
    S, N = 1000, 3
    ll = rng.normal(0.0, 1.0, size=(S, N))
    ll[:50] -= 1000.0
    yrep = rng.normal(0.0, 1.0, size=(S, N))
    return ll.reshape(1, S, N).transpose(0, 2, 1).copy(), yrep.reshape(1, S, N).transpose(0, 2, 1).copy(), np.array([0.1, -0.4, 1.2])


CASES = {
    "normal": (case_normal, 1.0, "norm"),
    "pois": (case_pois, 1.0, "pois"),
    "bern": (case_bern, 1.0, "bern"),
    "nan_yrep": (_nan_yrep, 1.0, "norm"),
    "non_finite": (_non_finite, 1.0, "norm"),
    "tail_of_four": (lambda: case_normal(rows=1, chains=20, N=5, seed=6), 1.0, "norm"),
    "dbl_min_floor": (_dbl_min_floor, 1.0, "norm"),
    "r_eff": (lambda: case_normal(rows=2, chains=400, N=6, seed=9), 0.3, "norm"),
    "one_chain": (lambda: case_pois(rows=400, chains=1, N=5, seed=31), 1.0, "pois"),
    "grid_stride": (lambda: case_normal(rows=2, chains=1184 * 256 + 77, N=3, seed=33), 1.0, "norm"),
}


@pytest.mark.parametrize("name", list(CASES))
def test_reductions_equal_the_restatement(gpu_pkg, name):
    build, r_eff, fam = CASES[name]
    ll3, yrep3, y = build()
    ref = loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), y, r_eff)
    out = _device_pit(ll3, yrep3, y, r_eff, family=fam)
    assert_pit_matches(out["loo_pit"], ref)
    for chunk in (1, 7):
        assert _same(out["loo_pit"], _device_pit(ll3, yrep3, y, r_eff, chunk, fam)["loo_pit"]), chunk


def _reduce_inputs(ll3, M):
    from bayes_js_b200.summary import LOG_TINY
    flat = _flat(ll3)
    llmin, llmax = flat.min(axis=0), flat.max(axis=0)
    cut = np.maximum(llmin - np.sort(flat, axis=0)[M], LOG_TINY)
    return llmin, llmax, cut


@pytest.mark.parametrize("name", ["normal", "pois", "bern", "grid_stride"])
def test_sums_and_fit_have_psis_loo_bits(gpu_pkg, name):
    """amwg_loo_pit_reduce's sum exp(lw) has the bits of amwg_loo_reduce's, and amwg_loo_pit_fit's k and sum w those of
    amwg_loo_fit, on the same chunk and tails"""
    from bayes_js_b200.summary import CudaBlockReducer, loo_tail_cap, loo_tail_length
    ll3, yrep3, y = CASES[name][0]()
    rows, P, chains = ll3.shape
    M = loo_tail_length(rows * chains, 1.0)
    cap = loo_tail_cap(M)
    llmin, llmax, cut = _reduce_inputs(ll3, M)
    red = CudaBlockReducer(0)
    ll, yr = CudaSource(ll3).x, CudaSource(yrep3).x
    sums, tails, counts = red.loo_reduce(ll, llmin, llmax, cut, cap)
    psums, ptails, flags, pcounts = red.loo_pit_reduce(ll, yr, llmin, cut, y, cap)
    assert sums[:, 1].tobytes() == psums[:, 0].tobytes()
    assert np.array_equal(counts.cpu().numpy(), pcounts.cpu().numpy())
    skip = np.zeros(P, dtype=np.int32)
    fit = red.loo_fit(tails[None], counts[None], llmin, cut, skip)
    pfit = red.loo_pit_fit(ptails[None], flags[None], pcounts[None], llmin, cut, skip)
    assert fit[:, :2].tobytes() == pfit[:, :2].tobytes() and np.array_equal(fit[:, 3], pfit[:, 4])
    assert np.all(pfit[:, 2] >= pfit[:, 3]) and np.all(pfit[:, 2] <= pfit[:, 1] * (1 + 1e-12))


@pytest.mark.parametrize("ranges", [[(0, 70), (70, 200)], [(0, 33), (33, 150), (150, 200)]])
def test_fit_over_uneven_chain_ranges_equals_one_range(gpu_pkg, ranges):
    """amwg_loo_pit_reduce per chain range, tails, flags and counts stacked as the multi-GPU path gathers them, one
    amwg_loo_pit_fit: byte-equal to one range and to a repeat (whose atomic slot order, and so the order of tied draws, differs)"""
    from bayes_js_b200.summary import CudaBlockReducer, loo_tail_cap, loo_tail_length
    ll3, yrep3, y = case_pois(rows=8, chains=200, N=9, seed=41)
    rows, P, chains = ll3.shape
    M = loo_tail_length(rows * chains, 1.0)
    cap = loo_tail_cap(M)
    llmin, _, cut = _reduce_inputs(ll3, M)
    red = CudaBlockReducer(0)
    ll, yr = CudaSource(ll3).x, CudaSource(yrep3).x
    skip = np.zeros(P, dtype=np.int32)

    def reduce_fit(parts):
        tails, flags, counts = [], [], []
        for lo, hi in parts:
            _, t, f, c = red.loo_pit_reduce(ll[:, :, lo:hi].contiguous(), yr[:, :, lo:hi].contiguous(), llmin, cut, y, cap)
            tails.append(t)
            flags.append(f)
            counts.append(c)
        return red.loo_pit_fit(torch.stack(tails), torch.stack(flags), torch.stack(counts), llmin, cut, skip)

    one, again, split = reduce_fit([(0, chains)]), reduce_fit([(0, chains)]), reduce_fit(ranges)
    assert one.tobytes() == again.tobytes() and one.tobytes() == split.tobytes()
    assert np.all(one[:, 4] <= M) and np.all(one[:, 4] > 4)


def test_device_index_out_of_range_is_refused(gpu_pkg):
    L = gpu_pkg._ffi.lib()
    buf = torch.zeros(64, dtype=torch.float64, device="cuda:0")
    p = buf.data_ptr()
    h = np.zeros(16)
    skip = np.zeros(2, dtype=np.int32)
    for device in (-1, 64):
        assert L.amwg_loo_pit_reduce(device, p, p, 1, 2, 3, h.ctypes.data, h.ctypes.data, h.ctypes.data, 8, p, p, p, h.ctypes.data) != 0
        assert L.amwg_last_error() == b"amwg_loo_pit_reduce: device index out of range"
        assert L.amwg_loo_pit_fit(device, p, p, p, 1, 2, 8, h.ctypes.data, h.ctypes.data, skip.ctypes.data, h.ctypes.data) != 0
        assert L.amwg_last_error() == b"amwg_loo_pit_fit: device index out of range"
    assert np.all(h == 0) and not buf.any()


# ---- config 2 end to end ---------------------------------------------------------------------------------------------------------------
def _twin_sources(s, f, points, rows):
    """the twin's next `rows` sweeps: (device block [rows, entries, chains], the library's ll of f as a CudaPointwise, a function
    giving a fresh CudaPpc of f, family, y)"""
    from bayes_js_b200 import _ffi
    from bayes_js_b200.summary import PPC_FAMILIES, CudaPointwise, CudaPpc
    from bayes_js_b200.tracer import trace_log_lik
    entries = list(range(s.n_comp))
    block = torch.empty((rows, len(entries), s.local_chains), dtype=torch.float64, device="cuda:0")
    mon = np.asarray(entries, dtype=np.int32)
    torch.cuda.synchronize()
    _ffi.check(_ffi.lib().amwg_sample_device(s._handle, rows, 1, mon.ctypes.data_as(C.POINTER(C.c_int32)), len(entries), block.data_ptr()))
    lik = trace_log_lik(f, s.params, s._offsets, s.data, points, what="ppc")
    fam, y, args = lik.observed_call(points)
    start = {name: s._offsets[name] for name in lik.reads}
    prog, offs = lik.lower_exprs(args, start)
    ll_src = CudaPointwise(s._handle, lik.lower(start), block, 0)
    return block, ll_src, (lambda: CudaPpc(s._handle, prog, offs, PPC_FAMILIES.index(fam), block, points)), fam, y


def _pair(gpu_pkg, chains, seed, data, burn=300, post=None, params=None):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = params or {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    post = post or models.norm_post_readme(ld)
    out = [mcmc.AmwgSampler(params, post, data, {"chains": chains, "seed": seed}) for _ in range(2)]
    for s in out:
        s.burn(burn)
    return out


def test_config2_end_to_end(gpu_pkg):
    from bayes_js_b200.summary import CudaBlockReducer, ppc_block
    ld = gpu_pkg.ld
    data = config2_data()
    N, rows, chains = 1024, 8, 4096
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    a, b = _pair(gpu_pkg, chains, 17, data.tolist())
    out = a.sample_summary(rows, probs=(0.05, 0.5, 0.95), ppc={"log_lik": f, "points": N, "loo_pit": True})["ppc"]
    block, ll_src, fresh, fam, y = _twin_sources(b, f, N, rows)
    ll3 = ll_src.chunk(0, N).cpu().numpy()
    yrep3 = fresh().chunk(0, N).cpu().numpy()
    blk = block.cpu().numpy()
    mu, sd = blk[:, 0, None, :], blk[:, 1, None, :]
    numpy_ll = -0.5 * np.log(2 * math.pi) - np.log(sd) - (data[None, :, None] - mu) ** 2 / ((2 * sd) * sd)
    assert np.allclose(ll3, numpy_ll, rtol=1e-13, atol=1e-13)        # the library's ll is the density of the draws
    ref = loo_pit_ref.loo_pit(_flat(ll3), _flat(yrep3), data)
    pit = out["loo_pit"]
    assert_pit_matches(pit, ref)
    assert set(pit) == {"pit", "pit_equal", "pareto_k", "pareto_k_threshold", "n_high_k", "r_eff"} and pit["r_eff"] == 1.0
    assert np.all(pit["pit_equal"] == 0) and np.all(np.isfinite(pit["pareto_k"]))
    # the twin's block in chunks of 1, 7 and all points: the same bytes as sample_summary's
    for chunk in (1, 7, N):
        other = ppc_block(CudaBlockReducer(0), fresh(), rows, chains, N, fam, y, (0.05, 0.5, 0.95), chunk, False, loo_pit=(ll_src, 1.0))
        assert _same(other["loo_pit"], pit), chunk


def test_other_keys_and_the_chains_keep_their_bits(gpu_pkg):
    ld = gpu_pkg.ld
    data = config2_data()[:200].tolist()
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    a, b = _pair(gpu_pkg, 1000, 9, data, burn=500)
    kw = dict(diagnostics=True, histogram=16, covariance=True, loo={"log_lik": f, "points": 200})
    plain = a.sample_summary(20, ppc={"log_lik": f, "points": 200}, **kw)
    with_pit = b.sample_summary(20, ppc={"log_lik": f, "points": 200, "loo_pit": {"r_eff": 0.7}}, **kw)
    assert set(with_pit) == set(plain) and set(with_pit["ppc"]) == set(plain["ppc"]) | {"loo_pit"}
    for key in plain:
        if key == "ppc":
            assert all(_same(plain["ppc"][k], with_pit["ppc"][k]) for k in plain["ppc"])
        else:
            assert _same(plain[key], with_pit[key]), key
    assert _same(a.state, b.state) and _same(a.log_post(), b.log_post())
    assert _same(a.sample_summary(3), b.sample_summary(3))           # the streams too


def test_pareto_k_is_loos(gpu_pkg):
    ld = gpu_pkg.ld
    data = config2_data()[:300].tolist()
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    s, _ = _pair(gpu_pkg, 2048, 5, data)
    out = s.sample_summary(6, loo={"log_lik": f, "points": 300, "r_eff": 0.6}, ppc={"log_lik": f, "points": 300, "loo_pit": {"r_eff": 0.6}})
    k = out["ppc"]["loo_pit"]["pareto_k"]
    assert k.tobytes() == out["loo"]["pointwise"]["pareto_k"].tobytes()
    assert out["ppc"]["loo_pit"]["n_high_k"] == out["loo"]["n_high_k"]
    assert out["ppc"]["loo_pit"]["pareto_k_threshold"] == out["loo"]["pareto_k_threshold"]


# ---- ties of repeated states on the device -------------------------------------------------------------------------------------------------
def test_ties_of_a_poisson_model(gpu_pkg):
    """a Poisson rate: a rejected step repeats the chain's state, so a chain's rows share ll, in and out of the Pareto tail. The
    device's pit equals the restatement, and so does the same block with its chains in reverse order (the tied draws reach the
    tail buffers in another order)"""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    y = np.random.default_rng(61).poisson(3.0, 40).astype(float)

    def post(t, d):
        lp = ld.gamma(t.lam, 2, 1)
        for i in range(len(d)):
            lp += ld.pois(d[i], t.lam)
        return lp
    f = lambda t, d, i: ld.pois(d[i], t.lam)
    s = mcmc.AmwgSampler({"lam": {"type": "real", "lower": 0}}, post, y.tolist(), {"chains": 4096, "seed": 62})
    s.burn(400)
    rows, N = 8, len(y)
    block, ll_src, fresh, fam, yy = _twin_sources(s, f, N, rows)
    ll3, yrep3 = ll_src.chunk(0, N), fresh().chunk(0, N)
    ref = loo_pit_ref.loo_pit(_flat(ll3.cpu().numpy()), _flat(yrep3.cpu().numpy()), y)
    lam = block.cpu().numpy()[:, 0, :]
    assert np.mean(lam[1:] == lam[:-1]) > 0.2                          # many repeated states
    flat = _flat(ll3.cpu().numpy())
    tied = 0
    for i in range(N):
        r = loo_ref.psis_point(flat[:, i])
        v = flat[r["tail"], i]
        tied += len(v) - len(np.unique(v))
    assert tied > 100, tied                                            # tied draws inside the tails
    fwd = _device_pit(ll3, yrep3, y, family="pois")["loo_pit"]
    rev = _device_pit(ll3.flip(2).contiguous(), yrep3.flip(2).contiguous(), y, family="pois")["loo_pit"]
    assert_pit_matches(fwd, ref)
    assert_pit_matches(rev, ref)
    assert np.all(fwd["pit_equal"] > 0)
    assert fwd["pareto_k"].tobytes() == rev["pareto_k"].tobytes()


# ---- calibration ----------------------------------------------------------------------------------------------------------------------------
def test_conjugate_normal_calibration(gpu_pkg):
    """y_i ~ N(mu, sigma) with sigma known and mu ~ N(m0, tau0): the leave-one-out predictive of y_i is N(m_-i, s_-i) in closed
    form. Each pit_i lies within five Monte Carlo standard errors of Phi((y_i - m_-i) / s_-i), the standard error the
    self-normalised importance-sampling one of the same weights and replicated data."""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    sigma, tau0, m0 = 1.5, 10.0, 0.0
    y = np.random.default_rng(43).normal(2.0, sigma, 20)
    y[7] = 6.0                                                       # far out: its leave-one-out predictive differs most

    def post(t, d):
        lp = ld.norm(t.mu, m0, tau0)
        for i in range(len(d)):
            lp += ld.norm(d[i], t.mu, sigma)
        return lp
    f = lambda t, d, i: ld.norm(d[i], t.mu, sigma)
    a = mcmc.AmwgSampler({"mu": {"type": "real"}}, post, y.tolist(), {"chains": 65536, "seed": 4})
    b = mcmc.AmwgSampler({"mu": {"type": "real"}}, post, y.tolist(), {"chains": 65536, "seed": 4})
    a.burn(1500); b.burn(1500)
    N = len(y)
    out = a.sample_summary(1, ppc={"log_lik": f, "points": N, "loo_pit": True})["ppc"]
    pit = out["loo_pit"]["pit"]
    _, ll_src, fresh, _, _ = _twin_sources(b, f, N, 1)
    ll, yrep = _flat(ll_src.chunk(0, N).cpu().numpy()), _flat(fresh().chunk(0, N).cpu().numpy())
    prec = 1 / tau0 ** 2 + (N - 1) / sigma ** 2
    m = (m0 / tau0 ** 2 + (y.sum() - y) / sigma ** 2) / prec
    s = np.sqrt(sigma ** 2 + 1 / prec)
    want = st.norm.cdf((y - m) / s)
    for i in range(N):
        w = np.exp(loo_ref.psis_point(ll[:, i])["lw"])
        h = (yrep[:, i] <= y[i]).astype(float)
        p = np.sum(w * h) / np.sum(w)
        assert abs(p - pit[i]) <= TOL
        se = np.sqrt(np.sum((w / np.sum(w)) ** 2 * (h - p) ** 2))
        assert abs(pit[i] - want[i]) <= 5 * se, (i, pit[i], want[i], se)
    in_sample = out["pointwise"]["pit"]
    assert abs(in_sample[7] - 0.5) < abs(pit[7] - 0.5)               # the outlier: in-sample PIT is pulled towards 0.5


# ---- config 2 at full scale -------------------------------------------------------------------------------------------------------------
def test_config2_at_full_scale_in_forced_chunks(gpu_pkg, monkeypatch):
    """sample_summary(10, ppc={..., "loo_pit": True}) at 2^20 chains and N = 1024, the free memory it sees lowered so that the chunks
    hold 100 points; the twin's ll and y_rep at chosen points against the restatement"""
    import bayes_js_b200.summary as summ
    ld = gpu_pkg.ld
    rows, chains, N, seed = 10, 1 << 20, 1024, 71
    data = config2_data()
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    a, b = _pair(gpu_pkg, chains, seed, data.tolist())
    M = summ.loo_tail_length(rows * chains, 1.0)
    per = summ.ppc_point_bytes(rows, chains) + summ.loo_pit_point_bytes(rows, chains, summ.loo_tail_cap(M), 1)
    need = rows * 2 * chains * 8 + summ.ppc_fixed_bytes(rows, chains) + 2 * 2 * chains * 8
    free = int((need + 100.5 * per) / 0.9)
    real = torch.cuda.mem_get_info
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (min(real(dev)[0], free), real(dev)[1]))
    chunks = []
    inner = summ.ppc_block

    def wrapped(*args, **kw):
        chunks.append(args[8])
        return inner(*args, **kw)
    monkeypatch.setattr(summ, "ppc_block", wrapped)
    out = a.sample_summary(rows, ppc={"log_lik": f, "points": N, "loo_pit": True})["ppc"]
    monkeypatch.undo()
    assert chunks == [100], chunks
    pit = out["loo_pit"]
    assert np.all(np.isfinite(pit["pit"])) and np.all(np.isfinite(pit["pareto_k"]))
    _, ll_src, fresh, _, _ = _twin_sources(b, f, N, rows)
    src = fresh()
    rng = np.random.default_rng(72)
    points = [0, 99, 100, 1023] + sorted(rng.choice(np.arange(101, 1023), 3, replace=False).tolist())
    for i in points:
        ll = ll_src.chunk(i, 1).cpu().numpy().reshape(-1)
        yrep = src.chunk(i, 1).cpu().numpy().reshape(-1)
        p, q, k = loo_pit_ref.point(ll, yrep, data[i])
        assert abs(pit["pit"][i] - p) <= TOL and pit["pit_equal"][i] == q == 0, (i, pit["pit"][i], p)
        assert abs(pit["pareto_k"][i] - k) <= TOL * max(1.0, abs(k)), (i, pit["pareto_k"][i], k)
