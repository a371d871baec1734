"""The device reductions of PSIS-LOO (amwg_loo_reduce, amwg_loo_fit and the shared summary passes) against the numpy restatement
of tests/loo_ref.py: summary.loo_block with CudaBlockReducer on the CPU tier's ll matrices (one case list, test_summary_loo_host.CASES)
and on chain counts of 1, ragged and past the reduce kernel's grid stride, byte-equal over chunk sizes; the fit kernel merging the
tails of 2 and 3 uneven chain ranges as the multi-GPU path gathers them, byte-equal to one range; tails at the limits (S = 10 x 2^20
with a 16384-slot sort, and M = 2^20, the largest tail the API accepts); and config 2 end to end at 2^20 chains and 10 kept rows
with loo= and ppc= together, in forced chunks of 100 points, against the restatements on an identically seeded twin's draws."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import loo_ref
import models
import ppc_ref
from conftest import config2_data
from test_summary_loo_host import CASES, _flat, _normal_ll, assert_matches

pytestmark = pytest.mark.gpu
RTOL = 1e-10                                                       # the config-2 test's tolerance against the restatement


def _reducer():
    from bayes_js_b200.summary import CudaBlockReducer

    class RecordingReducer(CudaBlockReducer):
        """CudaBlockReducer that records every point's tail as the fit kernel receives it (sorted ll, descending)"""

        def __init__(self, device):
            super().__init__(device)
            self.tails = []

        def loo_fit(self, tails, counts, llmin, cut, skip):
            out = super().loo_fit(tails, counts, llmin, cut, skip)
            t, c = tails.cpu().numpy(), counts.cpu().numpy()
            R, P, cap = t.shape
            for p in range(P):
                a = np.concatenate([t[r, p, :min(c[r, p], cap)] for r in range(R)])
                self.tails.append(-np.sort(-a))
            return out
    return RecordingReducer(0)


class CudaSource:
    """an ll block [rows, points, chains] held on the device, handed out in chunks of points"""

    def __init__(self, ll3):
        self.ll = torch.from_numpy(np.ascontiguousarray(ll3, dtype=np.float64)).to("cuda:0")

    def chunk(self, p0, P):
        return self.ll[:, p0:p0 + P, :].contiguous()


def _device_loo(src, rows, chains, points, r_eff, chunk):
    from bayes_js_b200.summary import loo_block
    red = _reducer()
    return loo_block(red, src, rows, chains, points, r_eff, chunk, False), red


def _same(x, y):
    """the same keys and, for numbers, the same bytes"""
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    a, b = np.asarray(x), np.asarray(y)
    if a.dtype.kind in "fiub":
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return x == y


# chain counts the CPU cases do not reach: one chain, and more than the reduce kernel's grid covers in one stride (1184 x 256)
DEVICE_CASES = {
    "one_chain": (lambda: _normal_ll(400, 1, np.random.default_rng(31).normal(0, 1, 5), 32), 1.0),
    "grid_stride": (lambda: _normal_ll(2, 1184 * 256 + 77, np.random.default_rng(33).normal(0, 1, 3), 34), 1.0),
}


@pytest.mark.parametrize("name", list(CASES) + list(DEVICE_CASES))
def test_reducer_equals_the_restatement_on_every_case(gpu_pkg, name):
    build, r_eff = CASES[name] if name in CASES else DEVICE_CASES[name]
    ll3 = build()
    rows, N, chains = ll3.shape
    ll = _flat(ll3)
    ref = loo_ref.loo(ll, r_eff)
    src = CudaSource(ll3)
    out, red = _device_loo(src, rows, chains, N, r_eff, N)
    assert_matches(out, ref, red, ll, rtol=RTOL)
    for chunk in (1, 7):
        other, _ = _device_loo(src, rows, chains, N, r_eff, chunk)
        assert _same(out, other), chunk


# ---- the fit kernel over several chain ranges ----------------------------------------------------------------------------------------
def _placed_block(rows, chains, seed):
    """ll3 [rows, 3, chains]: point 0 holds its smallest values in chains [0, 600), point 1 in chains [4000, 5000), point 2 is
    spread; each point a continuous draw, so its tail is the M smallest"""
    rng = np.random.default_rng(seed)
    ll3 = np.empty((rows, 3, chains))
    for p, (lo, hi) in enumerate([(0, 600), (4000, 5000)]):
        v = np.sort(rng.normal(0.0, 1.0, rows * chains) + rng.standard_t(2, rows * chains) * (p + 1))
        k = rows * (hi - lo)
        inside = v[:k].reshape(rows, hi - lo)
        outside = rng.permutation(v[k:]).reshape(rows, chains - (hi - lo))
        ll3[:, p, lo:hi] = inside
        ll3[:, p, :lo] = outside[:, :lo]
        ll3[:, p, hi:] = outside[:, lo:]
    ll3[:, 2, :] = rng.normal(0.0, 1.0, (rows, chains)) - 0.5 * rng.exponential(1.0, (rows, chains)) ** 2
    return ll3


@pytest.mark.parametrize("ranges", [[(0, 1700), (1700, 5000)], [(0, 900), (900, 3333), (3333, 5000)]])
def test_fit_over_uneven_chain_ranges_equals_one_range(gpu_pkg, ranges):
    """amwg_loo_reduce per chain range, the tails and counts stacked as the multi-GPU path gathers them, one amwg_loo_fit: its
    [P, 4] output is byte-equal to the fit of the whole block in one range (the sort removes the arrival order) and to a repeat
    of it (whose atomic slot order differs). Range 0 holds point 0's whole tail and the last range point 1's; the others none."""
    from bayes_js_b200.summary import LOG_TINY, loo_tail_cap, loo_tail_length
    rows, chains = 2, 5000
    ll3 = _placed_block(rows, chains, 41)
    S, P = rows * chains, 3
    M = loo_tail_length(S, 1.0)
    cap = loo_tail_cap(M)
    flat = _flat(ll3)
    llmin, llmax = flat.min(axis=0), flat.max(axis=0)
    cut = np.maximum(llmin - np.sort(flat, axis=0)[M], LOG_TINY)
    red = _reducer()
    dev = torch.from_numpy(ll3).to("cuda:0")
    skip = np.zeros(P, dtype=np.int32)

    def reduce_fit(parts):
        tails, counts = [], []
        for lo, hi in parts:
            _, t, c = red.loo_reduce(dev[:, :, lo:hi].contiguous(), llmin, llmax, cut, cap)
            tails.append(t)
            counts.append(c)
        return red.loo_fit(torch.stack(tails), torch.stack(counts), llmin, cut, skip), torch.stack(counts).cpu().numpy()

    one, c1 = reduce_fit([(0, chains)])
    again, _ = reduce_fit([(0, chains)])
    split, cs = reduce_fit(ranges)
    assert np.all(c1[0] == M) and np.all(cs.sum(axis=0) == M)
    assert cs[0, 0] == M and np.all(cs[1:, 0] == 0)                  # point 0: all in range 0
    assert cs[-1, 1] == M and np.all(cs[:-1, 1] == 0)                # point 1: all in the last range
    assert np.count_nonzero(cs[:, 2]) == len(ranges)                 # point 2: spread over every range
    assert one.tobytes() == again.tobytes() and one.tobytes() == split.tobytes()
    for p in range(P):
        r = loo_ref.psis_point(flat[:, p])
        assert len(r["tail"]) == M == one[p, 3]
        assert abs(one[p, 0] - r["k"]) <= RTOL * max(1.0, abs(r["k"])), (p, one[p, 0], r["k"])


# ---- tails at the limits -----------------------------------------------------------------------------------------------------------
def test_config2_sized_tail_with_adversarial_points(gpu_pkg):
    """S = 10 x 2^20 (DESIGN.md §4.7's ten kept rows): M = 9715, a 16384-slot sort. Point 0 heavy-tailed (ratios with Pareto
    index 1/0.9), point 1 with its cut at the log DBL_MIN floor, point 2 a tail of 110 tied draws (one candidate b = 0), point 3
    holding a NaN"""
    from bayes_js_b200.summary import loo_tail_cap, loo_tail_length
    rows, chains = 10, 1 << 20
    S = rows * chains
    M = loo_tail_length(S, 1.0)
    assert M == 9715 and loo_tail_cap(M) == 16384
    rng = np.random.default_rng(51)
    ll = np.empty((S, 4))
    ll[:, 0] = 0.9 * np.log(rng.uniform(size=S))
    ll[:, 1] = rng.normal(0.0, 1.0, S)
    ll[rng.choice(S, 5000, replace=False), 1] -= 1000.0               # 5000 <= M draws far below: the cut is log(DBL_MIN)
    ll[:, 2] = np.log(0.8)
    ll[rng.choice(S, 110, replace=False), 2] = np.log(0.2)
    ll[:, 3] = rng.normal(0.0, 1.0, S)
    ll[12345, 3] = np.nan
    ref = loo_ref.loo(ll)
    assert ref["tails"][1].size == 5000 and loo_ref.psis_point(ll[:, 1])["cut"] == loo_ref.LOG_TINY
    assert ref["tails"][2].size == 110
    ll3 = np.ascontiguousarray(ll.reshape(rows, chains, 4).transpose(0, 2, 1))
    out, red = _device_loo(CudaSource(ll3), rows, chains, 4, 1.0, 4)
    del ll3
    assert_matches(out, ref, red, ll, rtol=RTOL)
    k = out["pointwise"]["pareto_k"]
    assert k[0] > 0.7 and np.isfinite(k[1]) and np.isfinite(k[2]) and np.isnan(k[3])
    assert np.isfinite(out["pointwise"]["elpd_loo"][2])


def test_largest_tail_the_api_accepts(gpu_pkg):
    """r_eff chosen so that M = 2^20 exactly at S = 10 x 2^20: the tail fills the fit kernel's 2^20 slots and its 1054 candidates
    fill its shared arrays (kMaxM); against the restatement with its blocked fit"""
    from bayes_js_b200.summary import MAX_LOO_TAIL, loo_tail_cap, loo_tail_length
    rows, chains = 10, 1 << 20
    S = rows * chains
    r_eff = 9.0 * S / (MAX_LOO_TAIL - 0.5) ** 2
    M = loo_tail_length(S, r_eff)
    assert M == MAX_LOO_TAIL == loo_tail_cap(M) and 30 + int(M ** 0.5) == 1054
    rng = np.random.default_rng(53)
    ll = np.empty((S, 2))
    ll[:, 0] = rng.normal(0.0, 1.0, S)
    ll[:, 1] = 0.8 * np.log(rng.uniform(size=S))
    ref = loo_ref.loo(ll, r_eff)
    assert all(t.size == M for t in ref["tails"])
    ll3 = np.ascontiguousarray(ll.reshape(rows, chains, 2).transpose(0, 2, 1))
    out, red = _device_loo(CudaSource(ll3), rows, chains, 2, r_eff, 2)
    del ll3
    assert_matches(out, ref, red, ll, rtol=RTOL)
    assert np.all(np.isfinite(out["pointwise"]["pareto_k"]))


# ---- config 2 end to end at the size DESIGN.md measured ---------------------------------------------------------------------------------
def test_config2_loo_and_ppc_at_full_scale_in_forced_chunks(gpu_pkg, orc, monkeypatch):
    """sample_summary(10, loo=..., ppc=...) at 2^20 chains and N = 1024, the free memory it sees lowered so the LOO chunks hold
    100 points (11 chunks); the twin's draws of the same sweeps give ll (numpy's log) and y_rep at chosen points"""
    import bayes_js_b200.summary as summ
    from bayes_js_b200 import _ffi
    from bayes_js_b200.tracer import trace_log_lik
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    O = orc.lib()
    rows, chains, N, seed = 10, 1 << 20, 1024, 61
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    data = config2_data()
    f = lambda t, d, i: ld.norm(d[i], t.mu, t.sigma)
    a = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data.tolist(), {"chains": chains, "seed": seed})
    b = mcmc.AmwgSampler(params, models.norm_post_readme(ld), data.tolist(), {"chains": chains, "seed": seed})
    a.burn(300); b.burn(300)

    M = summ.loo_tail_length(rows * chains, 1.0)
    per = summ.loo_point_bytes(rows, chains, summ.loo_tail_cap(M), 1)
    need = rows * 2 * chains * 8 + summ.ppc_fixed_bytes(rows, chains) + 2 * 2 * chains * 8
    free = int((need + 100.5 * per) / 0.9)
    real = torch.cuda.mem_get_info
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (min(real(dev)[0], free), real(dev)[1]))
    chunks = {}
    for name in ("loo_block", "ppc_block"):
        inner = getattr(summ, name)

        def wrapped(*args, _inner=inner, _name=name, **kw):
            chunks[_name] = args[-2]
            return _inner(*args, **kw)
        monkeypatch.setattr(summ, name, wrapped)
    out = a.sample_summary(rows, loo={"log_lik": f, "points": N}, ppc={"log_lik": f, "points": N})
    monkeypatch.undo()
    assert chunks["loo_block"] == 100 and 1 < chunks["ppc_block"] < N, chunks
    loo, ppc = out["loo"], out["ppc"]
    assert loo["n_draws"] == ppc["n_draws"] == rows * chains and loo["points"] == ppc["points"] == N

    # the twin: the same sweeps into a device block [rows, (mu, sigma), chains]
    block = torch.empty((rows, 2, chains), dtype=torch.float64, device="cuda:0")
    mon = np.array([0, 1], dtype=np.int32)
    torch.cuda.synchronize()
    _ffi.check(_ffi.lib().amwg_sample_device(b._handle, rows, 1, mon.ctypes.data_as(C.POINTER(C.c_int32)), 2, block.data_ptr()))
    lik = trace_log_lik(f, b.params, b._offsets, b.data, N, what="ppc")
    fam, _, args = lik.observed_call(N)
    prog, offs = lik.lower_exprs(args, {name: b._offsets[name] for name in lik.reads})
    src = summ.CudaPpc(b._handle, prog, offs, summ.PPC_FAMILIES.index(fam), block, N)
    blk = block.cpu().numpy()
    mu, sd = blk[:, 0, :].reshape(-1), blk[:, 1, :].reshape(-1)           # draw s = r * chains + c
    k1 = -0.5 * np.log(2 * math.pi) - np.log(sd)
    k2 = (2 * sd) * sd
    rng = np.random.default_rng(62)
    points = [0, 99, 100, 511, 1023] + sorted(rng.choice(np.arange(1, 1023), 3, replace=False).tolist())
    for i in points:
        dy = data[i] - mu
        ref = loo_ref.loo((k1 - (dy * dy) / k2)[:, None])
        for key, want in ref["pointwise"].items():
            got, w = loo["pointwise"][key][i], want[0]
            tol = RTOL * (max(1.0, abs(w)) if key == "pareto_k" else max(1.0, abs(ref["pointwise"]["lppd"][0])) * 8)
            assert abs(got - w) <= tol, (i, key, got, w)
        yrep = src.chunk(i, 1).cpu().numpy()[:, 0, :]                     # [rows, chains]
        v = yrep.reshape(-1)
        pw = ppc["pointwise"]
        assert pw["n_below"][i] == np.sum(v < data[i]) and pw["n_equal"][i] == np.sum(v == data[i]), i
        assert pw["n_nan"][i] == 0 and pw["pit"][i] == (np.sum(v < data[i]) + np.sum(v == data[i])) / v.size, i
        assert np.isclose(pw["mean"][i], v.mean(), rtol=1e-12) and np.isclose(pw["sd"][i], v.std(ddof=1), rtol=1e-10), i
        for _ in range(375):                                           # 3000 draws over the 8 points, bit for bit
            r, c = int(rng.integers(rows)), int(rng.integers(chains))
            want, _ = ppc_ref.draw_at(O, "norm", (blk[r, 0, c], blk[r, 1, c]), seed, c, r, N, i)
            assert np.float64(yrep[r, c]).tobytes() == np.float64(want).tobytes(), (i, r, c)
