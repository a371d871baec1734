"""Posterior summaries formed on the device (SURVEY 8(f).3): pooled mean / sd, exact quantiles and the Gelman-Rubin
statistic per monitored entry, over all chains and kept rows of one `sample()` block that never leaves HBM.

The reference returns raw draws (mcmc.js:1029) and its README summarises them on the caller's side (README.md:44-52); at
2^20..2^22 chains the raw block is GBs per call, so `AmwgSampler.sample_summary(n)` keeps it on the GPU and moves a few
hundred bytes instead. Multi-GPU (one process per GPU): every rank reduces its own shard, and the functions under "combining
shards" below (gather, gather_tensor, sum_counts, merged_extremes, pooled_moment_record) are the only code here that combines
shards, so every rank returns the same numbers as a single GPU holding all chains.

Host logic here is plain numpy (tested on CPU); the device work is behind `CudaBlockReducer` (C ABI: amwg_summary_moments,
amwg_summary_digit_hist, amwg_summary_autocov for the split-chain ESS / MCSE / R-hat of diagnostics=True, and
amwg_summary_rank_sort / _rank_count / _rank_z for the rank-normalised R-hat and bulk ESS of diagnostics="rank", and
amwg_summary_finite_range / _histogram / _histogram2d for the posterior histograms of histogram=..., amwg_summary_comoments for
the posterior covariance of covariance=..., and amwg_summary_nested for the nested R-hat of nested=...). There is no CPU fallback:
without the library or a GPU the reducer raises. Every reducer call first waits for torch's current stream, which wrote its
inputs. The library's summary calls take their device scratch from one pool per device, grown on demand and held by each call
until it returns; the memory checks add up the calls' requests, which bounds that pool from above.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

MAX_PREFIXES = 32                      # include/amwg.h: n_prefix <= 32
_SIGN = np.uint64(1 << 63)


# ---------------------------------------------------------------------------------------------------------------------
# moments
def merge_moment_records(records: Sequence[np.ndarray]) -> np.ndarray:
    """Chan merge of per-shard records [entries, 4] = (chains, mean of chain means, M2 of chain means, sum of within-chain M2),
    in the order given (rank order): the same arithmetic as the device tree, so shards combine exactly."""
    acc = np.array(records[0], dtype=np.float64, copy=True)
    for rec in records[1:]:
        b = np.asarray(rec, dtype=np.float64)
        n = acc[:, 0] + b[:, 0]
        d = b[:, 1] - acc[:, 1]
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = np.where(b[:, 0] == 0, acc[:, 1], np.where(acc[:, 0] == 0, b[:, 1], acc[:, 1] + d * (b[:, 0] / n)))
            m2 = np.where(b[:, 0] == 0, acc[:, 2], np.where(acc[:, 0] == 0, b[:, 2], acc[:, 2] + b[:, 2] + d * d * (acc[:, 0] * b[:, 0] / n)))
        acc = np.stack([n, mean, m2, acc[:, 3] + b[:, 3]], axis=1)
    return acc


def finalize_moments(rec: np.ndarray, rows: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(mean, sd, rhat) per entry from the merged record. sd: pooled over all rows*chains draws, ddof=1. rhat: Gelman-Rubin
    potential scale reduction sqrt(((n-1)/n W + B/n) / W) with n = rows, W the mean within-chain variance, B/n the variance of
    the chain means. NaN with fewer than 2 rows or chains, or when W = 0 and B = 0: an entry whose draws all equal one value,
    whose chain means are that value exactly (run_mean, csrc/amwg_nested.cuh), so its sd is 0. +inf when W = 0 < B: every chain
    stuck at a value of its own."""
    G, mean, b2, sw = rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3]
    M = G * rows
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = np.sqrt((sw + rows * b2) / (M - 1))
        W = sw / (G * (rows - 1))
        varplus = (rows - 1) / rows * W + b2 / (G - 1)
        rhat = np.sqrt(varplus / W)
    return mean, sd, rhat


# ---------------------------------------------------------------------------------------------------------------------
# exact quantiles: MSD radix select on the order-preserving key of an IEEE double
def key_to_double(keys: np.ndarray) -> np.ndarray:
    k = np.asarray(keys, dtype=np.uint64)
    u = np.where((k & _SIGN) != 0, k ^ _SIGN, ~k)
    return u.view(np.float64) if u.ndim else np.array([u], dtype=np.uint64).view(np.float64)[0]


def double_to_key(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    return np.where((u & _SIGN) != 0, ~u, u | _SIGN)


def quantile_targets(M: int, probs: Sequence[float]):
    """numpy.quantile's default (linear) rule: position p*(M-1) between order statistics lo and lo+1.
    Returns (sorted distinct 0-based ranks, per-prob (index of lo, index of hi, fraction))."""
    ranks: List[int] = []
    plan = []
    for p in probs:
        if not (0.0 <= p <= 1.0):
            raise ValueError("probs must be in [0, 1]")
        pos = p * (M - 1)
        lo = int(np.floor(pos))
        hi = min(lo + 1, M - 1)
        plan.append((lo, hi, pos - lo))
        ranks += [lo, hi]
    uniq = sorted(set(ranks))
    index = {r: i for i, r in enumerate(uniq)}
    return np.asarray(uniq, dtype=np.int64), [(index[lo], index[hi], g) for lo, hi, g in plan]


def _lerp(a, b, t):
    """numpy's _lerp (lib/_function_base_impl.py): a + (b-a)*t, computed from b when t >= 0.5."""
    d = b - a
    return np.where(t >= 0.5, b - d * (1 - t), a + d * t)


class RadixSelect:
    """Host side of the 8-pass select: which prefixes the device should histogram next, and how the summed counts narrow
    each wanted order statistic down by one byte. ranks: sorted 0-based ranks [T], shared by all entries, or [entries, T], each
    entry's own (mcse_quantile's ranks depend on each entry's ESS); at most MAX_PREFIXES distinct ranks per entry."""

    def __init__(self, entries: int, ranks: np.ndarray):
        r = np.asarray(ranks, dtype=np.int64)
        self.E = entries
        self.T = r.shape[-1]
        self.prefix = np.zeros((entries, self.T), dtype=np.uint64)
        self.rem = np.tile(r, (entries, 1)) if r.ndim == 1 else np.array(r.reshape(entries, self.T), copy=True)
        self.npass = 0

    def prefixes(self) -> Tuple[np.ndarray, np.ndarray]:
        """([entries, n_prefix] uint64 distinct prefixes padded with repeats, [entries, T] index of each target's prefix)."""
        uniq = [np.unique(self.prefix[e]) for e in range(self.E)]
        n = max(len(u) for u in uniq)
        if n > MAX_PREFIXES:
            raise ValueError("too many quantiles at once: %d distinct order statistics (max %d)" % (n, MAX_PREFIXES))
        table = np.empty((self.E, n), dtype=np.uint64)
        which = np.empty((self.E, self.T), dtype=np.int64)
        for e, u in enumerate(uniq):
            table[e, :len(u)] = u
            table[e, len(u):] = u[0]
            which[e] = np.searchsorted(u, self.prefix[e])
        return table, which

    def advance(self, counts: np.ndarray, which: np.ndarray) -> None:
        """counts [entries, n_prefix, 256] summed over all shards for the prefixes handed out by prefixes()."""
        sel = np.take_along_axis(np.asarray(counts, dtype=np.int64), which[:, :, None], axis=1)      # [E, T, 256]: each target's histogram
        cum = np.cumsum(sel, axis=2)
        d = (cum <= self.rem[:, :, None]).sum(axis=2)                                             # first byte whose cumulative count exceeds the rank
        if np.any(d > 255):
            raise RuntimeError("radix select: rank beyond the counted values (inconsistent histogram)")
        below = np.take_along_axis(cum, np.maximum(d - 1, 0)[:, :, None], axis=2)[:, :, 0]
        self.rem = self.rem - np.where(d > 0, below, 0)
        self.prefix = (self.prefix << np.uint64(8)) | d.astype(np.uint64)
        self.npass += 1

    def values(self) -> np.ndarray:
        assert self.npass == 8
        return key_to_double(self.prefix)


# ---------------------------------------------------------------------------------------------------------------------
# combining shards: every rank ends with the same bits. Records are gathered and merged in rank order, integer counts are
# summed, extremes are taken as the maximum of order-preserving keys. The collectives run on the device of the tensor they are
# given (NCCL for CUDA tensors, gloo for the CPU stand-in of the tests); with distributed=False each function is the identity.
def gather_tensor(t, distributed: bool):
    """This rank's tensor -> [world, *t.shape] in rank order ([1, *t.shape] when not distributed), on t's device."""
    if not distributed:
        return t[None]
    import torch
    import torch.distributed as dist
    ws = dist.get_world_size()
    out = torch.empty((ws * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous())
    return out.reshape((ws,) + tuple(t.shape))


def gather(rec: np.ndarray, like, distributed: bool) -> np.ndarray:
    """This rank's numpy record -> [world, *rec.shape] in rank order ([1, *rec.shape] when not distributed); it travels on
    `like`'s device."""
    rec = np.ascontiguousarray(rec)
    if not distributed:
        return rec[None]
    import torch
    return gather_tensor(torch.from_numpy(rec).to(like.device), True).cpu().numpy()


def sum_counts(t, distributed: bool):
    """In-place SUM all-reduce of an integer tensor: exact, independent of the number of GPUs. -> t"""
    if distributed:
        import torch.distributed as dist
        dist.all_reduce(t)
    return t


def merged_extremes(rng: np.ndarray, like, distributed: bool) -> np.ndarray:
    """This rank's [entries, 2] (smallest, largest) -> the smallest and the largest over all ranks: one MAX all-reduce of
    [-key(smallest), key(largest)], the keys of double_to_key as signed integers, on `like`'s device."""
    if not distributed:
        return rng
    import torch
    import torch.distributed as dist
    k = (double_to_key(rng) ^ _SIGN).view(np.int64)
    t = torch.from_numpy(np.concatenate([-k[:, 0], k[:, 1]])).to(like.device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    k = t.cpu().numpy()
    return key_to_double(np.stack([-k[:len(rng)], k[len(rng):]], axis=1).view(np.uint64) ^ _SIGN)


def pooled_moment_record(reducer, block, distributed: bool) -> np.ndarray:
    """reducer.moments of every shard, merged in rank order (merge_moment_records)."""
    return merge_moment_records(gather(reducer.moments(block), block, distributed))


# ---------------------------------------------------------------------------------------------------------------------
class CudaBlockReducer:
    """The device reductions over a torch CUDA tensor block[rows, entries, chains] (fp64, contiguous)."""

    def __init__(self, device: int):
        from . import _ffi
        self.L = _ffi.lib()                       # raises when the extension is missing: no CPU fallback
        self._ffi = _ffi
        self.device = device

    def _call(self, t, fn, *args) -> None:
        """fn(device, *args), an ABI call on the library's default stream, once torch's current stream on t's device has finished
        writing the tensors it reads (the caller's stream need not be the default one)."""
        import torch
        torch.cuda.current_stream(t.device).synchronize()
        self._ffi.check(fn(self.device, *args))

    def moments(self, block) -> np.ndarray:
        rows, entries, chains = block.shape
        out = np.empty((entries, 4), dtype=np.float64)
        self._call(block, self.L.amwg_summary_moments, block.data_ptr(), rows, entries, chains, out.ctypes.data)
        return out

    def digit_counts(self, block, npass: int, prefix_table: np.ndarray):
        """-> torch int64 CUDA tensor [entries, n_prefix, 256] (this shard's counts)."""
        import torch
        rows, entries, chains = block.shape
        n_prefix = prefix_table.shape[1]
        dev = block.device
        pre = torch.from_numpy(prefix_table.view(np.int64).copy()).to(dev)
        counts = torch.zeros((entries, n_prefix, 256), dtype=torch.int64, device=dev)
        self._call(block, self.L.amwg_summary_digit_hist, block.data_ptr(), rows, entries, chains, npass, pre.data_ptr(), n_prefix,
                   counts.data_ptr())
        return counts

    def autocov(self, block, thresholds, lag0: int, n_lags: int) -> np.ndarray:
        """-> [entries, series, 4 + n_lags] split-chain records and lag sums of this shard (series: 1, or 3 with thresholds
        [entries, 2]); see amwg_summary_autocov in include/amwg.h."""
        rows, entries, chains = block.shape
        ns = 1 if thresholds is None else 3
        out = np.empty((entries, ns, 4 + n_lags), dtype=np.float64)
        thr = None if thresholds is None else np.ascontiguousarray(thresholds, dtype=np.float64).reshape(entries, 2)
        self._call(block, self.L.amwg_summary_autocov, block.data_ptr(), rows, entries, chains, None if thr is None else thr.ctypes.data,
                   lag0, n_lags, out.ctypes.data)
        return out

    def autocov_sq(self, block, centre, scale, lag0: int, n_lags: int) -> np.ndarray:
        """-> [entries, 1, 4 + n_lags]: autocov's draws record of y = ((x - centre[e]) * scale[e])^2 for this shard; see
        amwg_summary_autocov_sq in include/amwg.h."""
        rows, entries, chains = block.shape
        out = np.empty((entries, 1, 4 + n_lags), dtype=np.float64)
        c = np.ascontiguousarray(centre, dtype=np.float64)
        s = np.ascontiguousarray(scale, dtype=np.float64)
        self._call(block, self.L.amwg_summary_autocov_sq, block.data_ptr(), rows, entries, chains, c.ctypes.data, s.ctypes.data, lag0,
                   n_lags, out.ctypes.data)
        return out

    def indicator_autocov(self, block, thresholds, lag0: int, n_lags: int) -> np.ndarray:
        """-> int64 [entries, K, 2 + 2 n_lags] = {C1, C2, P_t..., G_t...} of the indicators 1[x <= thresholds[e][k]] (thresholds
        [entries, K], K <= 16, n_lags <= 64) for this shard; see amwg_summary_indicator_autocov in include/amwg.h."""
        rows, entries, chains = block.shape
        thr = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(entries, -1)
        out = np.empty((entries, thr.shape[1], 2 + 2 * n_lags), dtype=np.int64)
        self._call(block, self.L.amwg_summary_indicator_autocov, block.data_ptr(), rows, entries, chains, thr.ctypes.data, thr.shape[1],
                   lag0, n_lags, out.ctypes.data)
        return out

    def rank_sort(self, block, entry: int, centre: float, keys, index) -> int:
        """Sorts the half-chain keys of `entry` (centre NaN: the draws; else |x - centre|) into keys[:n] (int64 tensor holding the
        uint64 keys, 2n long) with their positions in index[:n] (int32 tensor, 2n long); -> radix passes run. See
        amwg_summary_rank_sort in include/amwg.h."""
        rows, entries, chains = block.shape
        passes = C.c_int32(0)
        self._call(block, self.L.amwg_summary_rank_sort, block.data_ptr(), rows, entries, chains, entry, centre, keys.data_ptr(),
                   index.data_ptr(), C.byref(passes))
        return passes.value

    def rank_count(self, q, nq: int, r, nr: int, acc) -> None:
        """acc[:nq] += #(r[:nr] < q[i]) + #(r[:nr] <= q[i]) for sorted key tensors q and r."""
        self._call(acc, self.L.amwg_summary_rank_count, q.data_ptr(), nq, r.data_ptr(), nr, acc.data_ptr())

    def rank_z(self, acc, index, n: int, total: int, z) -> None:
        """z.view(-1)[index[i]] = Phi^-1(((acc[i] + 1) / 2 - 3/8) / (total + 1/4)) for i < n."""
        self._call(acc, self.L.amwg_summary_rank_z, acc.data_ptr(), index.data_ptr(), n, total, z.data_ptr())

    def finite_range(self, block):
        """-> (float64 tensor [entries, 2]: smallest and largest finite draw, +inf / -inf when there is none; int64 tensor
        [entries, 3]: the counts of -inf, +inf and NaN draws), this shard's, on the block's device."""
        import torch
        rows, entries, chains = block.shape
        rng = torch.empty((entries, 2), dtype=torch.float64, device=block.device)
        nonfinite = torch.empty((entries, 3), dtype=torch.int64, device=block.device)
        self._call(block, self.L.amwg_summary_finite_range, block.data_ptr(), rows, entries, chains, rng.data_ptr(), nonfinite.data_ptr())
        return rng, nonfinite

    def histogram(self, block, edges: np.ndarray, bins: int):
        """-> int64 tensor [entries, bins + 3]: this shard's counts per bin over edges [entries, bins + 1], then below, above, NaN."""
        import torch
        rows, entries, chains = block.shape
        ed = torch.from_numpy(np.ascontiguousarray(edges, dtype=np.float64)).to(block.device)
        counts = torch.zeros((entries, bins + 3), dtype=torch.int64, device=block.device)
        self._call(block, self.L.amwg_summary_histogram, block.data_ptr(), rows, entries, chains, ed.data_ptr(), bins, counts.data_ptr())
        return counts

    def histogram2d(self, block, pairs: np.ndarray, edges: np.ndarray, bins: int):
        """-> int64 tensor [n_pairs, bins, bins]: this shard's 2-D counts of the entry pairs [n_pairs, 2] over edges [entries, bins + 1]."""
        import torch
        rows, entries, chains = block.shape
        pr = np.ascontiguousarray(pairs, dtype=np.int32)
        ed = torch.from_numpy(np.ascontiguousarray(edges, dtype=np.float64)).to(block.device)
        counts = torch.zeros((len(pr), bins, bins), dtype=torch.int64, device=block.device)
        self._call(block, self.L.amwg_summary_histogram2d, block.data_ptr(), rows, entries, chains, pr.ctypes.data, len(pr), ed.data_ptr(),
                   bins, counts.data_ptr())
        return counts

    def comoments(self, block, sel) -> np.ndarray:
        """-> flat record [1 + n + 2 n^2] {chains, m[n], B[n][n], W[n][n]} of the n selected entries of this shard; see
        amwg_summary_comoments in include/amwg.h."""
        rows, entries, chains = block.shape
        s = np.ascontiguousarray(sel, dtype=np.int32)
        n = len(s)
        out = np.empty(1 + n + 2 * n * n, dtype=np.float64)
        self._call(block, self.L.amwg_summary_comoments, block.data_ptr(), rows, entries, chains, s.ctypes.data, n, out.ctypes.data)
        return out

    def nested(self, block, first_chain: int, superchain_size: int) -> np.ndarray:
        """-> [entries, 14]: this shard's complete-superchain record and its two cut records; see amwg_summary_nested in
        include/amwg.h."""
        rows, entries, chains = block.shape
        out = np.empty((entries, NESTED_RECORD), dtype=np.float64)
        self._call(block, self.L.amwg_summary_nested, block.data_ptr(), rows, entries, chains, first_chain, superchain_size,
                   out.ctypes.data)
        return out

    def threshold_counts(self, block, thresholds):
        """-> torch int64 CUDA tensor [entries, 4]: this shard's draws <, ==, > thresholds[entry] and NaN (amwg_summary_threshold_counts)"""
        import torch
        rows, entries, chains = block.shape
        out = torch.empty((entries, 4), dtype=torch.int64, device=block.device)
        thr = np.ascontiguousarray(thresholds, dtype=np.float64)
        self._call(block, self.L.amwg_summary_threshold_counts, block.data_ptr(), rows, entries, chains, thr.ctypes.data, out.data_ptr())
        return out

    def loo_reduce(self, ll, llmin, llmax, cut, cap: int):
        """-> (sums [P, 3], tails float64 tensor [P, cap], counts int32 tensor [P]) of this shard; see amwg_loo_reduce in include/amwg.h."""
        import torch
        rows, P, chains = ll.shape
        tails = torch.empty((P, cap), dtype=torch.float64, device=ll.device)
        counts = torch.zeros(P, dtype=torch.int32, device=ll.device)
        sums = np.empty((P, 3), dtype=np.float64)
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        mn, mx, ct = f(llmin), f(llmax), f(cut)
        self._call(ll, self.L.amwg_loo_reduce, ll.data_ptr(), rows, P, chains, mn.ctypes.data, mx.ctypes.data, ct.ctypes.data, cap,
                   tails.data_ptr(), counts.data_ptr(), sums.ctypes.data)
        return sums, tails, counts

    def loo_fit(self, tails, counts, llmin, cut, skip) -> np.ndarray:
        """tails [shards, P, cap], counts int32 [shards, P] (device) -> [P, 4]; see amwg_loo_fit in include/amwg.h."""
        shards, P, cap = tails.shape
        out = np.empty((P, 4), dtype=np.float64)
        mn, ct = np.ascontiguousarray(llmin, dtype=np.float64), np.ascontiguousarray(cut, dtype=np.float64)
        sk = np.ascontiguousarray(skip, dtype=np.int32)
        self._call(tails, self.L.amwg_loo_fit, tails.data_ptr(), counts.data_ptr(), shards, P, cap, mn.ctypes.data, ct.ctypes.data,
                   sk.ctypes.data, out.ctypes.data)
        return out

    def loo_pit_reduce(self, ll, yrep, llmin, cut, y, cap: int):
        """-> (sums [P, 3], tails float64 tensor [P, cap], flags uint8 tensor [P, cap], counts int32 tensor [P]) of this shard; see
        amwg_loo_pit_reduce in include/amwg.h."""
        import torch
        rows, P, chains = ll.shape
        assert tuple(yrep.shape) == tuple(ll.shape)
        tails = torch.empty((P, cap), dtype=torch.float64, device=ll.device)
        flags = torch.empty((P, cap), dtype=torch.uint8, device=ll.device)
        counts = torch.zeros(P, dtype=torch.int32, device=ll.device)
        sums = np.empty((P, 3), dtype=np.float64)
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        mn, ct, yy = f(llmin), f(cut), f(y)
        self._call(ll, self.L.amwg_loo_pit_reduce, ll.data_ptr(), yrep.data_ptr(), rows, P, chains, mn.ctypes.data, ct.ctypes.data,
                   yy.ctypes.data, cap, tails.data_ptr(), flags.data_ptr(), counts.data_ptr(), sums.ctypes.data)
        return sums, tails, flags, counts

    def loo_pit_fit(self, tails, flags, counts, llmin, cut, skip) -> np.ndarray:
        """tails [shards, P, cap], flags uint8 [shards, P, cap], counts int32 [shards, P] (device) -> [P, 5]; see amwg_loo_pit_fit in
        include/amwg.h."""
        shards, P, cap = tails.shape
        out = np.empty((P, 5), dtype=np.float64)
        mn, ct = np.ascontiguousarray(llmin, dtype=np.float64), np.ascontiguousarray(cut, dtype=np.float64)
        sk = np.ascontiguousarray(skip, dtype=np.int32)
        self._call(tails, self.L.amwg_loo_pit_fit, tails.data_ptr(), flags.data_ptr(), counts.data_ptr(), shards, P, cap, mn.ctypes.data,
                   ct.ctypes.data, sk.ctypes.data, out.ctypes.data)
        return out


# ---------------------------------------------------------------------------------------------------------------------
# split-chain effective sample size (Vehtari et al. 2021, §3; Stan's `ess` on split chains, ArviZ's method="mean"/"tail")
MAX_LAGS = 32                          # include/amwg.h: n_lags <= 32 per amwg_summary_autocov call
MIN_ROWS = 10                          # h = rows // 2 >= 5: Geyer's sequence can take at least one pair step


def merge_autocov_records(records: Sequence[np.ndarray]) -> np.ndarray:
    """Per-shard [entries, series, 4 + n] records in rank order -> one: moment part by merge_moment_records, lag sums added in
    the order given."""
    first = np.asarray(records[0], dtype=np.float64)
    E, S, W = first.shape
    mom = merge_moment_records([np.asarray(r, dtype=np.float64)[:, :, :4].reshape(E * S, 4) for r in records]).reshape(E, S, 4)
    sums = np.array(first[:, :, 4:], copy=True)
    for r in records[1:]:
        sums = sums + np.asarray(r, dtype=np.float64)[:, :, 4:]
    return np.concatenate([mom, sums], axis=2)


class GeyerESS:
    """ESS of one series from its merged split-chain record, one lag window at a time. Geyer's initial positive sequence and
    then the initial monotone sequence, exactly as written in the docstring of `split_chain_diagnostics`; NaN at once when W is 0
    or not finite (the caller settles constant series before). `need()` is the first
    lag it has not got yet (None once done); `add(sums)` appends the lag sums of the next window."""

    def __init__(self, record: np.ndarray, h: int):
        self.record = np.asarray(record[:4], dtype=np.float64)
        M, _mean, m2, sum_w = self.record                              # numpy scalars: 0/0 is NaN, not an exception
        self.h, self.M = h, M
        with np.errstate(invalid="ignore", divide="ignore"):
            self.W = sum_w / (M * (h - 1))                        # h/(h-1) * mean_m acov_m(0)
            B = m2 / (M - 1)                                      # variance (ddof 1) of the half-chain means
            self.varplus = (h - 1) / h * self.W + B
        self.rho: List[float] = []
        self.r = [1.0, 0.0]
        self.ev, self.od, self.t = 1.0, None, 1
        self.ess = None

    def _rho(self, sums: np.ndarray) -> np.ndarray:
        with np.errstate(invalid="ignore", divide="ignore"):
            return 1.0 - (self.W - np.asarray(sums, dtype=np.float64) / (self.M * self.h)) / self.varplus

    def need(self):
        return None if self.ess is not None else len(self.rho)

    def add(self, sums: np.ndarray) -> None:
        self.rho.extend(float(v) for v in self._rho(sums))
        self._run()

    def _run(self) -> None:
        h, rho, r = self.h, self.rho, self.r
        if not (0.0 < self.W < np.inf):
            self.ess = np.nan                                     # no within-chain spread to measure (or its sums overflowed)
            return
        if self.od is None:
            if len(rho) < 2:
                return
            self.od = rho[1]
            r[1] = self.od
        while self.t < h - 3 and self.ev + self.od > 0:
            if self.t + 2 >= len(rho):
                return                                            # the next pair is in the next lag window
            ev, od = rho[self.t + 1], rho[self.t + 2]
            self.ev, self.od = ev, od
            r.extend([0.0] * (self.t + 3 - len(r)))
            if ev + od >= 0:
                r[self.t + 1], r[self.t + 2] = ev, od
            self.t += 2
        max_t = self.t - 2
        r.extend([0.0] * (max_t + 2 - len(r)))
        if self.ev > 0:
            r[max_t + 1] = self.ev
        t = 1
        while t <= max_t - 2:
            if r[t + 1] + r[t + 2] > r[t - 1] + r[t]:
                r[t + 1] = r[t + 2] = (r[t - 1] + r[t]) / 2
            t += 2
        Mh = self.M * h
        tau = -1.0 + 2.0 * sum(r[:max_t + 1]) + r[max_t + 1]
        tau = max(tau, 1.0 / np.log10(Mh))
        self.ess = Mh / tau


def split_chain_diagnostics(reducer, block, rows: int, sd: np.ndarray, lo: np.ndarray, hi: np.ndarray, vmin: np.ndarray,
                            vmax: np.ndarray, distributed: bool, max_lags: int = MAX_LAGS):
    """-> ({"ess_mean", "ess_tail", "mcse_mean", "rhat_split"} per entry, number of lag windows used).

    Every chain is split into rows [0, h) and [rows-h, rows), h = rows // 2 (for odd rows the middle row is in neither half):
    M = 2 * chains half-chains of h draws. For a series y, with acov_m(t) = (1/h) sum_{n<h-t} (y_mn - ybar_m)(y_m,n+t - ybar_m):
    W = h/(h-1) mean_m acov_m(0), B = variance (ddof 1) of the ybar_m, var+ = (h-1)/h W + B, rho(t) = 1 - (W - mean_m acov_m(t)) / var+.
    Geyer's initial positive sequence, then the initial monotone sequence, give tau; tau = max(tau, 1/log10(M h)); ESS = M h / tau.
      ess_mean   ESS of the draws
      ess_tail   min of the ESS of 1[x <= q05] and of 1[x <= q95] (lo, hi: the pooled exact quantiles; ties count as <=)
      mcse_mean  sd / sqrt(ess_mean), sd the pooled sd
      rhat_split sqrt(var+ / W) of the draws (not rank-normalised)
    The device scales the draws series by a power of two taken from q95/2 - q05/2 (autocov_scale in csrc/amwg_autocov.cuh; 1 when
    q05 == q95), applied to the centred values and the half-chain means alike. Scaling by a power of two is exact, and every value
    above is a ratio of these sums, so draws x and x * 2^j give the same bits of ess_mean, ess_tail and rhat_split while the
    scaled values stay normal: tiny or huge draws (1e-170, 1e160) neither underflow nor overflow their squares. The scale leaves
    about 2^511 of headroom between that spread and the largest |x - mean|: draws with a narrow centre and far outliers (spread
    1e-10, outliers near 1e150) overflow once scaled and give NaN where the unscaled squares were finite.
    Edge cases: fewer than 10 rows (h < 5): all NaN. A constant entry (vmin == vmax) has ESS = M h, MCSE 0 and rhat_split NaN
    (its half-chains are centred on their value, so W = 0 and B = 0); half-chains each constant at a value of their own give
    rhat_split +inf and ESS NaN. An indicator that is constant (all 1 when the quantile equals the maximum) has ESS = M h. Any other
    series whose W is 0 or not finite (its sums underflowed or overflowed) has ESS NaN, never a finite value, and ess_tail is NaN
    when either indicator's ESS is. A non-finite minimum or maximum (an infinite or NaN draw) makes all four values NaN.
    The lag windows are those of `geyer_windows`."""
    entries = block.shape[1]
    h = rows // 2
    nan = np.full(entries, np.nan)
    out = {"ess_mean": nan.copy(), "ess_tail": nan.copy(), "mcse_mean": nan.copy(), "rhat_split": nan.copy()}
    if rows < MIN_ROWS:
        return out, 0
    thr = np.stack([np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)], axis=1)
    est, windows = geyer_windows(reducer, block, thr, h, distributed, max_lags)
    Mh = est[0][0].M * h
    finite = np.isfinite(np.asarray(vmin, dtype=np.float64)) & np.isfinite(np.asarray(vmax, dtype=np.float64))
    for e in range(entries):
        if not finite[e]:
            continue
        const = (vmin[e] == vmax[e], thr[e, 0] >= vmax[e] or thr[e, 0] < vmin[e], thr[e, 1] >= vmax[e] or thr[e, 1] < vmin[e])
        ess = [Mh if c else g.ess for g, c in zip(est[e], const)]
        out["ess_mean"][e] = ess[0]
        out["ess_tail"][e] = np.minimum(ess[1], ess[2])
        with np.errstate(invalid="ignore", divide="ignore"):
            out["mcse_mean"][e] = 0.0 if vmin[e] == vmax[e] else sd[e] / np.sqrt(ess[0])
            out["rhat_split"][e] = np.sqrt(est[e][0].varplus / est[e][0].W)
    return out, windows


def autocov_record(reducer, block, thresholds, lag0: int, n_lags: int, distributed: bool) -> np.ndarray:
    """reducer.autocov of every shard, merged in rank order (merge_autocov_records)."""
    return merge_autocov_records(gather(reducer.autocov(block, thresholds, lag0, n_lags), block, distributed))


def geyer_windows(reducer, block, thresholds, h: int, distributed: bool, max_lags: int = MAX_LAGS):
    """-> (the GeyerESS of every entry and series of reducer.autocov(block, thresholds, ...) [entries][series], the number of
    lag windows used), by geyer_loop over autocov_record."""
    return geyer_loop(lambda lag0, n_lags: autocov_record(reducer, block, thresholds, lag0, n_lags, distributed), h, max_lags)


def geyer_loop(fetch, h: int, max_lags: int):
    """-> (the GeyerESS of every entry and series of the merged records fetch(lag0, n_lags) -> [entries, series, 4 + n_lags],
    the number of lag windows used). The first window holds lags [0, min(max_lags, h)); the next window of at most `max_lags`
    consecutive lags is asked for only while some estimator still needs a lag it has not got, the way RadixSelect asks for its
    next pass."""
    est: Optional[List[List[GeyerESS]]] = None
    windows = lag0 = 0
    while est is None or (lag0 < h and any(g.need() is not None for row in est for g in row)):
        n_lags = min(max_lags, h - lag0)
        rec = fetch(lag0, n_lags)
        if est is None:
            est = [[GeyerESS(r, h) for r in series] for series in rec]
        for row, series in zip(est, rec):
            for g, r in zip(row, series):
                if g.need() is not None:
                    g.add(r[4:])
        lag0 += n_lags
        windows += 1
    return est, windows


# ---------------------------------------------------------------------------------------------------------------------
# rank-normalised split R-hat and bulk ESS (Vehtari et al. 2021, §4; what Stan, ArviZ and posterior print by default)
def rank_diagnostics(reducer, block, rows: int, med: np.ndarray, vmin: np.ndarray, vmax: np.ndarray, distributed: bool,
                     max_lags: int = MAX_LAGS) -> dict:
    """-> {"ess_bulk", "rhat_rank"} per entry; vmin / vmax are the exact smallest and largest kept draws (a NaN draw makes one
    of them NaN: its key lies below -inf's or above +inf's).

    The halves are those of `split_chain_diagnostics`: h = rows // 2, rows [0, h) and [rows-h, rows) of every chain (for odd
    rows the middle row is in neither half and is not ranked). S = 2 h * (chains over all GPUs) draws per entry are ranked
    together. r(x) is the average rank of x among them (1-based, ties averaged, as scipy.stats.rankdata(method="average")),
    with -0.0 and +0.0 equal, and z = Phi^-1((r - 3/8) / (S + 1/4)). The folded draws f = |x - med|, med the pooled exact 0.5
    quantile over all kept rows (numpy.quantile's rule), are ranked and z-scaled the same way into z_f.
      ess_bulk   the ESS of z, by the estimator of `split_chain_diagnostics` (Geyer's initial positive, then initial monotone
                 sequence over the split-chain autocorrelations of z)
      rhat_rank  max(sqrt(var+ / W) of z, sqrt(var+ / W) of z_f), var+ and W as in `split_chain_diagnostics`
    Edge cases: fewer than 10 rows: NaN. A NaN draw anywhere in the kept rows (vmin or vmax NaN): both NaN. +-inf draws are
    ranked like any other value, so both stay finite. A constant entry (all ranked draws equal): ess_bulk = M h (M = 2 * chains),
    rhat_rank NaN. A constant folded series (for example draws +-1 with median 0): rhat_rank is the R-hat of z alone. med not
    finite (+-inf, or NaN when numpy.quantile's rule interpolates towards an infinite draw): rhat_rank NaN. Half-chains each
    constant at a value of their own (W = 0 for z): ess_bulk NaN (GeyerESS) and rhat_rank +inf.
    Device work per entry and series (CudaBlockReducer): a radix sort of the shard's keys, rank counts against every shard's
    sorted keys, and z written into a [2h][1][chains] block that amwg_summary_autocov splits into exactly the ranked halves.
    Distributed: the sorted key arrays travel around a ring of torch.distributed send / recv (W - 1 steps, two buffers,
    `_ring_counts`); the counts are integers, so the ranks and z do not depend on the number of GPUs. The shard sizes and the
    end keys are gathered, and the autocovariance records of z merged, by the functions of "combining shards", so every rank
    returns the same numbers."""
    import torch
    entries, chains = block.shape[1], block.shape[2]
    h = rows // 2
    out = {"ess_bulk": np.full(entries, np.nan), "rhat_rank": np.full(entries, np.nan)}
    if rows < MIN_ROWS:
        return out
    dev = block.device
    n = 2 * h * chains
    sizes = gather(np.array([n], dtype=np.int64), block, distributed)[:, 0]
    total = int(sizes.sum())
    M = total // h
    keys = torch.empty(n + int(sizes.max()), dtype=torch.int64, device=dev)     # sorted keys + the sort's scratch / a ring buffer
    index = torch.empty(2 * n, dtype=torch.int32, device=dev)
    acc = torch.empty(n, dtype=torch.int64, device=dev)
    ring = torch.empty(int(sizes.max()), dtype=torch.int64, device=dev)
    z = torch.empty((2, 2 * h, 1, chains), dtype=torch.float64, device=dev)

    def ranked(e: int, centre: float, zb) -> bool:
        """z-scaled ranks of one series into zb; -> whether all its keys are equal over all shards."""
        reducer.rank_sort(block, e, centre, keys, index)
        ends = gather(keys[[0, n - 1]].cpu().numpy(), block, distributed).view(np.uint64)
        acc.zero_()
        _ring_counts(reducer, keys, n, sizes, acc, ring, distributed)
        reducer.rank_z(acc, index, n, total, zb)
        return bool(ends[:, 0].min() == ends[:, 1].max())

    for e in range(entries):
        if np.isnan(vmin[e]) or np.isnan(vmax[e]):
            continue
        if vmin[e] == vmax[e] or ranked(e, float("nan"), z[0]):
            out["ess_bulk"][e] = M * h
            continue
        g = geyer_windows(reducer, z[0], None, h, distributed, max_lags)[0][0][0]
        out["ess_bulk"][e] = g.ess
        with np.errstate(invalid="ignore", divide="ignore"):
            rhat = np.sqrt(g.varplus / g.W)
            if not np.isfinite(med[e]):
                continue
            if ranked(e, float(med[e]), z[1]):
                out["rhat_rank"][e] = rhat
                continue
            gf = GeyerESS(autocov_record(reducer, z[1], None, 0, 1, distributed)[0, 0], h)     # W and var+ only: one lag
            out["rhat_rank"][e] = max(rhat, np.sqrt(gf.varplus / gf.W))
    return out


def _ring_counts(reducer, keys, n: int, sizes: np.ndarray, acc, ring, distributed: bool) -> None:
    """acc += the rank counts of this shard's sorted keys[:n] against every shard's sorted keys: its own first, then the others
    as they come round the ring (step s brings the keys of rank - s, sent on by the ranks in between)."""
    reducer.rank_count(keys, n, keys, n, acc)
    if not distributed:
        return
    import torch.distributed as dist
    ws, rank = dist.get_world_size(), dist.get_rank()
    bufs = (keys[n:], ring)
    cur = keys[:n]
    for step in range(1, ws):
        src = (rank - step) % ws
        recv = bufs[(step - 1) % 2][:int(sizes[src])]
        ops = [dist.P2POp(dist.isend, cur, (rank + 1) % ws), dist.P2POp(dist.irecv, recv, (rank - 1) % ws)]
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        reducer.rank_count(keys, n, recv, int(sizes[src]), acc)
        cur = recv


DIAGNOSTIC_PROBS = (0.0, 0.05, 0.95, 1.0)
RANK_PROBS = (0.5,)                   # the median that centres the folded draws of diagnostics="rank"


def check_diagnostics(diagnostics) -> None:
    if not (isinstance(diagnostics, bool) or (isinstance(diagnostics, str) and diagnostics == "rank")):
        raise ValueError("diagnostics must be False, True or \"rank\", not %r" % (diagnostics,))


def summarise_block(reducer, block, rows: int, total_chains: int, probs: Sequence[float], distributed: bool, diagnostics=False):
    """-> (mean, sd, rhat, quantiles[len(probs)]) per entry, over all shards. `reducer` does the per-shard device work; the
    moment records merge by pooled_moment_record and the select's digit counts add up by sum_counts. diagnostics=True appends
    (split_chain_diagnostics' dict, lag windows used): the select also forms the minimum, q05, q95 and the maximum (each
    quantile is its own order statistics, so the requested ones are unchanged). diagnostics="rank" also forms
    the median and adds rank_diagnostics' "ess_bulk" and "rhat_rank" to that dict; every other value is the same bits. The mean
    and the returned quantiles of an entry with NaN or infinite draws are numpy's (nonfinite_as_numpy); the internal order
    statistics that feed the diagnostics keep their bits."""
    check_diagnostics(diagnostics)
    entries = block.shape[1]
    user_probs = [float(p) for p in probs]
    if diagnostics:
        probs = user_probs + list(DIAGNOSTIC_PROBS) + (list(RANK_PROBS) if diagnostics == "rank" else [])
    mean, sd, rhat = finalize_moments(pooled_moment_record(reducer, block, distributed), rows)

    probs = [float(p) for p in probs]
    q = np.empty((len(probs), entries))
    low = np.empty((len(probs), entries))                     # the lower order statistic of each probability, not interpolated
    per_select = MAX_PREFIXES // 2                            # every probability needs at most two order statistics
    for first in range(0, len(probs), per_select):            # long probability grids (equal-mass histograms): several selects
        chunk = probs[first:first + per_select]
        ranks, plan = quantile_targets(rows * total_chains, chunk)
        sel = _select(reducer, block, ranks, distributed)
        vals = sel.values()                                   # [entries, T]
        for i, (lo, hi, g) in enumerate(plan):
            q[first + i] = _lerp(vals[:, lo], vals[:, hi], g)
            low[first + i] = vals[:, lo]
    mean, q_user = nonfinite_as_numpy(reducer, block, mean, q[:len(user_probs)], rows * total_chains, distributed)
    if not diagnostics:
        return mean, sd, rhat, q_user
    vmin, q05, q95, vmax = q[len(user_probs):len(user_probs) + len(DIAGNOSTIC_PROBS)]
    diag = split_chain_diagnostics(reducer, block, rows, sd, q05, q95, vmin, vmax, distributed)
    if diagnostics == "rank":
        # the exact minimum and maximum: interpolating an infinite extreme with itself gives NaN, and these must tell +-inf from NaN
        lo_min, lo_max = low[len(user_probs)], low[len(user_probs) + 3]
        diag[0].update(rank_diagnostics(reducer, block, rows, q[-1], lo_min, lo_max, distributed))
    return mean, sd, rhat, q_user, diag


def _select(reducer, block, ranks: np.ndarray, distributed: bool) -> RadixSelect:
    """The 8 passes of the radix select of the sorted 0-based `ranks` over all shards; -> the finished RadixSelect."""
    sel = RadixSelect(block.shape[1], ranks)
    for npass in range(8):
        table, which = sel.prefixes()
        sel.advance(sum_counts(reducer.digit_counts(block, npass, table), distributed).cpu().numpy(), which)
    return sel


_KEY_NEG_INF, _KEY_POS_INF = double_to_key(np.array([-np.inf, np.inf]))


def nonfinite_as_numpy(reducer, block, mean: np.ndarray, q_user: np.ndarray, M: int, distributed: bool):
    """-> (mean, quantiles) with the entries that hold NaN or infinite draws summarised as numpy.mean / numpy.quantile
    summarise them; M: the draws per entry over all shards. The merged mean of such an entry is not finite, but not always
    numpy's: once a record's mean is +inf, the Chan merge with a finite record forms inf + (x - inf) w = NaN. And the select
    orders NaN by its sign bit (below -inf or above +inf), so only one end of an entry with a NaN draw comes out NaN.
    So when some mean is not finite, one more radix select finds the smallest and the largest key of every entry (ranks 0 and
    M - 1; distributed: its counts are all-reduced like the quantiles', and every rank takes this branch because the merged mean
    is the same on all of them). The key order puts every NaN outside [-inf, +inf], so an entry holds a NaN exactly when one of
    its extreme keys lies outside, and otherwise holds -inf (+inf) exactly when its smallest (largest) draw is -inf (+inf).
    An entry with a NaN draw gets mean NaN and NaN at every probability; +inf and -inf both: mean NaN; +inf only: mean +inf;
    -inf only: mean -inf. sd and R-hat of all of these are NaN already, and so are their quantiles where numpy.quantile's
    interpolation meets an infinity. An entry with finite draws only whose sum overflowed keeps its merged mean (numpy may differ
    there). When every mean is finite nothing runs and nothing changes."""
    if np.all(np.isfinite(mean)):
        return mean, q_user
    keys = _select(reducer, block, np.unique([0, M - 1]), distributed).prefix
    kmin, kmax = keys[:, 0], keys[:, -1]
    nan = (kmin < _KEY_NEG_INF) | (kmax > _KEY_POS_INF)
    mean, q_user = mean.copy(), q_user.copy()
    mean[(kmin == _KEY_NEG_INF) & (kmax == _KEY_POS_INF)] = np.nan
    mean[(kmax == _KEY_POS_INF) & (kmin != _KEY_NEG_INF)] = np.inf
    mean[(kmin == _KEY_NEG_INF) & (kmax != _KEY_POS_INF)] = -np.inf
    mean[nan] = np.nan
    q_user[:, nan] = np.nan
    return mean, q_user


# ---------------------------------------------------------------------------------------------------------------------
# Monte Carlo standard errors of the quantiles and of the sd (Vehtari et al. 2021, §4.3; ArviZ's mcse(method="quantile") / "sd")
MAX_IND_THRESHOLDS = 16                # include/amwg.h: amwg_summary_indicator_autocov, n_thresholds <= 16 per call
MAX_IND_LAGS = 64                      # and n_lags <= 64 per window
MCSE_BETA_PROBS = (0.1586553, 0.8413447)    # Phi(-1), Phi(1): the +-1 sd points of the beta posterior of the rank


def check_mcse(mcse) -> None:
    if not isinstance(mcse, bool):
        raise ValueError("mcse must be True or False, not %r" % (mcse,))


def check_mcse_size(rows: int, total_chains: int) -> None:
    """mcse=True before the chains move: the indicator counters (each below 2 M h^2, M = 2 * chains, h = rows // 2) must fit in
    int64, and scipy's beta inverse must be importable."""
    h = rows // 2
    if 2 * (2 * total_chains) * h * h >= 1 << 63:
        raise ValueError("mcse=True: %d chains x %d kept rows is too many for the exact indicator counts (2 M h^2 >= 2^63, M = 2 x "
                         "chains, h = rows // 2); raise thin() or lower n" % (total_chains, rows))
    try:
        from scipy.special import betaincinv  # noqa: F401
    except ImportError:
        raise ValueError("mcse=True needs scipy (scipy.special.betaincinv, the beta quantile of the quantiles' standard errors); "
                         "install scipy or call with mcse=False") from None


def mcse_scratch_bytes(entries: int, n_probs: int) -> int:
    """device scratch of mcse_block's calls at most: the indicator thresholds and counters of one call, and the records of
    amwg_summary_autocov_sq (per-CTA moments and lag sums of 1184 CTAs)"""
    k = min(max(n_probs, 1), MAX_IND_THRESHOLDS)
    return entries * (k * (8 + 8 * (2 + 2 * MAX_IND_LAGS)) + 1184 * (32 + 8 * MAX_LAGS) + 8 * (6 + MAX_LAGS))


def indicator_record(sums: np.ndarray, M: int, h: int, lag0: int) -> np.ndarray:
    """Exact integer sums [entries, K, 2 + 2 n] = {C1, C2, P_t..., G_t...} (t = lag0 + i) -> GeyerESS records [entries, K, 4 + n]
    {M, C1 / (M h), (M C2 - C1^2) / (M h^2), (h C1 - C2) / h, (h^2 P_t - h (2 C2 - G_t) + (h - t) C2) / h^2 ...}: each rational
    correctly rounded once (Python's int / int), so the record is a function of the integers only."""
    E, K, W = sums.shape
    n = (W - 2) // 2
    v = sums.astype(object)                                   # Python ints: no intermediate overflows or roundings
    C1, C2 = v[:, :, 0], v[:, :, 1]
    P, G = v[:, :, 2:2 + n], v[:, :, 2 + n:]
    t = np.arange(lag0, lag0 + n, dtype=object)
    out = np.empty((E, K, 4 + n), dtype=object)
    out[:, :, 0] = M
    out[:, :, 1] = C1 / (M * h)
    out[:, :, 2] = (M * C2 - C1 * C1) / (M * h * h)
    out[:, :, 3] = (h * C1 - C2) / h
    out[:, :, 4:] = (h * h * P - h * (2 * C2[:, :, None] - G) + (h - t) * C2[:, :, None]) / (h * h)
    return out.astype(np.float64)


def _indicator_sums(reducer, block, thr, lag0: int, n_lags: int, distributed: bool) -> np.ndarray:
    """reducer.indicator_autocov of every shard, summed (sum_counts)"""
    got = reducer.indicator_autocov(block, thr, lag0, n_lags)
    if not distributed:
        return np.asarray(got, dtype=np.int64)
    import torch
    return sum_counts(torch.from_numpy(np.ascontiguousarray(got, dtype=np.int64)).to(block.device), True).cpu().numpy()


def quantile_ess(reducer, block, rows: int, total_chains: int, thr: np.ndarray, distributed: bool, max_lags: int = MAX_IND_LAGS):
    """-> (ESS [entries, K] of the indicators 1[x <= thr[e][k]] on the split halves, lag windows used). K thresholds go in calls
    of at most MAX_IND_THRESHOLDS; each call's windows are those of geyer_loop over indicator_record. An indicator that is
    constant (C1 = 0 or C1 = M h) has ESS = M h."""
    entries, K = thr.shape
    h, M = rows // 2, 2 * total_chains
    ess = np.empty((entries, K))
    windows = 0
    for k0 in range(0, K, MAX_IND_THRESHOLDS):
        t = np.ascontiguousarray(thr[:, k0:k0 + MAX_IND_THRESHOLDS])
        first = []

        def fetch(lag0, n_lags):
            sums = _indicator_sums(reducer, block, t, lag0, n_lags, distributed)
            if not first:
                first.append(sums[:, :, 0])
            return indicator_record(sums, M, h, lag0)

        est, w = geyer_loop(fetch, h, max_lags)
        windows += w
        C1 = first[0]
        for e in range(entries):
            for k, g in enumerate(est[e]):
                ess[e, k0 + k] = M * h if C1[e, k] == 0 or C1[e, k] == M * h else g.ess
    return ess, windows


def quantile_mcse_ranks(ess: np.ndarray, probs: Sequence[float], S: int):
    """ArviZ's _mcse_quantile ranks: (a1, a2) = the MCSE_BETA_PROBS quantiles of Beta(ess p + 1, ess (1 - p) + 1), i1 =
    rint(max(a1 S - 1, 0)), i2 = rint(min(a2 S - 1, S - 1)) (rint: half to even). ess [P, entries] -> (i1, i2) int64 [P, entries],
    and where ess is NaN (ranks 0 there)."""
    from scipy.special import betaincinv
    p = np.asarray(probs, dtype=np.float64)[:, None]
    bad = ~np.isfinite(ess)
    e = np.where(bad, 1.0, ess)
    a1 = betaincinv(e * p + 1, e * (1 - p) + 1, MCSE_BETA_PROBS[0])
    a2 = betaincinv(e * p + 1, e * (1 - p) + 1, MCSE_BETA_PROBS[1])
    i1 = np.rint(np.maximum(a1 * S - 1, 0))
    i2 = np.rint(np.minimum(a2 * S - 1, S - 1))
    bad |= ~(np.isfinite(i1) & np.isfinite(i2))
    return np.where(bad, 0, i1).astype(np.int64), np.where(bad, 0, i2).astype(np.int64), bad


def pow2_scale(sd: np.ndarray) -> np.ndarray:
    """2^-ilogb(sd) clamped to [2^-1022, 2^1023]; 1 where sd is 0 or not finite"""
    out = np.ones(len(sd))
    for e, v in enumerate(np.asarray(sd, dtype=np.float64)):
        if np.isfinite(v) and v > 0:
            out[e] = math.ldexp(1.0, min(max(1 - math.frexp(float(v))[1], -1022), 1023))
    return out


def mcse_block(reducer, block, rows: int, total_chains: int, probs: Sequence[float], mean: np.ndarray, sd: np.ndarray, q_user: np.ndarray,
               distributed: bool, max_lags: int = MAX_IND_LAGS) -> dict:
    """-> {"ess_quantile" [len(probs), entries], "mcse_quantile" [len(probs), entries], "mcse_sd" [entries]} over all shards;
    mean, sd and q_user are summarise_block's. Only reads the block.

    h = rows // 2 and the halves are those of `split_chain_diagnostics`; M = 2 * chains over all GPUs; S = rows * chains, every
    kept draw; q_p the returned quantile (numpy's linear rule).
      ess_quantile   the split-chain ESS of b = 1[x <= q_p]. Per half-chain m with positions 0..h-1: c_m = sum_n b_mn, F_mt and
                     L_mt the count among its first and last t positions. The integers C1 = sum c_m, C2 = sum c_m^2, P_t = sum_m
                     sum_{n<h-t} b_mn b_m,n+t and G_t = sum_m c_m (F_mt + L_mt) (amwg_summary_indicator_autocov, summed over shards
                     by sum_counts) give GeyerESS its exact inputs: mean of the half-chain means C1 / (M h), m2 = (M C2 - C1^2) /
                     (M h^2), sum_w = (h C1 - C2) / h and lag sum_t = (h^2 P_t - h (2 C2 - G_t) + (h - t) C2) / h^2 (sum_w at t =
                     0), each rounded once to the nearest double (indicator_record). So the ESS is a function of integers only:
                     the same for any sharding, number of GPUs, chain order or launch shape. A constant indicator (C1 = 0 or
                     C1 = M h) gives M h, as in split_chain_diagnostics; W = 0 otherwise gives NaN (GeyerESS).
      mcse_quantile  ArviZ's rule: (a1, a2) the 0.1586553 and 0.8413447 quantiles of Beta(ess p + 1, ess (1 - p) + 1)
                     (scipy.special.betaincinv), i1 = rint(max(a1 S - 1, 0)), i2 = rint(min(a2 S - 1, S - 1)) (half to even, as
                     numpy.rint), and mcse = (x_(i2) - x_(i1)) / 2 with x_(i) the exact 0-based order statistics over all S
                     draws (one more radix select at per-entry ranks, at most 16 probabilities per select). Unlike ArviZ, an ess of
                     NaN gives NaN (ArviZ's nanmax / nanmin would take the extreme draws).
      mcse_sd        the delta-method estimator of posterior / ArviZ: with x_bar the returned mean and s = 2^-ilogb(sd) (clamped
                     to normal powers of two; 1 when sd is 0 or not finite), y = ((x - x_bar) s)^2 on the split halves
                     (amwg_summary_autocov_sq, records merged by merge_autocov_records); y_bar = the mean of the half-chain means,
                     v = (sum of within M2 + h * M2 of the half means) / (M h), the ddof-0 variance of y, ess_y = GeyerESS of y;
                     mcse_sd = sqrt(v / (4 y_bar ess_y)) / s. For even rows y_bar and v are over all draws, as in ArviZ; for odd
                     rows the middle row is left out of them, as it is out of every split-chain quantity.
    Edge cases: fewer than 10 rows (MIN_ROWS): all NaN. A NaN draw in an entry: all three NaN. +-inf draws without NaN:
    ess_quantile as defined (the indicators are finite), mcse_quantile by IEEE arithmetic on the two order statistics, mcse_sd
    NaN. A constant entry (sd 0): ess_quantile M h, mcse_quantile 0, mcse_sd 0. Multiplying the draws by 2^j (no overflow or
    underflow) leaves ess_quantile's bits and multiplies mcse_quantile and mcse_sd by exactly 2^j."""
    entries = block.shape[1]
    P = len(probs)
    out = {"ess_quantile": np.full((P, entries), np.nan), "mcse_quantile": np.full((P, entries), np.nan),
           "mcse_sd": np.full(entries, np.nan)}
    if rows < MIN_ROWS:
        return out
    h, M, S = rows // 2, 2 * total_chains, rows * total_chains
    nan_e = np.zeros(entries, dtype=bool)
    inf_e = np.zeros(entries, dtype=bool)
    if not np.all(np.isfinite(mean)):                         # which entries hold a NaN, which +-inf only (nonfinite_as_numpy)
        keys = _select(reducer, block, np.unique([0, S - 1]), distributed).prefix
        kmin, kmax = keys[:, 0], keys[:, -1]
        nan_e = (kmin < _KEY_NEG_INF) | (kmax > _KEY_POS_INF)
        inf_e = ~nan_e & ((kmin == _KEY_NEG_INF) | (kmax == _KEY_POS_INF))
    if P:
        ess, _ = quantile_ess(reducer, block, rows, total_chains, np.ascontiguousarray(np.asarray(q_user, dtype=np.float64).T), distributed,
                              max_lags)
        ess = ess.T                                           # [P, entries]
        ess[:, nan_e] = np.nan
        i1, i2, bad = quantile_mcse_ranks(ess, probs, S)
        mq = np.empty((P, entries))
        per_select = MAX_PREFIXES // 2
        for first in range(0, P, per_select):
            n = min(per_select, P - first)
            ranks = np.empty((entries, 2 * n), dtype=np.int64)
            ranks[:, 0::2] = i1[first:first + n].T
            ranks[:, 1::2] = i2[first:first + n].T
            vals = _select(reducer, block, ranks, distributed).values()
            with np.errstate(invalid="ignore", over="ignore"):
                mq[first:first + n] = ((vals[:, 1::2] - vals[:, 0::2]) / 2).T
        mq[bad] = np.nan
        out["ess_quantile"], out["mcse_quantile"] = ess, mq

    ok = ~nan_e & ~inf_e & np.isfinite(mean)
    scale = pow2_scale(sd)
    centre = np.where(ok, mean, 0.0)
    est, _ = geyer_loop(lambda lag0, n_lags: merge_autocov_records(gather(reducer.autocov_sq(block, centre, scale, lag0, n_lags), block,
                                                                              distributed)), h, MAX_LAGS)
    for e in range(entries):
        if not ok[e]:
            continue
        if sd[e] == 0:
            out["mcse_sd"][e] = 0.0
            continue
        g = est[e][0]
        _, ybar, m2, sum_w = g.record
        v = (sum_w + h * m2) / (M * h)
        with np.errstate(invalid="ignore", divide="ignore"):
            out["mcse_sd"][e] = np.sqrt(v / (4.0 * ybar * g.ess)) / scale[e]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# posterior histograms: equal-width 1-D bins per entry and 2-D counts of entry pairs, equal to numpy's on the raw draws
MAX_HIST_BINS = 4096                   # include/amwg.h: amwg_summary_histogram, bins <= 4096
MAX_PAIR_BINS = 128                    # amwg_summary_histogram2d: bins <= 128 per axis
MAX_PAIRS = 64                         # amwg_summary_histogram2d: n_pairs <= 64
PAIR_BINS = 50                         # default bins per axis of a 2-D histogram
_HIST_KEYS = ("bins", "range", "pairs", "pair_bins")


class HistogramPlan(NamedTuple):
    """A checked `histogram=` argument. bins: 1-D bins per entry (None: pairs only); fixed: [entries, 2] user (lo, hi), NaN where
    the range comes from the draws; pairs: (key as given, entry a, entry b); pair_bins: bins per axis of every pair."""
    bins: Optional[int]
    fixed: np.ndarray
    pairs: List[Tuple[object, int, int]]
    pair_bins: int


def _is_int(v) -> bool:
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def entry_spans(names: Sequence[str], dims) -> dict:
    """{name: (first entry, number of entries)} of the names laid out in order in a sample block, prod(dims[name]) entries each
    (row-major). A name listed twice in monitor: its last block, as sample_summary returns it."""
    spans = {}
    first = 0
    for name in names:
        n = int(np.prod(dims[name]))
        spans[name] = (first, n)
        first += n
    return spans


def selector(sel, spans: dict, what: str) -> Tuple[object, int]:
    """One entry selector, a scalar's name or (name, flat_index) -> (label, block entry); the label is the name, or
    (name, int(flat_index)). `what` starts every error message."""
    if isinstance(sel, str):
        if sel not in spans:
            raise ValueError("%s: %r is not a monitored parameter or derived quantity" % (what, sel))
        if spans[sel][1] != 1:
            raise ValueError("%s: %r has %d components; select one as (%r, flat_index)" % (what, sel, spans[sel][1], sel))
        return sel, spans[sel][0]
    if isinstance(sel, (tuple, list)) and len(sel) == 2 and isinstance(sel[0], str) and _is_int(sel[1]):
        name, i = sel
        if name not in spans:
            raise ValueError("%s: %r is not a monitored parameter or derived quantity" % (what, name))
        if not 0 <= i < spans[name][1]:
            raise ValueError("%s: component %d of %r is outside [0, %d)" % (what, i, name, spans[name][1]))
        return (name, int(i)), spans[name][0] + int(i)
    raise ValueError("%s selector must be a name or (name, flat_index), not %r" % (what, sel))


def resolve_histogram(spec, names: Sequence[str], dims) -> Optional[HistogramPlan]:
    """Checks the `histogram=` argument of sample_summary against the monitored names (in sample-block order, only those with
    entries) and their dims ({name: dim list}; the entries of a name are prod(dim), row-major) and returns the plan, or None for
    None. Pure: raises ValueError before any device work."""
    if spec is None:
        return None
    if _is_int(spec):
        spec = {"bins": spec}
    elif not isinstance(spec, dict):
        raise ValueError("histogram must be None, an int number of bins or a dict, not %r" % (spec,))
    unknown = [k for k in spec if k not in _HIST_KEYS]
    if unknown:
        raise ValueError("histogram has unknown key(s) %s; the keys are %s" % (", ".join(map(repr, unknown)), ", ".join(_HIST_KEYS)))
    span = entry_spans(names, dims)
    entries = sum(span[name][1] for name in names)

    bins = spec.get("bins")
    if "bins" in spec and not (_is_int(bins) and 1 <= bins <= MAX_HIST_BINS):
        raise ValueError("histogram bins must be an int in 1..%d, not %r" % (MAX_HIST_BINS, bins))
    pair_bins = spec.get("pair_bins", PAIR_BINS)
    if not (_is_int(pair_bins) and 1 <= pair_bins <= MAX_PAIR_BINS):
        raise ValueError("histogram pair_bins must be an int in 1..%d, not %r" % (MAX_PAIR_BINS, pair_bins))

    fixed = np.full((entries, 2), np.nan)
    ranges = spec.get("range", {})
    if not isinstance(ranges, dict):
        raise ValueError("histogram range must be a dict {name: (lo, hi)}, not %r" % (ranges,))
    for name, r in ranges.items():
        if name not in span:
            raise ValueError("histogram range: %r is not a monitored parameter or derived quantity" % (name,))
        ok = isinstance(r, (tuple, list)) and len(r) == 2 and all(isinstance(v, numbers.Real) and not isinstance(v, bool) for v in r)
        if not ok or not (np.isfinite(r[0]) and np.isfinite(r[1])) or not r[0] < r[1]:
            raise ValueError("histogram range of %r must be (lo, hi) with finite lo < hi, not %r" % (name, r))
        s0, n = span[name]
        fixed[s0:s0 + n] = (float(r[0]), float(r[1]))

    def entry(sel) -> Tuple[object, int]:
        label, e = selector(sel, span, "histogram pair")
        return label if isinstance(sel, list) else sel, e          # a tuple selector keys the pair as given

    given = spec.get("pairs", [])
    if not isinstance(given, (tuple, list)):
        raise ValueError("histogram pairs must be a list of (a, b) selectors, not %r" % (given,))
    if len(given) > MAX_PAIRS:
        raise ValueError("histogram pairs: %d pairs (max %d)" % (len(given), MAX_PAIRS))
    pairs: List[Tuple[object, int, int]] = []
    for p in given:
        if not (isinstance(p, (tuple, list)) and len(p) == 2):
            raise ValueError("histogram pair must be (a, b), not %r" % (p,))
        (ka, ea), (kb, eb) = entry(p[0]), entry(p[1])
        key = (ka, kb)                                       # the pair as given (a list selector becomes a tuple: keys must hash)
        if all(key != q[0] for q in pairs):
            pairs.append((key, ea, eb))
    if bins is None and not pairs:
        raise ValueError("histogram needs bins, pairs or both")
    return HistogramPlan(bins, fixed, pairs, pair_bins)


def histogram_block(reducer, block, rows: int, plan: HistogramPlan, distributed: bool) -> dict:
    """-> {"hist" [entries, bins] int64, "hist_edges" [entries, bins + 1], "hist_outside" [entries, 3] int64 (when plan.bins),
    "pairs": {key: {"hist" [pair_bins, pair_bins] int64, "xedges", "yedges"}}} over all shards; only reads the block.

    Range of an entry: plan.fixed when given, else (lo, hi) = the smallest and largest finite draw over all rows, chains and
    shards (numpy.histogram's default on the finite draws); lo == hi gives (lo - 0.5, hi + 0.5), no finite draw (0, 1). Edges:
    numpy.linspace(lo, hi, bins + 1). A draw lo <= x <= hi goes to numpy.histogram's bin (csrc/amwg_hist.cuh); hist_outside counts
    the draws < lo (-inf included), > hi (+inf included) and NaN, so hist.sum() + hist_outside.sum() is the number of draws.
    A pair's axes are its two entries' ranges at plan.pair_bins; a draw counts when both values lie inside their axis's edges,
    each binned as numpy.histogramdd bins it (searchsorted right, the last edge in the last bin).
    Distributed: the extremes combine by merged_extremes and all the counts add up in one sum_counts, so every rank returns the
    same bits whatever the number of GPUs."""
    import torch
    entries = block.shape[1]
    lo, hi = plan.fixed[:, 0].copy(), plan.fixed[:, 1].copy()
    used = np.zeros(entries, dtype=bool)
    used[:] = plan.bins is not None
    for _key, a, b in plan.pairs:
        used[a] = used[b] = True
    auto = np.isnan(lo)
    if np.any(auto & used):
        rng = merged_extremes(reducer.finite_range(block)[0].cpu().numpy(), block, distributed)
        for e in np.flatnonzero(auto):
            a, b = rng[e]
            lo[e], hi[e] = (0.0, 1.0) if not a <= b else (a - 0.5, b + 0.5) if a == b else (a, b)
    lo[auto & ~used], hi[auto & ~used] = 0.0, 1.0

    def edges(k: int) -> np.ndarray:
        return np.stack([np.linspace(lo[e], hi[e], k + 1) for e in range(entries)])

    parts = []
    if plan.bins is not None:
        e1 = edges(plan.bins)
        parts.append(reducer.histogram(block, e1, plan.bins))
    if plan.pairs:
        e2 = edges(plan.pair_bins)
        pair_idx = np.array([(a, b) for _k, a, b in plan.pairs], dtype=np.int32)
        parts.append(reducer.histogram2d(block, pair_idx, e2, plan.pair_bins))
    if distributed:                                           # one all-reduce for all the counts
        flat = sum_counts(torch.cat([p.reshape(-1) for p in parts]), distributed)
        parts = list(torch.split(flat, [p.numel() for p in parts]))
    counts = [p.cpu().numpy().astype(np.int64, copy=False) for p in parts]
    out = {"pairs": {}}
    if plan.bins is not None:
        c1 = counts.pop(0).reshape(entries, plan.bins + 3)
        out.update(hist=c1[:, :plan.bins].copy(), hist_edges=e1, hist_outside=c1[:, plan.bins:].copy())
    if plan.pairs:
        c2 = counts.pop(0).reshape(len(plan.pairs), plan.pair_bins, plan.pair_bins)
        for i, (key, a, b) in enumerate(plan.pairs):
            out["pairs"][key] = {"hist": c2[i].copy(), "xedges": e2[a].copy(), "yedges": e2[b].copy()}
    return out


# ---------------------------------------------------------------------------------------------------------------------
# posterior covariance: cross-products of the draws on the fp64 tensor core, correlations, multivariate R-hat
MAX_COV_ENTRIES = 128                  # include/amwg.h: amwg_summary_comoments, n_sel <= 128


class CovariancePlan(NamedTuple):
    """A checked `covariance=` argument: labels (the selectors in matrix order) and the block entry of each."""
    labels: List[object]
    entries: np.ndarray


def resolve_covariance(spec, names: Sequence[str], dims) -> Optional[CovariancePlan]:
    """Checks the `covariance=` argument of sample_summary against the monitored names (in sample-block order, only those with
    entries) and their dims, as resolve_histogram does, and returns the plan, or None for None / False. True covers every
    monitored entry (a scalar labelled by its name, a component of a multi-dim name by (name, flat_index), row-major); a list
    covers the selectors it holds, in its order, each a scalar's name or (name, flat_index). Pure: raises ValueError before any
    device work."""
    if spec is None or spec is False:
        return None
    _check_result_key("covariance", names)
    span = entry_spans(names, dims)
    if spec is True:
        labels = [name if span[name][1] == 1 else (name, i) for name in span for i in range(span[name][1])]
        idx = [span[name][0] + i for name in span for i in range(span[name][1])]
    elif isinstance(spec, (list, tuple)):
        labels, idx = [], []
        for sel in spec:
            label, e = selector(sel, span, "covariance")
            if e in idx:
                raise ValueError("covariance: %r selects an entry already selected" % (sel,))
            labels.append(label)
            idx.append(e)
        if not idx:
            raise ValueError("covariance: the selector list is empty")
    else:
        raise ValueError("covariance must be None, True or a list of selectors, not %r" % (spec,))
    if len(idx) > MAX_COV_ENTRIES:
        raise ValueError("covariance: %d entries (max %d)" % (len(idx), MAX_COV_ENTRIES))
    return CovariancePlan(labels, np.asarray(idx, dtype=np.int32))


def comoments_scratch_bytes(n_sel: int, chains: int) -> int:
    """Device scratch of amwg_summary_comoments (include/amwg.h)."""
    up = lambda b: -(-b // 256) * 256
    nb = -(-n_sel // 8)
    tiles = nb * (nb + 1) // 2
    reps = 1 if tiles >= 16 else 16 // tiles
    ctas = min(-(-chains // 32), 264)
    return up(8 * n_sel * chains) + up(8 * n_sel) + up(8 * 64 * tiles * ctas * reps) + up(8 * 128 * tiles)


def split_comoment_record(rec: np.ndarray):
    """flat record [1 + n + 2 n^2] -> (chains, m [n], B [n, n], W [n, n])."""
    rec = np.asarray(rec, dtype=np.float64)
    n = int(round((np.sqrt(8.0 * (rec.size - 1) + 1.0) - 1.0) / 4.0))
    assert 1 + n + 2 * n * n == rec.size, rec.size
    return rec[0], rec[1:1 + n], rec[1 + n:1 + n + n * n].reshape(n, n), rec[1 + n + n * n:].reshape(n, n)


def merge_comoment_records(records: Sequence[np.ndarray]) -> np.ndarray:
    """Chan merge of per-shard flat records {C, m[n], B[n][n], W[n][n]} in the order given (rank order), in matrix form:
    B = B_a + B_b + (n_a n_b / n) d d^T with d = m_b - m_a, W adds. The arithmetic of merge_moment_records."""
    na, ma, Ba, Wa = split_comoment_record(records[0])
    ma, Ba, Wa = ma.copy(), Ba.copy(), Wa.copy()
    for rec in records[1:]:
        nb, mb, Bb, Wb = split_comoment_record(rec)
        if nb == 0:
            continue
        if na == 0:
            na, ma, Ba, Wa = nb, mb.copy(), Bb.copy(), Wb.copy()
            continue
        n = na + nb
        d = mb - ma
        ma = ma + d * (nb / n)
        Ba = Ba + Bb + np.outer(d, d) * (na * nb / n)
        Wa = Wa + Wb
        na = n
    return np.concatenate([[na], ma, Ba.ravel(), Wa.ravel()])


def finalize_comoments(rec: np.ndarray, rows: int) -> dict:
    """{"mean", "cov", "corr", "within", "between", "rhat_multivariate", "n_draws"} from the merged record. With C chains and
    M = C rows draws: cov = (W + rows B) / (M - 1) (ddof 1; its diagonal is finalize_moments' sd squared), corr = cov / (sd sd^T)
    in numpy.corrcoef's operations (clipped to [-1, 1]), within = W / (C (rows - 1)), between = B / (C - 1) and Brooks & Gelman's
    (1998) multivariate potential scale reduction (n - 1)/n + (C + 1)/C lambda_max(within^-1 between), n = rows, from a Cholesky
    factor of within and eigvalsh. The R-hat is NaN when rows < 2, C < 2, any entry is non-finite, or within is not positive
    definite (a constant entry, or one that is linear in others). An entry whose draws all equal one value is centred on that
    value exactly on the device, so its rows and columns of cov, within and between are 0 and its correlations NaN, as
    numpy.corrcoef gives for a row of zero variance."""
    G, m, B, W = split_comoment_record(rec)
    M = G * rows
    with np.errstate(invalid="ignore", divide="ignore"):
        cov = (W + rows * B) / (M - 1)
        sd = np.sqrt(np.diag(cov))
        corr = cov / sd[:, None]
        corr /= sd[None, :]
        np.clip(corr, -1, 1, out=corr)
        within = W / (G * (rows - 1))
        between = B / (G - 1)
    rhat = np.nan
    if rows >= 2 and G >= 2 and np.all(np.isfinite(within)) and np.all(np.isfinite(between)):
        try:
            L = np.linalg.cholesky(within)
        except np.linalg.LinAlgError:
            L = None
        if L is not None:
            Li = np.linalg.inv(L)
            S = Li @ between @ Li.T
            lam = np.linalg.eigvalsh((S + S.T) / 2).max()
            rhat = float((rows - 1) / rows + (G + 1) / G * lam)
    return {"mean": m.copy(), "cov": cov, "corr": corr, "within": within, "between": between, "rhat_multivariate": rhat,
            "n_draws": int(M)}


def covariance_block(reducer, block, rows: int, plan: CovariancePlan, distributed: bool) -> dict:
    """-> finalize_comoments' dict plus "labels", over all shards; only reads the block. Each shard's record comes from
    reducer.comoments; distributed: the fixed-size records are gathered (gather) and merged on the host in rank order
    (merge_comoment_records), so every rank returns the same bits."""
    rec = merge_comoment_records(gather(reducer.comoments(block, plan.entries), block, distributed))
    out = {"labels": list(plan.labels)}
    out.update(finalize_comoments(rec, rows))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# nested R-hat (Margossian et al., "Nested R-hat", Bayesian Analysis 2024): superchains of M chains that start together
NESTED_RECORD = 14                     # include/amwg.h: amwg_summary_nested, doubles per entry


def resolve_nested(spec, superchain_size: Optional[int], first_chain: int, chains: int) -> Optional[int]:
    """Checks the `nested=` argument of sample_summary and returns the superchain size M, or None for None / False. True takes
    options.superchain_size (`superchain_size`, None when it was not set); an int >= 1 is M itself. Superchain k is the global
    chains [kM, (k + 1)M), and the chains summarised, [first_chain, first_chain + chains) (all of them with options.distributed),
    must be whole superchains. Pure: raises ValueError before any device work."""
    if spec is None or spec is False:
        return None
    if spec is True:
        if superchain_size is None:
            raise ValueError("nested=True needs options.superchain_size")
        M = int(superchain_size)
    elif _is_int(spec) and spec >= 1:
        M = int(spec)
    else:
        raise ValueError("nested must be None, False, True or an int superchain size >= 1, not %r" % (spec,))
    if first_chain % M or (first_chain + chains) % M:
        raise ValueError("nested: the chains summarised, [%d, %d), are not whole superchains of %d chains"
                         % (first_chain, first_chain + chains, M))
    return M


def nested_scratch_bytes(entries: int, chains: int, first_chain: int, superchain_size: int) -> int:
    """Device scratch of amwg_summary_nested (include/amwg.h)."""
    up = lambda b: -(-b // 256) * 256
    n_seg = (first_chain + chains - 1) // superchain_size - first_chain // superchain_size + 1
    ctas = min(-(-n_seg // 256), 1184)
    return up(16 * entries * chains) + up(32 * entries * ctas) + up(32 * entries) + up(64 * entries)


def nested_unit(rec: np.ndarray, M: int, rows: int) -> np.ndarray:
    """Chain-level records [..., 4] of whole superchains (M chains, mean of the chain means, M2 of the chain means, sum of the
    within-chain M2) -> their units (1, superchain mean, 0, B~_k + W-_k) of the superchain-to-total level: B~_k = M2 / (M - 1)
    (0 when M = 1), W-_k = sum / (M (rows - 1)) (0 when rows = 1). The arithmetic of nested_unit in csrc/amwg_nested.cuh."""
    rec = np.asarray(rec, dtype=np.float64)
    b = rec[..., 2] / float(M - 1) if M > 1 else np.zeros_like(rec[..., 2])
    w = rec[..., 3] / (float(M) * float(rows - 1)) if rows > 1 else np.zeros_like(rec[..., 3])
    return np.stack([np.ones_like(rec[..., 0]), rec[..., 1], np.zeros_like(rec[..., 0]), b + w], axis=-1)


def merge_nested_records(records: Sequence[np.ndarray], M: int, rows: int) -> np.ndarray:
    """Per-shard [entries, 14] records of amwg_summary_nested in rank order -> one [entries, 4] superchain-to-total record
    (superchains, mean of the superchain means, M2 of the superchain means, sum over superchains of B~_k + W-_k). The complete
    records merge in rank order (merge_moment_records). The cut records are grouped by superchain id and merged in rank order
    into chain-level records, which must then hold all M chains; each becomes its unit (nested_unit) and is folded in, in the
    order of the superchain ids."""
    recs = [np.asarray(r, dtype=np.float64) for r in records]
    total = merge_moment_records([r[:, :4] for r in recs])
    cut = {}
    for r in recs:
        for slot in range(2):
            part = r[:, 4 + 5 * slot:9 + 5 * slot]
            if part[0, 0] < 0:
                continue
            k = int(part[0, 0])
            cut[k] = part[:, 1:] if k not in cut else merge_moment_records([cut[k], part[:, 1:]])
    for k in sorted(cut):
        if not np.all(cut[k][:, 0] == M):
            raise RuntimeError("nested: superchain %d has %d of its %d chains over all shards" % (k, int(cut[k][0, 0]), M))
        total = merge_moment_records([total, nested_unit(cut[k], M, rows)])
    return total


def finalize_nested(rec: np.ndarray) -> np.ndarray:
    """rhat_nested per entry from the merged [entries, 4] superchain-to-total record (K, mean of the superchain means, M2 of the
    superchain means, sum over superchains of B~_k + W-_k): with B^ = M2 / (K - 1) and W^ = sum / K,
    rhat_nested = sqrt(1 + B^ / W^). NaN when K < 2, when W^ = 0 (an entry whose draws all equal one value, whose chain records
    then hold that mean and M2 = 0 exactly; or M = 1 with N = 1), or when any value of the record is not finite (a NaN or +-inf
    draw of the entry)."""
    rec = np.asarray(rec, dtype=np.float64)
    K, mean, m2, sw = rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3]
    with np.errstate(invalid="ignore", divide="ignore"):
        B = m2 / (K - 1)
        W = sw / K
        rhat = np.sqrt(1.0 + B / W)
    ok = (K >= 2) & (W > 0) & np.isfinite(mean) & np.isfinite(B) & np.isfinite(W)
    return np.where(ok, rhat, np.nan)


def nested_block(reducer, block, rows: int, first_chain: int, M: int, distributed: bool) -> np.ndarray:
    """-> rhat_nested per entry over all shards; only reads the block. Each shard's record comes from reducer.nested;
    distributed: the fixed-size records are gathered (gather) and merged on the host in rank order (merge_nested_records), so
    every rank returns the same bits."""
    return finalize_nested(merge_nested_records(gather(reducer.nested(block, first_chain, M), block, distributed), M, rows))


# ---------------------------------------------------------------------------------------------------------------------
# PSIS-LOO and WAIC (Vehtari, Gelman & Gabry 2017; Vehtari et al., JMLR 2024), in ArviZ's conventions: DESIGN.md §4.7
LOO_KEYS = ("log_lik", "points", "r_eff")
MAX_LOO_TAIL = 1 << 20                 # include/amwg.h: amwg_loo_fit, tail_cap <= 2^20
LOG_TINY = float(np.log(np.finfo(float).tiny))


class LooPlan(NamedTuple):
    """A checked `loo=` argument."""
    log_lik: object
    points: int
    r_eff: float


def resolve_loo(spec, names: Sequence[str]) -> Optional[LooPlan]:
    """Checks the `loo=` argument of sample_summary: None, or {"log_lik": callable (state, data, i), "points": int >= 1,
    "r_eff": finite float > 0 (default 1.0)}, with no monitored name "loo" (the key the result uses). Pure: raises ValueError
    before any device work (tracing log_lik is the caller's next check)."""
    if spec is None:
        return None
    log_lik, points = _log_lik_spec(spec, "loo", LOO_KEYS, "the log-likelihood of point i")
    r_eff = spec.get("r_eff", 1.0)
    if not (isinstance(r_eff, numbers.Real) and not isinstance(r_eff, bool) and np.isfinite(r_eff) and r_eff > 0):
        raise ValueError("loo r_eff must be a finite number > 0, not %r" % (r_eff,))
    _check_result_key("loo", names)
    return LooPlan(log_lik, points, float(r_eff))


def _log_lik_spec(spec, what: str, keys: Sequence[str], value: str) -> Tuple[object, int]:
    """The checks `loo=` and `ppc=` share: a dict of `keys` with a callable "log_lik" and an int "points" >= 1; -> (log_lik,
    points). `value` says what log_lik returns."""
    if not isinstance(spec, dict):
        raise ValueError("%s must be None or a dict {\"log_lik\": ..., \"points\": ...}, not %r" % (what, spec))
    unknown = [k for k in spec if k not in keys]
    if unknown:
        raise ValueError("%s has unknown key(s) %s; the keys are %s" % (what, ", ".join(map(repr, unknown)), ", ".join(keys)))
    if not callable(spec.get("log_lik")):
        raise ValueError("%s needs \"log_lik\": a function (state, data, i) -> %s" % (what, value))
    points = spec.get("points")
    if not (_is_int(points) and points >= 1):
        raise ValueError("%s points must be an int >= 1, not %r" % (what, points))
    return spec["log_lik"], int(points)


def _check_result_key(key: str, names: Sequence[str]) -> None:
    if key in names:
        raise ValueError("%s: a monitored parameter or derived quantity is named '%s', the key the result would use" % (key, key))


def loo_tail_length(S: int, r_eff: float) -> int:
    """M = ceil(min(0.2 S, 3 sqrt(S / r_eff))): the Pareto tail holds the draws above the (M + 1)-th largest log weight."""
    return int(np.ceil(min(0.2 * S, 3 * np.sqrt(S / r_eff))))


def loo_tail_cap(M: int) -> int:
    """The tail buffers' length per point: the power of two >= max(M, 8) (the fit kernel's bitonic sort)."""
    cap = 8
    while cap < M:
        cap *= 2
    return cap


def loo_point_bytes(rows: int, chains: int, cap: int, world: int) -> int:
    """Device bytes one point of a chunk takes, from the sizes the calls allocate (include/amwg.h): its ll column of the chunk; its
    tail buffer and count (this rank's, and with world > 1 every rank's gathered); the fit's sort and value scratch (16 cap) and its
    llmin / cut / skip / out (56); the per-CTA records of amwg_summary_moments (32 G + 32) and the sums of amwg_loo_reduce
    (24 G + 48), G = min(ceil(chains / 256), 1184) CTAs; the select's prefix and digit counts (8 + 8 x 256); the finite range and
    non-finite counts (16 + 24 + 16 + 24: the device keys and the returned tensors)."""
    G = min(-(-chains // 256), 1184)
    tails = (8 * cap + 4) * (1 + (world if world > 1 else 0))
    return 8 * rows * chains + tails + 16 * cap + 56 + (32 * G + 32) + (24 * G + 48) + (8 + 8 * 256) + 80


def check_loo_size(S: int, r_eff: float, what: str = "loo") -> int:
    """-> M, or ValueError when S < 2 or the tail exceeds what the fit kernel holds. `what` names the option in the message."""
    if S < 2:
        raise ValueError("%s needs at least 2 draws (kept rows x chains), not %d" % (what, S))
    M = loo_tail_length(S, r_eff)
    if M > MAX_LOO_TAIL:
        raise ValueError("%s: a Pareto tail of %d draws per point (S = %d, r_eff = %g) exceeds %d" % (what, M, S, r_eff, MAX_LOO_TAIL))
    return M


def loo_cut(reducer, ll, M: int, distributed: bool):
    """The steps of PSIS-LOO before the tail pass, over a chunk ll [rows, P, chains] of every shard: -> (llmin, llmax, skip, cut),
    [P] each. llmin / llmax: the smallest / largest finite ll (merged_extremes over the shards' finite ranges); skip: the points
    with a non-finite ll (sum_counts of the non-finite counts); cut = max(llmin - (the M-th smallest ll, 0-based, by the radix
    select), log(DBL_MIN)), so the tail holds the draws with lw = llmin - ll > cut."""
    rng, nonfinite = reducer.finite_range(ll)
    llmin, llmax = merged_extremes(rng.cpu().numpy(), ll, distributed).T
    skip = sum_counts(nonfinite, distributed).cpu().numpy().sum(axis=1) > 0
    llM = _select(reducer, ll, np.array([M], dtype=np.int64), distributed).values()[:, 0]
    with np.errstate(invalid="ignore"):
        cut = np.maximum(llmin - llM, LOG_TINY)
    return llmin, llmax, skip, cut


def _program_arrays(prog):
    """(code, consts, fold_prog, fold_dst, n_fold) of a traced program as the pointwise ABI calls take them: contiguous arrays,
    an empty table padded to one unused element so that its pointer is valid."""
    consts = np.ascontiguousarray(prog.consts if prog.consts else [0.0], dtype=np.float64)
    fold_prog = np.ascontiguousarray(prog.fold_prog if prog.fold_prog else [0], dtype=np.int32)
    fold_dst = np.ascontiguousarray(prog.fold_dst if prog.fold_dst else [0], dtype=np.int32)
    return np.ascontiguousarray(prog.code, dtype=np.int32), consts, fold_prog, fold_dst, len(prog.fold_prog)


class CudaPointwise:
    """The pointwise log-likelihood chunks of one sample block: amwg_loo_pointwise over the handle's data columns."""

    def __init__(self, handle, prog, block, device: int):
        from . import _ffi
        self.L, self._ffi = _ffi.lib(), _ffi
        self.h, self.block, self.device = handle, block, device
        self.code, self.consts, self.fold_prog, self.fold_dst, self.n_fold = _program_arrays(prog)
        self.body = prog.logpost_prog

    def chunk(self, p0: int, P: int):
        """-> float64 CUDA tensor [rows, P, chains]: ll of points p0 .. p0 + P - 1 at every kept draw of the block."""
        import torch
        rows, entries, chains = self.block.shape
        out = torch.empty((rows, P, chains), dtype=torch.float64, device=self.block.device)
        torch.cuda.current_stream(self.block.device).synchronize()
        i32p = C.POINTER(C.c_int32)
        self._ffi.check(self.L.amwg_loo_pointwise(self.h, self.code.ctypes.data_as(i32p), self.code.size,
                                                  self.consts.ctypes.data_as(C.POINTER(C.c_double)), self.consts.size, self.body,
                                                  self.fold_prog.ctypes.data_as(i32p), self.fold_dst.ctypes.data_as(i32p), self.n_fold,
                                                  self.block.data_ptr(), rows, entries, p0, P, out.data_ptr()))
        return out


def loo_block(reducer, source, rows: int, total_chains: int, points: int, r_eff: float, chunk_points: int, distributed: bool) -> dict:
    """-> the "loo" dict of sample_summary over all shards: PSIS-LOO and WAIC from the pointwise log-likelihood ll[s, i] of the
    S = rows x total_chains kept draws. `source.chunk(p0, P)` gives ll of points p0 .. p0 + P - 1 as a [rows, P, chains] block
    (this shard's chains); the points go in chunks of at most `chunk_points`. Per chunk, on the device: the finite range and
    non-finite counts (amwg_summary_finite_range), the moments (amwg_summary_moments: var_s ll = (sum of within-chain M2 +
    rows x M2 of the chain means) / S), the M-th smallest ll (0-based; the radix select of the quantiles), M =
    ceil(min(0.2 S, 3 sqrt(S / r_eff))), so the (M + 1)-th largest lw = llmin - ll is c = llmin - that value and
    cut = max(c, log(DBL_MIN)); then one pass for the sums and the tail (reducer.loo_reduce) and the Pareto fit over the tail
    (reducer.loo_fit). Per point i, with lw = llmin - ll:
      lppd_i      = llmax + log(sum exp(ll - llmax)) - log S
      p_waic_i    = var_s ll (ddof 0),  elpd_waic_i = lppd_i - p_waic_i
      elpd_loo_i  = llmin + log(sum exp(lw' + ll - llmin)) - log(sum exp(lw')), lw' the smoothed log weights
                    (logsumexp(lw' - logsumexp(lw') + ll)),  p_loo_i = lppd_i - elpd_loo_i
      pareto_k_i  the fitted k (+inf for a tail of <= 4 draws, or when no candidate of the fit has a finite profile value)
    A point with any non-finite ll gets NaN in every value. Totals: sums of the pointwise values, se_* = sqrt(points var_i(elpd_*_i))
    (ddof 0), looic = -2 elpd_loo, waic = -2 elpd_waic, pareto_k_threshold = min(1 - 1 / log10 S, 0.7), n_high_k = #{k > threshold}.
    Distributed: the extremes combine by merged_extremes, the non-finite counts and the select's counts add up by sum_counts,
    the moment records merge by pooled_moment_record, the sums are gathered and added in rank order, and the tails are gathered
    (gather_tensor; at most M values per point in all); the fit runs on the merged tail, so every rank returns the same
    numbers."""
    S = rows * total_chains
    M = check_loo_size(S, r_eff)
    cap = loo_tail_cap(M)
    cols = {k: np.full(points, np.nan) for k in ("elpd_loo", "lppd", "p_loo", "elpd_waic", "p_waic", "pareto_k")}
    for p0 in range(0, points, chunk_points):
        P = min(chunk_points, points - p0)
        ll = source.chunk(p0, P)
        llmin, llmax, skip, cut = loo_cut(reducer, ll, M, distributed)
        rec = pooled_moment_record(reducer, ll, distributed)
        var = (rec[:, 3] + rows * rec[:, 2]) / S
        # a point with a non-finite ll is NaN throughout: keep its draws out of the tail
        mn, mx, ct = np.where(skip, 0.0, llmin), np.where(skip, 0.0, llmax), np.where(skip, np.inf, cut)
        sums, tails, counts = reducer.loo_reduce(ll, mn, mx, ct, cap)
        del ll
        parts = gather(sums, tails, distributed)
        sums = parts[0]
        for q in parts[1:]:
            sums = sums + q
        fit = reducer.loo_fit(gather_tensor(tails, distributed), gather_tensor(counts, distributed), mn, ct, skip.astype(np.int32))
        del tails, counts
        if np.any(fit[~skip, 3] > M):
            raise RuntimeError("loo: a point's tail holds more than M = %d draws (inconsistent select)" % M)
        with np.errstate(invalid="ignore", divide="ignore"):
            lppd = llmax + np.log(sums[:, 0]) - np.log(float(S))
            elpd = llmin + np.log(sums[:, 2] + fit[:, 2]) - np.log(sums[:, 1] + fit[:, 1])
        sl = slice(p0, p0 + P)
        cols["lppd"][sl], cols["p_waic"][sl], cols["elpd_waic"][sl] = lppd, var, lppd - var
        cols["elpd_loo"][sl], cols["p_loo"][sl], cols["pareto_k"][sl] = elpd, lppd - elpd, fit[:, 0]
        for key in cols:
            cols[key][sl][skip] = np.nan
    thr = min(1.0 - 1.0 / np.log10(S), 0.7)
    with np.errstate(invalid="ignore"):
        n_high = int(np.sum(cols["pareto_k"] > thr))
        out = {"elpd_loo": float(np.sum(cols["elpd_loo"])), "se_elpd_loo": float(np.sqrt(points * np.var(cols["elpd_loo"]))),
               "p_loo": float(np.sum(cols["p_loo"])), "elpd_waic": float(np.sum(cols["elpd_waic"])),
               "se_elpd_waic": float(np.sqrt(points * np.var(cols["elpd_waic"]))), "p_waic": float(np.sum(cols["p_waic"]))}
    out["looic"], out["waic"] = -2.0 * out["elpd_loo"], -2.0 * out["elpd_waic"]
    out.update(pointwise=cols, pareto_k_threshold=float(thr), n_high_k=n_high, r_eff=float(r_eff), n_draws=int(S), points=int(points))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# posterior predictive checks (BDA3 ch. 6; ArviZ's plot_ppc / plot_bpv): DESIGN.md §4.8
PPC_KEYS = ("log_lik", "points", "loo_pit")
# the families with a sampler, in the order of the family codes of csrc/amwg_ppc.cuh (amwg_ppc_pointwise)
PPC_FAMILIES = ("norm", "lnorm", "cauchy", "laplace", "logis", "exp", "weibull", "pareto", "unif", "gamma", "invgamma", "beta", "t",
                "bern", "pois", "binom", "nbinom")
PPC_STATS = ("mean", "sd", "min", "max")
MAX_PPC_DRAWS = 1 << 46                # rows x points: the stream region of amwg_ppc_pointwise (2^16 uniforms each below 2^63)


class PpcPlan(NamedTuple):
    """A checked `ppc=` argument; loo_pit is the r_eff of LOO-PIT, None without it."""
    log_lik: object
    points: int
    loo_pit: Optional[float] = None


def resolve_ppc(spec, names: Sequence[str]) -> Optional[PpcPlan]:
    """Checks the `ppc=` argument of sample_summary: None, or {"log_lik": callable (state, data, i), "points": int >= 1, optional
    "loo_pit": True (r_eff = 1.0) or {"r_eff": finite float > 0}}, with no monitored name "ppc" (the key the result uses). Pure:
    raises ValueError before any device work (tracing log_lik and check_ppc_call are the caller's next checks)."""
    if spec is None:
        return None
    log_lik, points = _log_lik_spec(spec, "ppc", PPC_KEYS, "one ld.* call at data point i")
    r_eff = None
    if "loo_pit" in spec:
        pit = spec["loo_pit"]
        if pit is True:
            r_eff = 1.0
        elif isinstance(pit, dict) and list(pit) == ["r_eff"]:
            r_eff = pit["r_eff"]
            if not (isinstance(r_eff, numbers.Real) and not isinstance(r_eff, bool) and np.isfinite(r_eff) and r_eff > 0):
                raise ValueError("ppc loo_pit r_eff must be a finite number > 0, not %r" % (r_eff,))
            r_eff = float(r_eff)
        else:
            raise ValueError("ppc loo_pit must be True or {\"r_eff\": a finite number > 0}, not %r" % (pit,))
    _check_result_key("ppc", names)
    return PpcPlan(log_lik, points, r_eff)


def check_ppc_call(family: str, rows: int, points: int) -> int:
    """-> the family code of amwg_ppc_pointwise, or ValueError for a family without a sampler or rows x points >= 2^46."""
    if family not in PPC_FAMILIES:
        raise ValueError("ppc: ld.%s has no sampler; the families are %s" % (family, ", ".join(PPC_FAMILIES)))
    if rows * points >= MAX_PPC_DRAWS:
        raise ValueError("ppc: kept rows x points = %d must stay below 2^46" % (rows * points))
    return PPC_FAMILIES.index(family)


def dataset_stats(y) -> np.ndarray:
    """T(y) = (mean, sd, min, max) of one dataset, the points in index order, with the device's operations: sequential Welford
    (d = y - m; m += d / j; M2 += d (y - m)), sd = sqrt(M2 / (N - 1)) (NaN for N = 1), min and max propagating NaN."""
    m = M2 = 0.0
    mn = mx = float("nan")
    for j, v in enumerate(np.asarray(y, dtype=np.float64).tolist(), 1):
        d = v - m
        m += d / j
        M2 += d * (v - m)
        if j == 1:
            mn = mx = v
        elif mn != mn or v != v:
            mn = mx = float("nan")
        else:
            mn, mx = (v if v < mn else mn), (v if v > mx else mx)
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = float(np.sqrt(np.float64(M2) / np.float64(len(y) - 1)))
    return np.array([m, sd, mn, mx])


def ppc_point_bytes(rows: int, chains: int) -> int:
    """Device bytes one point of a chunk takes, from the sizes the calls allocate (include/amwg.h): its y_rep column of the chunk,
    the per-CTA records of amwg_summary_moments (32 G + 32, G = min(ceil(chains / 256), 1184)) and the threshold and counts of
    amwg_summary_threshold_counts (8 + 32)."""
    G = min(-(-chains // 256), 1184)
    return 8 * rows * chains + (32 * G + 32) + 40


def loo_pit_point_bytes(rows: int, chains: int, cap: int, world: int) -> int:
    """Device bytes one point of a chunk takes for LOO-PIT on top of ppc_point_bytes, from the sizes the calls allocate
    (include/amwg.h): its ll column of the chunk; its tail buffer, flags and count (this rank's, and with world > 1 every rank's
    gathered); the fit's sort, value and flag scratch (17 cap) and its llmin / cut / skip / out (64); the llmin / cut / y and the
    sums of amwg_loo_pit_reduce (24 G + 48), G = min(ceil(chains / 256), 1184) CTAs; the select's prefix and digit counts
    (8 + 8 x 256); the finite range and non-finite counts (16 + 24 + 16 + 24: the device keys and the returned tensors)."""
    G = min(-(-chains // 256), 1184)
    tails = (9 * cap + 4) * (1 + (world if world > 1 else 0))
    return 8 * rows * chains + tails + 17 * cap + 64 + (24 * G + 48) + (8 + 8 * 256) + 80


def ppc_fixed_bytes(rows: int, chains: int) -> int:
    """Device bytes of the whole call: the statistics records T [rows][4][chains] (32 rows chains) and the scratch of summarising
    them as a 4-entry block (two entries' worth of chain records, as the base summary's check counts)."""
    return 32 * rows * chains + 2 * 4 * chains * 8


class CudaPpc:
    """The replicated data of one sample block, in chunks of points: amwg_ppc_pointwise over the handle's data columns. The
    statistics records live on the device from the first chunk to the last; `stats()` returns them once the last chunk ran."""

    def __init__(self, handle, prog, offsets, family: int, block, points: int):
        import torch
        from . import _ffi
        self.L, self._ffi = _ffi.lib(), _ffi
        self.h, self.block, self.family, self.points = handle, block, family, points
        self.code, self.consts, self.fold_prog, self.fold_dst, self.n_fold = _program_arrays(prog)
        self.args = np.ascontiguousarray(offsets, dtype=np.int32)
        rows, _, chains = block.shape
        self.T = torch.empty((rows, 4, chains), dtype=torch.float64, device=block.device)

    def chunk(self, p0: int, P: int):
        """-> float64 CUDA tensor [rows, P, chains]: y_rep of points p0 .. p0 + P - 1 at every kept draw of the block (chunks in order)."""
        import torch
        rows, entries, chains = self.block.shape
        out = torch.empty((rows, P, chains), dtype=torch.float64, device=self.block.device)
        torch.cuda.current_stream(self.block.device).synchronize()
        i32p = C.POINTER(C.c_int32)
        self._ffi.check(self.L.amwg_ppc_pointwise(self.h, self.code.ctypes.data_as(i32p), self.code.size,
                                                  self.consts.ctypes.data_as(C.POINTER(C.c_double)), self.consts.size, self.family,
                                                  self.args.ctypes.data_as(i32p), self.args.size, self.fold_prog.ctypes.data_as(i32p),
                                                  self.fold_dst.ctypes.data_as(i32p), self.n_fold, self.block.data_ptr(), rows, entries,
                                                  self.points, p0, P, out.data_ptr(), self.T.data_ptr()))
        return out

    def stats(self):
        """-> the [rows, 4, chains] block of every draw's (mean, sd, min, max), after the last chunk"""
        return self.T


def ppc_block(reducer, source, rows: int, total_chains: int, points: int, family: str, y, probs: Sequence[float], chunk_points: int,
              distributed: bool, loo_pit=None) -> dict:
    """-> the "ppc" dict of sample_summary over all shards, for the S = rows x total_chains kept draws. `source.chunk(p0, P)` gives
    y_rep of points p0 .. p0 + P - 1 as a [rows, P, chains] block (this shard's chains; chunks of at most `chunk_points`, in
    order), and `source.stats()` after the last chunk the [rows, 4, chains] block of each draw's T(y_rep) = (mean, sd, min,
    max) (amwg_ppc_pointwise). y: the observed y_0 .. y_{N-1}.
    pointwise: "mean" and "sd" of y_rep_i over the S draws as the base summary forms them (finalize_moments: pooled, ddof 1),
    "n_below" / "n_equal" / "n_nan" (int64: y_rep_i < y_i, == y_i, NaN), "pit" = (n_below + n_equal) / S (ArviZ's u-value).
    stats: per T, "observed" T(y) (dataset_stats), "mean", "sd" and "quantiles" (`probs`) of T(y_rep) from summarise_block,
    "n_greater", "n_equal", "n_nan" and "p_value" = (n_greater + n_equal) / S, Pr(T(y_rep) >= T(y)) with a NaN draw counted as
    not >= (and with T(y) NaN, no draw is). Distributed: the moment records merge by pooled_moment_record, the threshold counts
    (int64 [entries, 4]: <, ==, >, NaN) add up by sum_counts, and summarise_block takes its distributed path; every rank returns
    the same numbers.
    loo_pit = (ll_source, r_eff) adds "loo_pit" (loo_pit_chunk): ll_source.chunk(p0, P) gives the log-likelihood of the same ld.*
    call as a [rows, P, chains] block, taken while that chunk's y_rep is resident."""
    S = rows * total_chains
    y = np.ascontiguousarray(y, dtype=np.float64)
    pw = {"mean": np.empty(points), "sd": np.empty(points)}
    cnt = np.empty((points, 4), dtype=np.int64)
    if loo_pit is not None:
        ll_source, r_eff = loo_pit
        M = check_loo_size(S, r_eff, "ppc loo_pit")
        pit = {k: np.full(points, np.nan) for k in ("pit", "pit_equal", "pareto_k")}
    for p0 in range(0, points, chunk_points):
        P = min(chunk_points, points - p0)
        yrep = source.chunk(p0, P)
        sl = slice(p0, p0 + P)
        pw["mean"][sl], pw["sd"][sl], _rhat = finalize_moments(pooled_moment_record(reducer, yrep, distributed), rows)
        cnt[sl] = sum_counts(reducer.threshold_counts(yrep, y[sl]), distributed).cpu().numpy()
        if loo_pit is not None:
            pit["pit"][sl], pit["pit_equal"][sl], pit["pareto_k"][sl] = loo_pit_chunk(reducer, ll_source.chunk(p0, P), yrep, y[sl], M,
                                                                                     distributed)
        del yrep
    pw.update(n_below=cnt[:, 0], n_equal=cnt[:, 1], pit=(cnt[:, 0] + cnt[:, 1]) / S, n_nan=cnt[:, 3])
    T = source.stats()
    obs = dataset_stats(y)
    mean, sd, _rhat, q = summarise_block(reducer, T, rows, total_chains, probs, distributed)
    tc = sum_counts(reducer.threshold_counts(T, obs), distributed).cpu().numpy()
    stats = {}
    for k, name in enumerate(PPC_STATS):
        stats[name] = {"observed": float(obs[k]), "mean": float(mean[k]), "sd": float(sd[k]), "quantiles": q[:, k].copy(),
                       "n_greater": int(tc[k, 2]), "n_equal": int(tc[k, 1]), "n_nan": int(tc[k, 3]),
                       "p_value": float((tc[k, 2] + tc[k, 1]) / S)}
    out = {"family": family, "points": int(points), "n_draws": int(S), "pointwise": pw, "stats": stats}
    if loo_pit is not None:
        thr = min(1.0 - 1.0 / np.log10(S), 0.7)
        with np.errstate(invalid="ignore"):
            n_high = int(np.sum(pit["pareto_k"] > thr))
        pit.update(pareto_k_threshold=float(thr), n_high_k=n_high, r_eff=float(r_eff))
        out["loo_pit"] = pit
    return out


def loo_pit_chunk(reducer, ll, yrep, y, M: int, distributed: bool):
    """LOO-PIT of one chunk of points (DESIGN.md §4.9): ll and yrep [rows, P, chains] of this shard, y [P] the observations, M the
    tail length of every shard's S draws. -> (pit, pit_equal, pareto_k), [P] each. The steps of PSIS-LOO (loo_cut) give llmin, cut
    and the points with a non-finite ll; one pass (reducer.loo_pit_reduce) sums the weights exp(lw) of the draws outside the tail,
    in all and where y_rep <= y and y_rep == y, and collects the tail's ll with those two flags; the fit over the merged tail
    (reducer.loo_pit_fit) gives k, the tail's weights and their flag sums, each draw of a run of tied ll weighted by the run's mean
    weight. With D, LE and EQ the three sums over all draws: pit = min(1, LE / D), pit_equal = min(1, EQ / D); a point with a
    non-finite ll gets NaN in all three. Distributed: loo_cut's steps, the sums gathered and added in rank order, and the tails,
    flags and counts gathered (gather_tensor), so every rank returns the same numbers."""
    llmin, _llmax, skip, cut = loo_cut(reducer, ll, M, distributed)
    mn, ct = np.where(skip, 0.0, llmin), np.where(skip, np.inf, cut)
    sums, tails, flags, counts = reducer.loo_pit_reduce(ll, yrep, mn, ct, y, loo_tail_cap(M))
    del ll
    parts = gather(sums, tails, distributed)
    sums = parts[0]
    for q in parts[1:]:
        sums = sums + q
    fit = reducer.loo_pit_fit(gather_tensor(tails, distributed), gather_tensor(flags, distributed), gather_tensor(counts, distributed), mn,
                              ct, skip.astype(np.int32))
    del tails, flags, counts
    if np.any(fit[~skip, 4] > M):
        raise RuntimeError("ppc loo_pit: a point's tail holds more than M = %d draws (inconsistent select)" % M)
    with np.errstate(invalid="ignore", divide="ignore"):
        D = sums[:, 0] + fit[:, 1]
        pit = np.minimum(1.0, (sums[:, 1] + fit[:, 2]) / D)
        pit_equal = np.minimum(1.0, (sums[:, 2] + fit[:, 3]) / D)
    k = fit[:, 0].copy()
    for v in (pit, pit_equal, k):
        v[skip] = np.nan
    return pit, pit_equal, k
