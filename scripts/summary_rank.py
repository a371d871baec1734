"""Cost of the rank-normalised diagnostics of sample_summary at config-2 size on one GPU: 2^20 chains of Normal(mu, sigma) with
N = 1024 data points, burn(1000), then sample_summary(100) with diagnostics=True and diagnostics="rank", alternating the two.

Prints one JSON line: ms per call of each (median of --reps after --warmup of each), and for the "rank" calls the time of every
radix sort, rank count and z scatter (host clock around each entry, which ends in a device synchronise), the radix passes each
sort ran, and the sort's bytes (24 B per ranked draw per executed pass plus the 8 B per draw of the histogram read) over its
time against the H100 SXM data-sheet 3.35 TB/s. The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import __graft_entry__ as graft  # noqa: E402
from summary_diagnostics import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=1 << 20)
    ap.add_argument("--rows", type=int, default=100)
    ap.add_argument("--burn", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    pkg = graft.load_package()
    mcmc, ld, summary = pkg.mcmc, pkg.ld, pkg.summary

    def log_post(state, data):
        lp = 0
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], state.mu, state.sigma)
        return lp

    data = np.random.default_rng(1024).normal(184.5, 4.5, 1024).tolist()
    s = mcmc.AmwgSampler({"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}, log_post, data,
                         {"chains": args.chains, "seed": 1, "device": 0})
    s.burn(args.burn)
    calls = {"rank_sort": [], "rank_count": [], "rank_z": []}
    passes = []
    R = summary.CudaBlockReducer

    def timed_entry(name, fn):
        def wrapper(self, *a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(self, *a, **k)                               # every entry ends in a device synchronise
            calls[name].append(1e3 * (time.perf_counter() - t0))
            if name == "rank_sort":
                passes.append(out)
            return out
        return wrapper
    for name in calls:
        setattr(R, name, timed_entry(name, getattr(R, name)))

    def timed(diag):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = s.sample_summary(args.rows, diagnostics=diag)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), out

    for _ in range(args.warmup):
        timed(True)
        timed("rank")
    ms_true, ms_rank = [], []
    for _ in range(args.reps):
        ms_true.append(timed(True)[0])
        for v in calls.values():
            v.clear()
        passes.clear()
        ms, res = timed("rank")
        ms_rank.append(ms)
    name, limit = card()
    S = 2 * (args.rows // 2) * args.chains
    sort_bytes = [24 * S * p + 8 * S for p in passes]
    print(json.dumps({
        "workload": "config 2: Normal(mu,sigma), N=1024, %d chains, burn(%d), sample_summary(%d)" % (args.chains, args.burn, args.rows),
        "gpu": name, "power_limit_w": limit, "ranked_draws_per_sort": S, "reps": args.reps,
        "ms_per_call_true": round(float(np.median(ms_true)), 3), "ms_per_call_rank": round(float(np.median(ms_rank)), 3),
        "ms_rank_extra": round(float(np.median(ms_rank) - np.median(ms_true)), 3),
        "sorts_last_call": ["mu bulk", "mu folded", "sigma bulk", "sigma folded"][:len(passes)],
        "ms_per_sort": [round(v, 3) for v in calls["rank_sort"]], "passes_per_sort": passes,
        "sort_bytes_gb": [round(b / 1e9, 3) for b in sort_bytes],
        "sort_tb_per_s": [round(b / (ms * 1e-3) / 1e12, 3) for b, ms in zip(sort_bytes, calls["rank_sort"])],
        "sort_share_of_3_35_tb_s": [round(b / (ms * 1e-3) / HBM_BYTES_PER_S, 3) for b, ms in zip(sort_bytes, calls["rank_sort"])],
        "ms_per_rank_count": [round(v, 3) for v in calls["rank_count"]], "ms_per_rank_z": [round(v, 3) for v in calls["rank_z"]],
        "ess_bulk": {k: float(res[k]["ess_bulk"]) for k in res}, "rhat_rank": {k: float(res[k]["rhat_rank"]) for k in res},
        "ess_mean": {k: float(res[k]["ess_mean"]) for k in res}, "rhat_split": {k: float(res[k]["rhat_split"]) for k in res},
    }))


if __name__ == "__main__":
    main()
