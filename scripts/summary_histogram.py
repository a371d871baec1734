"""Cost of the posterior histograms of sample_summary at config-2 size on one GPU: 2^20 chains of Normal(mu, sigma) with
N = 1024 data points, burn(1000), then sample_summary(100) alternating with
sample_summary(100, histogram={"bins": 50, "pairs": [("mu", "sigma")]}).

Prints one JSON line: ms per call of each (median of --reps after --warmup of each) and the time of each of the three device
reductions (CUDA events around the reducer call, which includes its small buffer setup), median over the histogram calls.
The card's name and power limit are read in the same run."""
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
    kernel_ms = {"finite_range": [], "histogram": [], "histogram2d": []}

    def timed_method(name):
        method = getattr(summary.CudaBlockReducer, name)

        def wrapper(self, *a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = method(self, *a, **k)
            e1.record()
            e1.synchronize()
            kernel_ms[name].append(e0.elapsed_time(e1))
            return out
        setattr(summary.CudaBlockReducer, name, wrapper)
    for name in kernel_ms:
        timed_method(name)
    spec = {"bins": 50, "pairs": [("mu", "sigma")]}

    def timed(hist):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = s.sample_summary(args.rows, histogram=hist)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), out

    for _ in range(args.warmup):
        timed(None)
        timed(spec)
    for v in kernel_ms.values():
        v.clear()
    plain, hist = [], []
    for _ in range(args.reps):
        plain.append(timed(None)[0])
        ms, res = timed(spec)
        hist.append(ms)
    name, limit = card()
    ms_plain, ms_hist = float(np.median(plain)), float(np.median(hist))
    block_gb = args.rows * 2 * args.chains * 8 / 1e9
    print(json.dumps({
        "workload": "config 2: Normal(mu,sigma), N=1024, %d chains, burn(%d), sample_summary(%d), histogram=%r" % (args.chains, args.burn, args.rows, spec),
        "gpu": name, "power_limit_w": limit, "block_gb": round(block_gb, 3),
        "ms_per_call_plain": round(ms_plain, 3), "ms_per_call_histogram": round(ms_hist, 3),
        "ms_histogram_extra": round(ms_hist - ms_plain, 3), "reps": args.reps,
        "ms_per_reduction": {k: round(float(np.median(v)), 3) for k, v in kernel_ms.items()},
        "hbm_tb_per_s": {k: round(block_gb / float(np.median(v)), 3) for k, v in kernel_ms.items()},
        "hist_mu_max_bin": int(res["mu"]["hist"].max()), "pair_nonzero_cells": int((res[("mu", "sigma")]["hist"] > 0).sum()),
    }))


if __name__ == "__main__":
    main()
