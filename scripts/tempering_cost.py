"""Cost of tempered ladders (options.temperatures) on one GPU, for config 2: Normal(mu, sigma), N = 1024 data points, 2^20 chains,
interpreter kernels (AMWG_JIT=0, which tempered ladders always use). An untempered and a tempered sampler (K = 8, T = 1.5^r) run
burn(--sweeps) alternately, --reps times each after --warmup.

Prints one JSON line: per 100 sweeps, the sweep kernels' CUDA-event time (amwg_last_sweep_kernel_ms) and the host time of the whole
synchronised burn call, medians of each sampler; and, from a separate profiled burn of the tempered sampler (torch.profiler, CUDA
activities), the device time of amwg_swap_kernel per 100 sweeps. The card's name and power limit are read in the same run."""
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
    ap.add_argument("--rungs", type=int, default=8)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    os.environ["AMWG_JIT"] = "0"
    import torch
    pkg = graft.load_package()
    mcmc, ld = pkg.mcmc, pkg.ld
    name, limit = card()

    def log_post(state, data):
        lp = 0
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], state.mu, state.sigma)
        return lp
    data = np.random.default_rng(1024).normal(184.5, 4.5, 1024).tolist()
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    temps = [1.5 ** r for r in range(args.rungs)]
    plain = mcmc.AmwgSampler(params, log_post, data, {"chains": args.chains, "seed": 1, "device": 0})
    hot = mcmc.AmwgSampler(params, log_post, data, {"chains": args.chains, "seed": 1, "device": 0, "temperatures": temps})
    scale = 100.0 / args.sweeps

    def timed(s):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.burn(args.sweeps)
        return 1e3 * (time.perf_counter() - t0) * scale, s.last_sweep_kernel_ms() * scale

    for _ in range(args.warmup):
        timed(plain)
        timed(hot)
    res = {"plain": [], "tempered": []}
    for _ in range(args.reps):
        res["plain"].append(timed(plain))
        res["tempered"].append(timed(hot))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hot.burn(args.sweeps)
        torch.cuda.synchronize()
    swap_us = sum(e.device_time_total for e in prof.key_averages() if "amwg_swap_kernel" in e.key)
    t = hot.info()["tempering"]
    med = {k: (float(np.median([w for w, _ in v])), float(np.median([s for _, s in v]))) for k, v in res.items()}
    print(json.dumps({
        "card": name, "power_limit_w": limit, "chains": args.chains, "rungs": args.rungs, "sweeps_per_call": args.sweeps,
        "jit": [plain.jit_status()[1], hot.jit_status()[1]],
        "per_100_sweeps_ms": {
            "untempered": {"sweep_kernels": med["plain"][1], "burn_call": med["plain"][0]},
            "tempered": {"sweep_kernels": med["tempered"][1], "burn_call": med["tempered"][0], "swap_kernel": swap_us * 1e-3 * scale},
        },
        "swap_rate": [float(x) for x in t["swap_rate"]],
    }))


if __name__ == "__main__":
    main()
