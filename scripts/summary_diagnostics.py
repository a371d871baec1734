"""Cost of the split-chain diagnostics of sample_summary at config-2 size on one GPU: 2^20 chains of Normal(mu, sigma) with
N = 1024 data points, burn(1000), then sample_summary(100) with and without diagnostics=True, alternating the two.

Prints one JSON line: ms per call of each (median of --reps after --warmup of each), the lag windows one diagnostics call
asked for, ess_mean / ess_tail per parameter, and effective draws per second (ess_mean over the time of a sample_summary call
without diagnostics: the sweeps plus the moments and quantiles). The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        limit = float(out.stdout.strip().splitlines()[0])
    except Exception:                                            # no nvidia-smi: the number is reported without a power limit
        limit = None
    return name, limit


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
    windows = []
    autocov = summary.CudaBlockReducer.autocov

    def counted(self, *a, **k):                                  # counts the lag windows of one call
        windows.append(a[2])
        return autocov(self, *a, **k)
    summary.CudaBlockReducer.autocov = counted

    def timed(diag):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = s.sample_summary(args.rows, diagnostics=diag)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), out

    for _ in range(args.warmup):
        timed(False)
        timed(True)
    plain, diag = [], []
    for _ in range(args.reps):
        plain.append(timed(False)[0])
        windows.clear()
        ms, res = timed(True)
        diag.append(ms)
    name, limit = card()
    ms_plain, ms_diag = float(np.median(plain)), float(np.median(diag))
    draws = args.chains * args.rows
    print(json.dumps({
        "workload": "config 2: Normal(mu,sigma), N=1024, %d chains, burn(%d), sample_summary(%d)" % (args.chains, args.burn, args.rows),
        "gpu": name, "power_limit_w": limit,
        "ms_per_call_plain": round(ms_plain, 3), "ms_per_call_diagnostics": round(ms_diag, 3),
        "ms_diagnostics_extra": round(ms_diag - ms_plain, 3), "reps": args.reps,
        "lag_windows": len(windows), "lags_read": int(sum(min(32, args.rows // 2 - w) for w in windows)),
        "ess_mean": {k: float(res[k]["ess_mean"]) for k in res}, "ess_tail": {k: float(res[k]["ess_tail"]) for k in res},
        "rhat_split": {k: float(res[k]["rhat_split"]) for k in res},
        "draws_per_s": draws / (ms_plain / 1e3),
        "effective_draws_per_s": {k: float(res[k]["ess_mean"]) / (ms_plain / 1e3) for k in res},
    }))


if __name__ == "__main__":
    main()
