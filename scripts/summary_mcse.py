"""Cost of mcse=True in sample_summary on one GPU, for config 2: Normal(mu, sigma), N = 1024 data points, 2^20 chains.
burn(--burn), then sample_summary(--rows) alternating with sample_summary(--rows, mcse=True) at the default probs.

Prints one JSON line: ms per call of each (median of --reps after --warmup of each, a host clock around a synchronised call) and
their difference; the indicator and squared-deviation lag windows a call used; and, from a separate profiled call (torch.profiler,
CUDA activities), the device time of every kernel of one sample_summary(--rows, mcse=True) call by kernel name, with the bytes of
the block each indicator window reads over that kernel's time. The card's name and power limit are read in the same run."""
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
from summary_covariance import sampler  # noqa: E402
from summary_diagnostics import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100)
    ap.add_argument("--chains", type=int, default=1 << 20)
    ap.add_argument("--burn", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    pkg = graft.load_package()
    summary = pkg.summary
    windows = {"indicator": [], "sq": []}
    red_cls = summary.CudaBlockReducer

    class Counting(red_cls):
        def indicator_autocov(self, block, thresholds, lag0, n_lags):
            windows["indicator"].append((lag0, n_lags, int(np.asarray(thresholds).shape[1])))
            return super().indicator_autocov(block, thresholds, lag0, n_lags)

        def autocov_sq(self, block, centre, scale, lag0, n_lags):
            windows["sq"].append((lag0, n_lags))
            return super().autocov_sq(block, centre, scale, lag0, n_lags)
    summary.CudaBlockReducer = Counting
    name, limit = card()
    s = sampler(pkg, 2, args.chains)
    s.burn(args.burn)
    rows = args.rows

    def timed(mcse):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = s.sample_summary(rows, mcse=mcse)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), out

    for _ in range(args.warmup):
        timed(False)
        timed(True)
    plain, with_mcse = [], []
    res = None
    for _ in range(args.reps):
        plain.append(timed(False)[0])
        windows["indicator"].clear()
        windows["sq"].clear()
        ms, res = timed(True)
        with_mcse.append(ms)
    used = {k: list(v) for k, v in windows.items()}
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.sample_summary(rows, mcse=True)
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us > 0:
            per_kernel[e.key] = per_kernel.get(e.key, 0.0) + us / 1e3
    own = {k: v for k, v in per_kernel.items() if "amwg_indicator_kernel" in k or "amwg_autocov_sq_kernel" in k}
    if len(own) < 2:
        raise RuntimeError("the profile lacks the mcse kernels: %s" % sorted(per_kernel))
    entries = 2
    block_bytes = rows * entries * args.chains * 8
    ind_ms = sum(v for k, v in own.items() if "amwg_indicator_kernel" in k)
    # each indicator window reads the kept half-chain rows once per group of 4 thresholds (twice when lag0 >= 64)
    groups = sum(-(-k // 4) * (1 if l0 < 64 else 2) for l0, _, k in used["indicator"])
    ind_bytes = groups * 2 * (rows // 2) * entries * args.chains * 8
    top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:14]
    print(json.dumps({
        "workload": "config 2: N=1024, %d chains, burn(%d), sample_summary(%d) with and without mcse=True, default probs"
                    % (args.chains, args.burn, rows),
        "gpu": name, "power_limit_w": limit, "draws": rows * args.chains, "block_gb": round(block_bytes / 1e9, 3),
        "ms_per_call": round(float(np.median(plain)), 3), "ms_per_call_mcse": round(float(np.median(with_mcse)), 3),
        "ms_mcse_extra": round(float(np.median(with_mcse)) - float(np.median(plain)), 3), "reps": args.reps,
        "indicator_windows": used["indicator"], "sq_windows": used["sq"],
        "profiled_ms_mcse_kernels": {k[:90]: round(v, 3) for k, v in own.items()},
        "indicator_gb_read": round(ind_bytes / 1e9, 3),
        "indicator_gb_per_s": round(ind_bytes / 1e9 / (ind_ms / 1e3), 1) if ind_ms > 0 else None,
        "profiled_call_ms_by_kernel": {k[:90]: round(v, 3) for k, v in top},
        "mcse_quantile_mu": [float(v) for v in res["mu"]["mcse_quantile"]], "ess_quantile_mu": [float(v) for v in res["mu"]["ess_quantile"]],
        "mcse_sd_mu": float(res["mu"]["mcse_sd"]),
    }), flush=True)


if __name__ == "__main__":
    main()
