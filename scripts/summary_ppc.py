"""Cost of the posterior predictive checks in sample_summary on one GPU, for config 2: Normal(mu, sigma), N = 1024 data points,
2^20 chains, log_lik(state, data, i) = ld.norm(data[i], mu, sigma). burn(--burn), then for each number of kept rows (--rows,
default 1 and 10) sample_summary(rows) alternating with sample_summary(rows, ppc={...}).

Prints one JSON line per row count: ms per call of each (median of --reps after --warmup of each); the time of the replicated-data
calls (CUDA events around CudaPpc.chunk, summed over the chunks of one call: the chunk's allocation, the programs' checks and
uploads and the pointwise kernel); the draws of y_rep and the bytes of the y_rep chunks (8 S N), both from shapes; the chunks a
call used. Then, in a separate profiled call (torch.profiler, CUDA activities), the device time of every kernel of one
sample_summary(rows, ppc=...) call by kernel name. The card's name and power limit are read in the same run."""
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
    ap.add_argument("--rows", default="1,10")
    ap.add_argument("--chains", type=int, default=1 << 20)
    ap.add_argument("--burn", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    pkg = graft.load_package()
    summary, ld = pkg.summary, pkg.ld
    kernel_ms = []
    method = summary.CudaPpc.chunk

    def timed_chunk(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = method(self, *a, **k)
        e1.record()
        e1.synchronize()
        kernel_ms.append(e0.elapsed_time(e1))
        return out
    summary.CudaPpc.chunk = timed_chunk
    name, limit = card()
    s = sampler(pkg, 2, args.chains)
    s.burn(args.burn)
    N = 1024
    ppc = {"log_lik": lambda st, d, i: ld.norm(d[i], st.mu, st.sigma), "points": N}
    for rows in [int(r) for r in args.rows.split(",")]:
        def timed(with_ppc):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = s.sample_summary(rows, ppc=ppc if with_ppc else None)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), out

        for _ in range(args.warmup):
            timed(False)
            timed(True)
        plain, withp, kern, chunks = [], [], [], []
        res = None
        for _ in range(args.reps):
            plain.append(timed(False)[0])
            kernel_ms.clear()
            ms, res = timed(True)
            withp.append(ms)
            kern.append(sum(kernel_ms))
            chunks.append(len(kernel_ms))
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.sample_summary(rows, ppc=ppc)
            torch.cuda.synchronize()
        per_kernel = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                per_kernel[e.key] = per_kernel.get(e.key, 0.0) + us / 1e3
        pw = [k for k in per_kernel if "amwg_ppc_pointwise_kernel" in k]
        if not pw:
            raise RuntimeError("the profile holds no amwg_ppc_pointwise_kernel: %s" % sorted(per_kernel))
        ms_pw = sum(per_kernel[k] for k in pw)
        top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:14]
        S = rows * args.chains
        yrep_bytes = 8 * S * N
        ms_k = float(np.median(kern))
        print(json.dumps({
            "workload": "config 2: N=%d, %d chains, burn(%d), sample_summary(%d), ppc over %d points" % (N, args.chains, args.burn, rows, N),
            "gpu": name, "power_limit_w": limit, "draws": S, "yrep_draws": S * N, "yrep_gb": round(yrep_bytes / 1e9, 3),
            "ms_per_call_plain": round(float(np.median(plain)), 3), "ms_per_call_ppc": round(float(np.median(withp)), 3),
            "ms_ppc_extra": round(float(np.median(withp)) - float(np.median(plain)), 3), "reps": args.reps,
            "ms_pointwise_call": round(ms_k, 3), "chunks": int(np.median(chunks)),
            "ms_pointwise_kernel_profiled": round(ms_pw, 3), "yrep_draws_per_s_kernel": float(S * N / (ms_pw / 1e3)),
            "pointwise_write_tb_per_s_kernel": round(yrep_bytes / 1e9 / ms_pw, 3),
            "profiled_call_ms_by_kernel": {k[:90]: round(v, 3) for k, v in top},
            "max_p_value": res["ppc"]["stats"]["max"]["p_value"], "sd_p_value": res["ppc"]["stats"]["sd"]["p_value"],
        }), flush=True)


if __name__ == "__main__":
    main()
