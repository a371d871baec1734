"""Cost of LOO-PIT in sample_summary on one GPU, for config 2: Normal(mu, sigma), N = 1024 data points, 2^20 chains,
ppc={"log_lik": ld.norm(data[i], mu, sigma), "points": N}. burn(--burn), then for each number of kept rows (--rows, default 1 and
10) sample_summary(rows, ppc={...}) alternating with sample_summary(rows, ppc={..., "loo_pit": True}).

Prints one JSON line per row count: ms per call of each (median of --reps after --warmup of each) and their difference; the chunks
of points a call used. Then, in a separate profiled call (torch.profiler, CUDA activities), the device time of every kernel of one
sample_summary(rows, ppc={..., "loo_pit": True}) call by kernel name, so the two LOO-PIT kernels' own time is isolated. The card's
name and power limit are read in the same run."""
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
    chunks = []
    method = summary.loo_pit_chunk

    def counted(*a, **k):
        chunks.append(1)
        return method(*a, **k)
    summary.loo_pit_chunk = counted
    name, limit = card()
    s = sampler(pkg, 2, args.chains)
    s.burn(args.burn)
    N = 1024
    f = lambda st, d, i: ld.norm(d[i], st.mu, st.sigma)
    ppc = {"log_lik": f, "points": N}
    pit = dict(ppc, loo_pit=True)
    for rows in [int(r) for r in args.rows.split(",")]:
        def timed(spec):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = s.sample_summary(rows, ppc=spec)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), out

        for _ in range(args.warmup):
            timed(ppc)
            timed(pit)
        plain, withp, n_chunks = [], [], []
        res = None
        for _ in range(args.reps):
            plain.append(timed(ppc)[0])
            chunks.clear()
            ms, res = timed(pit)
            withp.append(ms)
            n_chunks.append(len(chunks))
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.sample_summary(rows, ppc=pit)
            torch.cuda.synchronize()
        per_kernel = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                per_kernel[e.key] = per_kernel.get(e.key, 0.0) + us / 1e3
        own = {k: v for k, v in per_kernel.items() if "amwg_loo_pit_" in k}
        if len(own) < 2:
            raise RuntimeError("the profile lacks the LOO-PIT kernels: %s" % sorted(per_kernel))
        top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:14]
        lp = res["ppc"]["loo_pit"]
        print(json.dumps({
            "workload": "config 2: N=%d, %d chains, burn(%d), sample_summary(%d), ppc over %d points with and without loo_pit"
                        % (N, args.chains, args.burn, rows, N),
            "gpu": name, "power_limit_w": limit, "draws": rows * args.chains,
            "ms_per_call_ppc": round(float(np.median(plain)), 3), "ms_per_call_ppc_loo_pit": round(float(np.median(withp)), 3),
            "ms_loo_pit_extra": round(float(np.median(withp)) - float(np.median(plain)), 3), "reps": args.reps,
            "chunks": int(np.median(n_chunks)),
            "profiled_ms_loo_pit_kernels": {k[:90]: round(v, 3) for k, v in own.items()},
            "profiled_call_ms_by_kernel": {k[:90]: round(v, 3) for k, v in top},
            "mean_pit": float(np.mean(lp["pit"])), "n_high_k": lp["n_high_k"],
        }), flush=True)


if __name__ == "__main__":
    main()
