"""Cost of the nested R-hat of sample_summary on one GPU, at two sizes:
  config 2: Normal(mu, sigma), N = 1024 data points, 2^20 chains (E = 2 entries), superchains of 64;
  config 4: hierarchical Normal, mu dim [64] + sigma, 64 groups x 1024 points, 2^16 chains (E = 65 entries), superchains of 16.
Each: burn(1000), then sample_summary(100) alternating with sample_summary(100, nested=M).

Prints one JSON line per config: ms per call of each (median of --reps after --warmup of each), the time of the reducer
(CUDA events around CudaBlockReducer.nested, which includes the copy of the records to the host), the bytes it must read (the
block twice, for the chain means and the chain M2, and the per-chain records written once and read once) and the achieved HBM
rate. The card's name and power limit are read in the same run."""
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
    ap.add_argument("--configs", default="2,4")
    ap.add_argument("--rows", type=int, default=100)
    ap.add_argument("--burn", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    pkg = graft.load_package()
    summary = pkg.summary
    reducer_ms = []
    method = summary.CudaBlockReducer.nested

    def timed_nested(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = method(self, *a, **k)
        e1.record()
        e1.synchronize()
        reducer_ms.append(e0.elapsed_time(e1))
        return out
    summary.CudaBlockReducer.nested = timed_nested
    name, limit = card()
    for config in [int(c) for c in args.configs.split(",")]:
        chains, M = ((1 << 20), 64) if config == 2 else ((1 << 16), 16)
        s = sampler(pkg, config, chains)
        s.burn(args.burn)

        def timed(nested):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = s.sample_summary(args.rows, nested=nested)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), out

        for _ in range(args.warmup):
            timed(None)
            timed(M)
        reducer_ms.clear()
        plain, withn = [], []
        for _ in range(args.reps):
            plain.append(timed(None)[0])
            ms, res = timed(M)
            withn.append(ms)
        E = 2 if config == 2 else 65
        block_bytes = args.rows * E * chains * 8
        read_bytes = 2 * block_bytes + 2 * 16 * E * chains                # the block twice; the chain records written and read
        ms_red = float(np.median(reducer_ms))
        rn = [float(np.max(res[k]["rhat_nested"])) for k in res]
        print(json.dumps({
            "workload": "config %d: E=%d, %d chains, burn(%d), sample_summary(%d), nested=%d" % (config, E, chains, args.burn, args.rows, M),
            "gpu": name, "power_limit_w": limit, "block_gb": round(block_bytes / 1e9, 3),
            "ms_per_call_plain": round(float(np.median(plain)), 3), "ms_per_call_nested": round(float(np.median(withn)), 3),
            "ms_nested_extra": round(float(np.median(withn)) - float(np.median(plain)), 3), "reps": args.reps,
            "ms_reducer": round(ms_red, 3), "read_gb": round(read_bytes / 1e9, 3), "hbm_tb_per_s": round(read_bytes / 1e9 / ms_red, 3),
            "max_rhat_nested": max(rn),
        }), flush=True)
        del s
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
