"""Cost of the posterior covariance of sample_summary on one GPU, at two sizes:
  config 2: Normal(mu, sigma), N = 1024 data points, 2^20 chains (E = 2 entries);
  config 4: hierarchical Normal, mu dim [64] + sigma, 64 groups x 1024 points, 2^16 chains (E = 65 entries).
Each: burn(1000), then sample_summary(100) alternating with sample_summary(100, covariance=True).

Prints one JSON line per config: ms per call of each (median of --reps after --warmup of each), the time of the reducer
(CUDA events around CudaBlockReducer.comoments, which includes the copy of the record to the host), the bytes it must read
(the block twice: once for the chain means, once for the Gram matrix), the tensor-core flop of the tiles it forms (2 x 64
multiply-adds per tile per four draws, padded blocks included) and the achieved HBM rate. The card's name and power limit are
read in the same run."""
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


def sampler(pkg, config, chains):
    mcmc, ld = pkg.mcmc, pkg.ld
    if config == 2:
        def log_post(state, data):
            lp = 0
            lp += ld.norm(state.mu, 0, 100)
            lp += ld.unif(state.sigma, 0, 100)
            for i in range(len(data)):
                lp += ld.norm(data[i], state.mu, state.sigma)
            return lp
        data = np.random.default_rng(1024).normal(184.5, 4.5, 1024).tolist()
        return mcmc.AmwgSampler({"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}, log_post, data,
                                {"chains": chains, "seed": 1, "device": 0})
    J, per = 64, 1024
    g = np.repeat(np.arange(J), per)
    y = np.random.default_rng(64).normal(100, 20, J)[g] + np.random.default_rng(65).normal(0, 5, J * per)

    def log_post(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        return lp
    return mcmc.AmwgSampler({"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}, log_post,
                            {"y": y, "g": g.astype(np.float64)}, {"chains": chains, "seed": 1, "device": 0})


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
    method = summary.CudaBlockReducer.comoments

    def timed_comoments(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = method(self, *a, **k)
        e1.record()
        e1.synchronize()
        reducer_ms.append(e0.elapsed_time(e1))
        return out
    summary.CudaBlockReducer.comoments = timed_comoments
    name, limit = card()
    for config in [int(c) for c in args.configs.split(",")]:
        chains = (1 << 20) if config == 2 else (1 << 16)
        s = sampler(pkg, config, chains)
        s.burn(args.burn)

        def timed(cov):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = s.sample_summary(args.rows, covariance=cov)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), out

        for _ in range(args.warmup):
            timed(None)
            timed(True)
        reducer_ms.clear()
        plain, withcov = [], []
        for _ in range(args.reps):
            plain.append(timed(None)[0])
            ms, res = timed(True)
            withcov.append(ms)
        E = 2 if config == 2 else 65
        nb = -(-E // 8)
        tiles = nb * (nb + 1) // 2
        block_bytes = args.rows * E * chains * 8
        read_bytes = 2 * block_bytes + 2 * E * chains * 8                 # the block twice, the chain means twice
        flop = 128 * tiles * (args.rows + 1) * chains                     # one DMMA (8 x 8 x 4 multiply-adds) per tile per four draws
        ms_red = float(np.median(reducer_ms))
        cov = res["covariance"]
        print(json.dumps({
            "workload": "config %d: E=%d, %d chains, burn(%d), sample_summary(%d), covariance=True" % (config, E, chains, args.burn, args.rows),
            "gpu": name, "power_limit_w": limit, "block_gb": round(block_bytes / 1e9, 3),
            "ms_per_call_plain": round(float(np.median(plain)), 3), "ms_per_call_covariance": round(float(np.median(withcov)), 3),
            "ms_covariance_extra": round(float(np.median(withcov)) - float(np.median(plain)), 3), "reps": args.reps,
            "ms_reducer": round(ms_red, 3), "read_gb": round(read_bytes / 1e9, 3), "hbm_tb_per_s": round(read_bytes / 1e9 / ms_red, 3),
            "tensor_gflop": round(flop / 1e9, 2), "tensor_tflop_per_s": round(flop / 1e9 / ms_red, 2), "tiles": tiles,
            "rhat_multivariate": cov["rhat_multivariate"], "max_abs_offdiag_corr": float(np.max(np.abs(cov["corr"] - np.eye(E)))),
        }), flush=True)
        del s
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
