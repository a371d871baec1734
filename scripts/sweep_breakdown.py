"""Where config 2's sweep time goes: the specialised statistics sweep of bench.py's config-2 model (Normal(mu, sigma), synthetic data
drawn like bench.py's) at 2^20 chains and N data points, for N in --points (default 64, 512, 1024, 2048).

Per N: a short burn, then --warmup launches of --sweeps sweeps each, then the median of --reps launches; the time is the sweep
kernel's own, measured with CUDA events (sampler.last_sweep_kernel_ms()). The per-point cost is the slope between the largest N
that keeps 8 CTAs per SM and N = 64; the O(1) part is the N = 64 time less 64 points at that slope. Prints a table, then one JSON
line with the times and the card's name and power limit, read in the same run (nvidia-smi --query-gpu, read only)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30)
    return out.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", default="64,512,1024,2048")
    ap.add_argument("--chains", type=int, default=1 << 20)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--burn", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=6)
    args = ap.parse_args()
    pkg = graft.load_package()
    mcmc, ld, ffi = pkg.mcmc, pkg.ld, pkg._ffi
    L = ffi.lib()
    import torch
    params = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}

    def log_post(state, data):                        # bench.py config 2 (README.md:26-36)
        lp = 0
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(len(data)):
            lp += ld.norm(data[i], state.mu, state.sigma)
        return lp

    rows = []
    for n in [int(v) for v in args.points.split(",")]:
        x = np.random.default_rng(1024).normal(184.5, 4.5, n)
        s = mcmc.AmwgSampler(params, log_post, x.tolist(), {"chains": args.chains, "seed": 0})
        assert s.jit_status()[0], s.jit_status()
        src = s.jit_compile_check()[2]
        shape = {k: v for k, v in (ln.split()[1:] for ln in src.splitlines() if ln.startswith("#define J") and len(ln.split()) == 3)}
        s.burn(args.burn)
        mon = np.arange(2, dtype=np.int32)
        out = torch.empty((args.sweeps, 2, s.local_chains), dtype=torch.float64, device="cuda:0")

        def launch():
            ffi.check(L.amwg_sample_device(s._handle, args.sweeps, 1, mon.ctypes.data_as(C.POINTER(C.c_int32)), 2, out.data_ptr()))
            return s.last_sweep_kernel_ms()
        for _ in range(args.warmup):
            launch()
        ts = sorted(launch() for _ in range(args.reps))
        rows.append({"N": n, "ms_per_100_sweeps": ts[len(ts) // 2] * 100.0 / args.sweeps, "min": ts[0] * 100.0 / args.sweeps,
                     "max": ts[-1] * 100.0 / args.sweeps, "threads": int(shape["JTHREADS"]), "ctas_per_sm": int(shape["JMINB"])})
        del out
        s.close()
    eight = [r for r in rows if r["ctas_per_sm"] == 8]
    lo = min(eight, key=lambda r: r["N"])
    hi = max(eight, key=lambda r: r["N"])
    per_point = (hi["ms_per_100_sweeps"] - lo["ms_per_100_sweeps"]) / (hi["N"] - lo["N"]) if hi["N"] > lo["N"] else float("nan")
    fixed = lo["ms_per_100_sweeps"] - lo["N"] * per_point
    print(f"{'N':>6} {'ms / 100 sweeps':>16} {'(min-max)':>16} {'CTA x per SM':>13}")
    for r in rows:
        print(f"{r['N']:>6} {r['ms_per_100_sweeps']:>16.2f} {r['min']:>7.2f}-{r['max']:<8.2f} {r['threads']:>6} x {r['ctas_per_sm']}")
    print(f"per point: {1e3 * per_point:.2f} us per 100 sweeps (N = {lo['N']}..{hi['N']}); O(1) part: {fixed:.2f} ms per 100 sweeps")
    print(json.dumps({"card": card(), "chains": args.chains, "rows": rows, "us_per_point_per_100_sweeps": 1e3 * per_point,
                      "o1_ms_per_100_sweeps": fixed}))


if __name__ == "__main__":
    main()
