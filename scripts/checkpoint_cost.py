"""Cost of sampler.checkpoint() and sampler.restore() on one GPU at the BASELINE sizes of config 2 (Normal(mu, sigma), N = 1024,
2^20 chains) and config 4 (hierarchical Normal, D = 65, N = 65536, 2^16 chains), with the models and data bench.py runs.

Per config: a short burn, then --warmup calls of each, then the median of --reps calls (host clock around the call; both calls
block until the device is done). restore() goes into a second handle of the same model. Prints one JSON line with the image
size, the times and the card's name and power limit, read in the same run (nvidia-smi --query-gpu, read only)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402
import bench  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip()


def median_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="2,4")
    ap.add_argument("--burn", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    pkg = graft.load_package()
    mcmc, ld = pkg.mcmc, pkg.ld
    res = {"card": card()}
    for k in [int(v) for v in args.configs.split(",")]:
        cfg = bench.Config(k, ld, mcmc)
        opts = {"chains": cfg.chains, "seed": 1, "device": 0}
        a = mcmc.AmwgSampler(cfg.params, cfg.log_post, cfg.data, dict(opts))
        b = mcmc.AmwgSampler(cfg.params, cfg.log_post, cfg.data, dict(opts, seed=2))
        a.burn(args.burn)
        img = a.checkpoint()
        save = median_ms(a.checkpoint, args.warmup, args.reps)
        load = median_ms(lambda: b.restore(img), args.warmup, args.reps)
        res["config %d" % k] = {"chains": cfg.chains, "image_bytes": len(img), "checkpoint_ms": round(save, 2), "restore_ms": round(load, 2),
                                "sweep_kernel": a.jit_status()[1]}
        a.close()
        b.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
