"""bench.py, the parts that run without a GPU: the reference arm (`--impl reference`: the CPU restatement of mcmc.js on the host
cores) prints ONE JSON line with the keys the driver's contract names, for the same metric / config / unit as the GPU arm; and the
GPU arm refuses to run without a GPU instead of falling back to anything. On a GPU: what `--dump-outputs` writes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, timeout=240):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, cwd=ROOT, capture_output=True, text=True, timeout=timeout)


def test_reference_arm_prints_the_contract_line():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "1"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 1 and d["warmup"] == 1
    assert d["metric"].startswith("posterior draws/sec") and d["unit"] == "draws/s" and d["higher_is_better"] is True
    assert d["dtype"] == "f64" and d["data"] == "synthetic" and d["vs_baseline"] is None
    assert "config 2" in d["config"]["workload"] and "model" not in d["config"]
    assert d["value"] > 0 and d["ms_per_step"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "draws per step" in cb["sample"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["unit"] == d["unit"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0


def _bench_module():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__ as graft
    import bench
    return graft.load_package(), bench


@pytest.mark.gpu
def test_dump_outputs_holds_the_last_timed_steps_draws(tmp_path):
    """--dump-outputs DIR: per parameter, what sample() returns for the last timed step, identical for identical arguments. A fresh
    sampler with bench's seed and data, burned in as bench burns it and sampling warmup + steps blocks, ends on the same block."""
    warmup, steps, iters, burn, chains = 1, 2, 3, 10, 4096
    got = []
    for k in range(2):
        d = tmp_path / f"run{k}"
        r = _run(["--chains", str(chains), "--iters", str(iters), "--burn", str(burn), "--steps", str(steps), "--warmup", str(warmup),
                  "--no-cpu", "--dump-outputs", str(d)])
        assert r.returncode == 0, r.stderr[-2000:]
        got.append({n: np.load(d / f"{n}.npy") for n in ("mu", "sigma")})
    pkg, bench = _bench_module()
    cfg = bench.Config(2, pkg.ld, pkg.mcmc)
    s = pkg.mcmc.AmwgSampler(cfg.params, cfg.log_post, cfg.data, {"chains": chains, "seed": 0, "device": 0})
    s.burn(burn)
    for _ in range(warmup + steps):
        last = s.sample(iters)
    s.close()
    for n in cfg.params:
        assert got[0][n].dtype == np.float64 and got[0][n].shape == (iters, chains)
        assert np.array_equal(got[0][n].view(np.uint64), got[1][n].view(np.uint64))
        assert np.array_equal(got[0][n].view(np.uint64), np.asarray(last[n], dtype=np.float64).view(np.uint64)), n


@pytest.mark.gpu
def test_dump_outputs_writes_a_fixed_sample_of_chains_above_the_byte_limit(tmp_path):
    """Above the byte limit the dump holds a seeded, sorted sample of the chains, each chain's own column of every row."""
    import torch
    pkg, bench = _bench_module()
    cfg = bench.Config(2, pkg.ld, pkg.mcmc)
    s = pkg.mcmc.AmwgSampler(cfg.params, cfg.log_post, cfg.data, {"chains": 64, "seed": 0, "device": 0})   # supplies the output shapes
    iters, entries, C, keep = 3, 2, 5000, 1000
    r_, e_, c_ = torch.meshgrid(torch.arange(iters), torch.arange(entries), torch.arange(C), indexing="ij")
    dev_out = (r_.double() * 1e6 + e_.double() * 1e5 + c_.double()).cuda()       # the value names its (row, entry, chain)
    limit = keep * iters * entries * 8
    bench.dump_outputs(str(tmp_path), s, cfg, dev_out, max_bytes=limit)
    s.close()
    pick = bench.dump_chains(C, iters * entries * 8, limit)
    assert len(pick) == keep and np.all(np.diff(pick) > 0) and pick[-1] < C
    assert np.array_equal(pick, bench.dump_chains(C, iters * entries * 8, limit))
    rows = np.arange(iters)[:, None] * 1e6
    assert np.array_equal(np.load(tmp_path / "mu.npy"), rows + pick[None, :])
    assert np.array_equal(np.load(tmp_path / "sigma.npy"), rows + 1e5 + pick[None, :])


def test_gpu_arm_needs_a_gpu():
    import torch
    if torch.cuda.is_available():
        return                                       # on a GPU box the arm itself is what the driver runs
    r = _run(["--steps", "1", "--warmup", "3", "--no-cpu"], timeout=120)
    assert r.returncode != 0
    assert not [l for l in r.stdout.splitlines() if l.startswith("{")]      # no number without the CUDA path
