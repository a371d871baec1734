"""Multi-GPU plumbing: one process per GPU (torch.distributed), chains sharded, no data-path collective.

Chains are independent (the reference runs exactly one, mcmc.js:940-966), so the path shards embarrassingly: rank r
owns the contiguous block of global chain ids [r*C/G, (r+1)*C/G).  The Philox stream is keyed by the GLOBAL chain id,
so the draws do not depend on G.  The only collective is the final all-gather of the sample blocks in `sample()`
(NCCL over NVLink on GPUs; gloo in the CPU tests).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Tuple

import numpy as np


def world() -> Tuple[int, int]:
    """(rank, world_size) from torch.distributed if initialised, else from the torchrun environment."""
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except Exception:
        pass
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


def shard_bounds(n_chains: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous block of rank `rank`: (first_chain, count). Remainder chains go to the lowest ranks."""
    base, rem = divmod(int(n_chains), int(world_size))
    first = rank * base + min(rank, rem)
    return first, base + (1 if rank < rem else 0)


def ladder_shard_error(n_chains: int, world_size: int, K: int):
    """None when every rank's shard (shard_bounds) starts at a multiple of K and holds a multiple of K chains, so that no ladder of K
    tempered chains straddles two GPUs (DESIGN.md §2 "Tempered ladders"); otherwise the message options.temperatures raises."""
    for r in range(int(world_size)):
        first, count = shard_bounds(n_chains, r, world_size)
        if first % K or count % K:
            return ("options.temperatures: with options.distributed every GPU must hold whole ladders; %d chains over %d GPUs give "
                    "rank %d the chains [%d, %d), which is not a multiple of %d" % (n_chains, world_size, r, first, first + count, K))
    return None


def check_ladder_shards(n_chains: int, K: int) -> None:
    from .tracer import JsThrow
    err = ladder_shard_error(n_chains, world()[1], K)
    if err:
        raise JsThrow(err)


def shard_chains(n_chains: int) -> Tuple[int, int]:
    rank, ws = world()
    return shard_bounds(n_chains, rank, ws)


def local_chain_rows(values: np.ndarray, first_chain: int, count: int) -> np.ndarray:
    """This rank's chains [first_chain, first_chain + count) of a per-chain array over all global chains (chain axis first)."""
    if values.shape[0] < first_chain + count:
        raise ValueError("the array covers %d chains, the shard ends at chain %d" % (values.shape[0], first_chain + count))
    return values[first_chain:first_chain + count]


def total_over_ranks(n: int, device: int = 0) -> int:
    """The sum of an integer over all ranks: one tiny all-reduce (on the GPU under NCCL, on the CPU under gloo), so that every rank
    takes the same decision from it."""
    import torch
    import torch.distributed as dist
    dev = torch.device("cuda", device) if dist.get_backend() == "nccl" else torch.device("cpu")
    t = torch.tensor([int(n)], dtype=torch.int64, device=dev)
    dist.all_reduce(t)
    return int(t.item())


def _rank_major_to_chain_axis(stacked, ws: int, rows: int, entries: int, cmax: int, counts):
    """`stacked[ws][rows][entries][cmax]` (what one collective delivers) -> `[rows, entries, sum(counts)]`, chains in global order:
    one strided device copy (the kernel's layout keeps the chain axis fastest, so the rank axis has to move inside)."""
    import torch
    full = stacked.view(ws, rows, entries, cmax).permute(1, 2, 0, 3).reshape(rows, entries, ws * cmax)
    if len(set(counts)) == 1:
        return full
    keep = torch.cat([torch.arange(k * cmax, k * cmax + c, device=full.device) for k, c in enumerate(counts)])
    return full.index_select(-1, keep)


def _padded(local, cmax: int):
    import torch
    if local.shape[-1] == cmax:
        return local.contiguous()
    pad = torch.zeros(local.shape[:-1] + (cmax - local.shape[-1],), dtype=local.dtype, device=local.device)
    return torch.cat([local, pad], dim=-1).contiguous()             # collectives want equal sizes: pad to the largest shard


def all_gather_chain_axis(local, counts):
    """All-gather `local[rows, entries, c_rank]` over its last (chain) axis -> `[rows, entries, sum(counts)]`, chains in
    global order. ONE collective per call (rank-major staging block), then one strided copy that moves the rank axis next to the
    chain axis. CUDA tensors over NCCL (NVLink), CPU tensors over gloo."""
    import torch
    import torch.distributed as dist
    ws = dist.get_world_size()
    rows, entries = local.shape[0], local.shape[1]
    cmax = max(counts)
    local = _padded(local, cmax)
    stacked = torch.empty((ws, rows, entries, cmax), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(stacked.view(-1), local.view(-1))
    return _rank_major_to_chain_axis(stacked, ws, rows, entries, cmax, counts)


def gather_chain_axis_to_root(local, counts, root: int = 0):
    """Gather `local[rows, entries, c_rank]` over the chain axis onto rank `root` only (returns None elsewhere): one collective
    per call. The host-memory-friendly variant when one process collects the draws."""
    import torch
    import torch.distributed as dist
    ws, rank = dist.get_world_size(), dist.get_rank()
    rows, entries = local.shape[0], local.shape[1]
    cmax = max(counts)
    local = _padded(local, cmax)
    if rank == root:
        stacked = torch.empty((ws, rows, entries, cmax), dtype=local.dtype, device=local.device)
        dist.gather(local, list(stacked.unbind(0)), dst=root)
        return _rank_major_to_chain_axis(stacked, ws, rows, entries, cmax, counts)
    dist.gather(local, None, dst=root)
    return None


def _parse_cpulist(text: str):
    cpus = []
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.extend(range(int(a), int(b) + 1))
        else:
            cpus.append(int(part))
    return cpus


def bind_to_gpu_numa_node(device: int):
    """Pin this process (and therefore its page-locked allocations: first touch, local policy) to the CPUs of the NUMA node the
    GPU hangs off. One process per GPU copies its own shard to its own host memory; with eight ranks left floating, most of those
    copies cross the socket interconnect (round-1 measurement: 213 GB/s aggregate instead of 8 x 38 GB/s). Call before the first
    pinned allocation. Returns a small record for the bench line, or None when the topology cannot be read (nothing is changed)."""
    import subprocess
    try:
        bus = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=pci.bus_id", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip().lower()
        if not bus:
            return None
        if len(bus.split(":")[0]) == 8:                          # nvidia-smi prints an 8-digit domain, sysfs a 4-digit one
            bus = bus[4:]
        base = "/sys/bus/pci/devices/" + bus
        with open(base + "/local_cpulist") as f:
            cpus = _parse_cpulist(f.read())
        node = -1
        try:
            with open(base + "/numa_node") as f:
                node = int(f.read().strip())
        except Exception:
            pass
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return {"gpu": device, "numa_node": node, "cpus": len(allowed)}
    except Exception:
        return None


def sample_and_gather(sampler, n: int, thin: int, mon: np.ndarray, rows: int) -> np.ndarray:
    """Distributed sample(): this rank's shard is sampled in row chunks; while chunk k+1 is being computed, chunk k is collected
    over the chain axis (NCCL over NVLink) and copied into a pinned host buffer on a side stream. `sampler.gather`: "all"
    (default; every rank returns all chains), "root" (rank 0 returns all chains, the others their own shard), "none" (own shard)."""
    import torch
    import torch.distributed as dist
    from . import _ffi
    from .mcmc import _pinned_empty
    from .tracer import JsThrow
    if not (dist.is_available() and dist.is_initialized()):
        raise JsThrow("options.distributed needs an initialised torch.distributed process group")
    L = _ffi.lib()
    dev = torch.device("cuda", sampler.device)
    ws, rank = dist.get_world_size(), dist.get_rank()
    K = sampler.n_chains // sampler.cold_chains                 # a tempered sampler records the T = 1 chain of every ladder
    counts = [shard_bounds(sampler.n_chains, r, ws)[1] // K for r in range(ws)]
    mode = getattr(sampler, "gather", "all")
    collect = mode == "all" or mode == "root"
    out_chains = sampler.cold_chains if (mode == "all" or (mode == "root" and rank == 0)) else sampler.local_cold
    host = _pinned_empty((rows, len(mon), out_chains))
    host_t = torch.from_numpy(host)
    monp = mon.ctypes.data_as(C.POINTER(C.c_int32))
    chunk_rows = max(1, min(rows, 10))
    side = torch.cuda.Stream(device=dev)
    done_events = []
    row0 = 0
    while row0 < rows:
        r = min(chunk_rows, rows - row0)
        n_chunk = min(n - row0 * thin, r * thin)               # sample(a) then sample(b) == sample(a+b) when a is a multiple of thin
        local = torch.empty((r, len(mon), sampler.local_cold), dtype=torch.float64, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        rc = L.amwg_sample_device(sampler._handle, n_chunk, thin, monp, len(mon), local.data_ptr())      # blocks until the chunk is in HBM
        if rc != 0:
            raise JsThrow(L.amwg_last_error().decode())
        with torch.cuda.stream(side):                            # collect + D2H of this chunk overlap the next chunk's sweeps
            if mode == "all":
                full = all_gather_chain_axis(local, counts)
            elif mode == "root":
                full = gather_chain_axis_to_root(local, counts, 0)
                if full is None:
                    full = local
            else:
                full = local
            host_t[row0:row0 + r].copy_(full, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
            done_events.append((ev, local, full))                # keep the device buffers alive until the copy has finished
        row0 += r
    side.synchronize()
    del done_events, collect
    return host
