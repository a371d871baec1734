"""The launch shape of the specialised sweeps, restated -- test infrastructure, CPU only.

choose_shape (csrc/amwg_jit.cuh) picks, per handle, the CTA size, the resident CTAs per SM and whether each chain's working set
lives in shared memory, from the handle's chain count and the device's SM count. Each shape is compiled in (__launch_bounds__,
JWS_SMEM / JWS_OFF), so each is a kernel of its own. This module restates the planner line for line, so that tests can list every
shape a model reaches over a range of chain counts and the smallest ragged chain count (C % threads != 0) that reaches it.

  plan(n_chains, sm_count, off, per_thread)   -> (threads, ctas_per_sm, ws_smem), as choose_shape decides
  inputs(sampler)                             -> PlanInputs of a model, read from its lowered program and one jit_compile_check
  shapes(pi, sm_count, lo, hi)                -> {(threads, ctas_per_sm, ws_smem): smallest ragged chain count in [lo, hi]}
  defines(src) / smem_declared(msg)           the generated #defines and the dynamic shared memory a launch declares
  count_with(pi, sm_count, threads, at_least) the smallest chain count from at_least on that plans `threads`-thread CTAs
"""
import math
import re
from dataclasses import dataclass

import numpy as np

CANDIDATES = (128, 64, 96, 160, 192, 224, 256)       # choose_shape's order: 128 is the default, the others must beat it
MARGIN = 0.15                                        # by this much in `eff`
WS_SMEM_LIMIT = 20 * 1024                            # kJitWsSmemLimit
SMEM_PER_SM = 227 * 1024                             # the opt-in shared memory of an sm_90 SM, as the planner counts it
RESERVED_PER_CTA = 1024                              # what the driver reserves per CTA
THREADS_PER_SM = 2048
MAX_CTAS = 8


def pad16(b):
    return (int(b) + 15) // 16 * 16


def plan(n_chains, sm_count, off, per_thread):
    """choose_shape, line for line -> (threads, ctas_per_sm, ws_smem)"""
    base = off
    best_t, best_r, best_ws = 0, 1, 0
    best_eff = -1.0
    for t in CANDIDATES:
        need = pad16(per_thread * t)
        ws_smem = 1 if need <= WS_SMEM_LIMIT else 0
        smem = max(pad16(base) + (need if ws_smem else 0), 16)
        r_max = min(min(SMEM_PER_SM // (smem + RESERVED_PER_CTA), THREADS_PER_SM // t), MAX_CTAS)
        if r_max < 1:
            continue
        ctas = float(math.ceil(n_chains / t))
        cap = float(sm_count * r_max)
        if ctas <= cap:
            per_sm = float(math.ceil(ctas / sm_count))
            eff = (n_chains / sm_count) / (per_sm * t)
            r_need = int(per_sm)
        else:
            eff = ctas / (math.ceil(ctas / cap) * cap) * (n_chains / (ctas * t))
            r_need = r_max
        if eff > best_eff + (0.0 if best_t == 0 else MARGIN):
            best_eff, best_t, best_r, best_ws = eff, t, r_need, ws_smem
    assert best_t, "no launch shape fits"
    return best_t, max(1, best_r), best_ws


def _plan_many(counts, sm_count, off, per_thread):
    """plan() over an array of chain counts at once (the same fp64 operations, elementwise) -> threads, ctas_per_sm, ws_smem arrays"""
    n = np.asarray(counts, dtype=np.float64)
    best_t = np.zeros(n.shape, np.int64)
    best_r = np.ones(n.shape, np.int64)
    best_ws = np.zeros(n.shape, np.int64)
    best_eff = np.full(n.shape, -1.0)
    for t in CANDIDATES:
        need = pad16(per_thread * t)
        ws_smem = 1 if need <= WS_SMEM_LIMIT else 0
        smem = max(pad16(off) + (need if ws_smem else 0), 16)
        r_max = min(min(SMEM_PER_SM // (smem + RESERVED_PER_CTA), THREADS_PER_SM // t), MAX_CTAS)
        if r_max < 1:
            continue
        ctas = np.ceil(n / t)
        cap = float(sm_count * r_max)
        fits = ctas <= cap
        per_sm = np.ceil(ctas / sm_count)
        eff = np.where(fits, (n / sm_count) / (per_sm * t), ctas / (np.ceil(ctas / cap) * cap) * (n / (ctas * t)))
        r_need = np.where(fits, per_sm, r_max).astype(np.int64)
        take = eff > best_eff + np.where(best_t == 0, 0.0, MARGIN)
        best_eff = np.where(take, eff, best_eff)
        best_t = np.where(take, t, best_t)
        best_r = np.where(take, r_need, best_r)
        best_ws = np.where(take, ws_smem, best_ws)
    return best_t, np.maximum(best_r, 1), best_ws


@dataclass(frozen=True)
class PlanInputs:
    full: bool          # the full-program sweep (amwg_jit_full_kernel.cuh) instead of the statistics sweep
    D: int              # components
    NT: int             # term-cache slots (statistics sweep)
    off: int            # shared memory planned before the working set: columns, ring, Bernoulli masks (pad16 is all the planner reads)

    @property
    def per_thread(self):
        """bytes of one chain's working set: [tval NT | tcand NT | bprop D | bcoin D | state D] doubles + vseq D u16, or the state alone"""
        return 8 * self.D if self.full else 8 * (2 * self.NT + 3 * self.D) + 2 * self.D


def defines(src):
    out = {}
    for ln in src.splitlines():
        if ln.startswith("#define ") and len(ln.split()) == 3:
            _, k, v = ln.split()
            out[k] = v
    return out


def smem_declared(msg):
    """the dynamic shared memory a launch of the compiled specialisation declares (amwg_jit_compile_check's message)"""
    m = re.search(r"(\d+) B shared memory", msg)
    assert m, msg
    return int(m.group(1))


def shape_of(dfn):
    """(threads, ctas_per_sm, ws_smem) of a generated source's #defines"""
    return int(dfn["JTHREADS"]), int(dfn["JMINB"]), int(dfn["JWS_SMEM"])


def inputs(sampler, n_chains=4096):
    """A model's plan inputs: D and NT from the lowered program, `off` from one jit_compile_check (the planner puts the working
    set at pad16(off) = JWS_OFF when it goes to shared memory; otherwise the declared shared memory is max(off, 16))."""
    rc, msg, src = sampler.jit_compile_check(n_chains)
    assert rc == 0, msg
    dfn = defines(src)
    off = int(dfn["JWS_OFF"]) if dfn["JWS_SMEM"] == "1" else smem_declared(msg)
    return PlanInputs(full=dfn.get("JFULL") == "1", D=int(dfn["JD"]), NT=int(dfn.get("JNT", 0)), off=off)


def shapes(pi, sm_count, lo, hi):
    """{(threads, ctas_per_sm, ws_smem): the smallest chain count C in [lo, hi] with C % threads != 0 that plans it}"""
    counts = np.arange(lo, hi + 1, dtype=np.int64)
    t, r, ws = _plan_many(counts, sm_count, pi.off, pi.per_thread)
    out = {}
    ragged = counts % t != 0
    for key in sorted(set(zip(t[ragged].tolist(), r[ragged].tolist(), ws[ragged].tolist()))):
        sel = ragged & (t == key[0]) & (r == key[1]) & (ws == key[2])
        out[key] = int(counts[np.argmax(sel)])
    return out


def count_with(pi, sm_count, threads, at_least, limit=1 << 22):
    """the smallest chain count >= at_least that plans `threads`-thread CTAs"""
    counts = np.arange(at_least, at_least + limit, dtype=np.int64)
    t, _, _ = _plan_many(counts, sm_count, pi.off, pi.per_thread)
    hit = np.flatnonzero(t == threads)
    assert hit.size, (threads, at_least)
    return int(counts[hit[0]])
