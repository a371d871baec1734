"""The launch shapes of the specialised sweeps, on the CPU: the planner's restatement (tests/launch_shape.py) against what
jit_compile_check generates, and the shared-memory layout of every shape the planner reaches.

Each shape (CTA size, CTAs per SM, working set in shared or global memory) is a kernel of its own: __launch_bounds__(JTHREADS,
JMINB) and the JWS_SMEM / JWS_OFF layout are compiled in. jit_compile_check plans for the 132 SMs of an H100 SXM. The chain counts
below are, per model, the smallest ragged count of every shape the restatement finds in [1, 300000] chains, plus 2^20 (config 2's
bench count) and a few counts where the planner moves between shapes."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import launch_shape as ls
import models
from conftest import config2_data, config3_data

SM = 132
LO, HI = 1, 300000


def _hier(J, per, seed=5):
    sizes = np.broadcast_to(per, (J,))
    g = np.repeat(np.arange(J), sizes)
    mu = np.random.default_rng(seed).normal(100, 20, J)
    y = mu[g] + np.random.default_rng(seed + 1).normal(0, 5, g.size)
    P = {"mu": {"type": "real", "dim": [J], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    return P, {"y": y.tolist(), "g": g.astype(float).tolist()}


def _sampler(pkg, name):
    ld, mcmc = pkg.ld, pkg.mcmc
    o = {"chains": 4096, "_model_only": True}
    if name == "config2":           # BASELINE config 2: Normal, 1024 points, one resident column, the statistics sweep
        return mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(ld), config2_data().tolist(), o)
    if name == "config4":           # BASELINE config 4: 64 groups x 1024 points, the streamed column and its TMA ring
        P, d = _hier(64, 1024)
        return mcmc.AmwgSampler(P, models.hier_norm_post(ld), d, o)
    if name == "spike":             # spike-and-slab Bernoulli on 256 points: the full-program sweep and its bit masks
        return mcmc.AmwgSampler(models.PARAMS_SPIKE, models.spike_bern(ld, mcmc), {"x": config3_data().tolist()}, o)
    raise KeyError(name)


MODELS = ["config2", "config4", "spike"]
EXTRA_COUNTS = (2 ** 20, 12672, 147841, 152069, 202756)      # config 2's bench count and counts where the shape changes


@pytest.fixture(scope="module")
def compiled(pkg):
    """{model: (PlanInputs, {chain count: (message, source)})}: one compilation per (model, count), eight at a time"""
    out = {}
    for name in MODELS:
        s = _sampler(pkg, name)
        pi = ls.inputs(s)
        counts = sorted(set(ls.shapes(pi, SM, LO, HI).values()) | set(EXTRA_COUNTS))

        def check(C, s=s):
            rc, msg, src = s.jit_compile_check(C)
            assert rc == 0, (C, msg)
            return C, (msg, src)
        with ThreadPoolExecutor(8) as ex:
            out[name] = (pi, dict(ex.map(check, counts)))
    return out


@pytest.mark.parametrize("name", MODELS)
def test_the_restated_planner_chooses_what_the_generator_compiles(compiled, name):
    pi, built = compiled[name]
    reached = set()
    for C, (msg, src) in built.items():
        got = ls.shape_of(ls.defines(src))
        assert ls.plan(C, SM, pi.off, pi.per_thread) == got, (name, C, got)
        assert f"{got[0]} threads x {got[1]} CTAs/SM" in msg, (name, C, msg)
        reached.add(got)
    want = set(ls.shapes(pi, SM, LO, HI))
    assert want <= reached, (name, sorted(want - reached))
    # the shapes this test exists for: CTA sizes other than 128, and config 2's working set in global memory
    assert {t for t, _, _ in want} >= {64, 96, 128, 160}, sorted(want)
    if name == "config2":
        assert (192, 6, 0) in want and (224, 7, 0) in want and (160, 8, 1) in want
    if name == "config4":
        assert (256, 5, 0) in want


def test_the_vectorised_planner_equals_the_line_for_line_one():
    rng = np.random.default_rng(7)
    counts = np.concatenate([np.arange(1, 3000), rng.integers(1, 1 << 21, 3000)])
    for off, per_thread in ((8192, 116), (32768, 4778), (2096, 16), (0, 2568)):
        t, r, ws = ls._plan_many(counts, SM, off, per_thread)
        for k in range(0, counts.size, 7):
            assert ls.plan(int(counts[k]), SM, off, per_thread) == (int(t[k]), int(r[k]), int(ws[k])), (off, per_thread, int(counts[k]))


def _table(src, name):
    """the values of a generated integer table `... NAME[n] = {...};`"""
    for ln in src.splitlines():
        if f" {name}[" in ln and "= {" in ln:
            return [int(v) for v in ln.split("= {")[1].split("}")[0].split(",")]
    raise KeyError(name)


def _regions(src, dfn):
    """every other thing the kernel keeps in dynamic shared memory: [(what, begin, end)]"""
    out = []
    for k in range(int(dfn["JN_RES"])):
        o, b = _table(src, "JRES_OFF")[k], _table(src, "JRES_BYTES")[k]
        out.append((f"resident column {k}", o, o + b))
    if dfn.get("JSTREAM") == "1":
        o = int(dfn["JRING_OFF"].rstrip("u"))
        out.append(("ring", o, o + int(dfn["JRING_STAGES"]) * int(dfn["JRING_TILE"]) * 8))
    for k in range(int(dfn.get("JN_BERN", "0"))):
        o, n = _table(src, "JBERN_MASK")[k], _table(src, "JBERN_N")[k]
        out.append((f"Bernoulli mask {k}", o, o + 4 * ((n + 31) // 32 + 1)))
    return out


def _working_set(dfn, lane):
    """the byte ranges of one lane's working set in shared memory, as the skeletons address it: [(what, begin, end)]"""
    T, D, off = int(dfn["JTHREADS"]), int(dfn["JD"]), int(dfn["JWS_OFF"])
    if dfn.get("JFULL") == "1":                                  # ST(c) = sp[c * JTHREADS], sp = smem + JWS_OFF + lane
        return [(f"state {c}", off + 8 * (c * T + lane), off + 8 * (c * T + lane) + 8) for c in range(D)]
    rows = 2 * int(dfn["JNT"]) + 3 * D                           # tval, tcand, bprop, bcoin, state: one double per row
    out = [(f"row {k}", off + 8 * (k * T + lane), off + 8 * (k * T + lane) + 8) for k in range(rows)]
    vq = off + rows * T * 8                                      # then vq: one u16 per component, JTHREADS apart
    out += [(f"vq {k}", vq + 2 * (k * T + lane), vq + 2 * (k * T + lane) + 2) for k in range(D)]
    return out


@pytest.mark.parametrize("name", MODELS)
def test_every_reachable_shape_keeps_its_shared_memory_regions_apart(compiled, name):
    """At every shape: the working-set columns and vq slots of lanes 0 and JTHREADS - 1 lie inside the declared dynamic shared
    memory and overlap none of the resident columns, the ring stages or the Bernoulli masks, which lie inside it too."""
    pi, built = compiled[name]
    seen = set()
    for C, (msg, src) in built.items():
        dfn = ls.defines(src)
        smem = ls.smem_declared(msg)
        shape = ls.shape_of(dfn)
        seen.add(shape)
        regions = _regions(src, dfn)
        for what, b, e in regions:
            assert 0 <= b < e <= smem, (name, C, shape, what, b, e, smem)
        for i, (w1, b1, e1) in enumerate(regions):
            for w2, b2, e2 in regions[i + 1:]:
                assert e1 <= b2 or e2 <= b1, (name, C, shape, w1, w2)
        if dfn["JWS_SMEM"] != "1":
            continue
        assert int(dfn["JWS_OFF"]) % 16 == 0, (name, C, dfn["JWS_OFF"])
        T = int(dfn["JTHREADS"])
        for lane in (0, T - 1):
            ws = _working_set(dfn, lane)
            lo, hi = min(b for _, b, _ in ws), max(e for _, _, e in ws)
            assert hi <= smem, (name, C, shape, lane, "working set ends past the declared shared memory", hi, smem)
            for what, b, e in regions:
                assert hi <= b or e <= lo, (name, C, shape, lane, "working set overlaps", what)
    assert seen >= set(ls.shapes(pi, SM, LO, HI)), (name, sorted(set(ls.shapes(pi, SM, LO, HI)) - seen))
