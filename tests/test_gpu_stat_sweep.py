"""The statistics sweeps on the GPU, held to exact references.

The specialised statistics sweep (csrc/amwg_jit_kernel.cuh, BASELINE configs 2 and 4) draws every proposal and accept uniform of a
sweep first, forms every plate statistic S = sum_i (x_i - mean)^2 at the proposals in one data pass, then decides each step from
differences of cached terms. With the oracle's Philox streams it must therefore make every decision the oracle makes, unless
exp(delta) lies within rounding of the accept uniform. Per case:

  draws    every chain, every recorded row and the final state against the oracle (orc_run_chains_mt), bit for bit; a chain that
           differs must pass tests/stat_check.audit_divergence (its first differing decision is a rounding tie);
  cache    after every burn / sample call, every slot of every chain's term cache (amwg_get_term_cache) against tests/plate_ref.py at
           the chain's own state: priors, plate terms, and each plate's S with the kernel's ring tile -- on the specialised sweep
           and on the interpreter's statistics sweep (amwg_stat_sweep_kernel, AMWG_JIT=0).

Each case asserts the kernel path it is meant to cover from the generated source (JSTREAM, JWS_SMEM, JBLOCK, JTHREADS)."""
import os
import time

import numpy as np
import pytest

import models
import plate_ref as pr
import prog_eval
import stat_check as sc
from conftest import config2_data

pytestmark = pytest.mark.gpu

RAGGED = (9, 2500, 37, 1111, 3001, 14, 777, 1500, 614)      # test_gpu_jit.py's unequal groups: 9563 points


def _defines(src):
    out = {}
    for ln in src.splitlines():
        if ln.startswith("#define ") and len(ln.split()) == 3:
            _, k, v = ln.split()
            out[k] = v
    return out


def _hier(J, per, seed=5):
    sizes = np.broadcast_to(per, (J,))
    g = np.repeat(np.arange(J), sizes)
    mu = np.random.default_rng(seed).normal(100, 20, J)
    y = mu[g] + np.random.default_rng(seed + 1).normal(0, 5, g.size)
    P = {"mu": {"type": "real", "dim": [J], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    return P, y, g


def _norm_error(x):
    def err(st):
        return pr.oracle_norm_error(x, st[0], st[1], [pr.norm_term([st[0]], 0.0, 100.0), pr.unif_term([st[1]], 0, 100)])
    return err


def _hier_error(y, g, J):
    def err(st):
        priors = [pr.norm_term([st[j]], 0.0, 100.0) for j in range(J)] + [pr.unif_term([st[J]], 0, 100)]
        return pr.oracle_norm_error(y, st[:J][g], st[J], priors)
    return err


def _case(name, ld):
    """-> dict: params, log_post, GPU data, oracle model + data, chains, first_chain, seed, burn, sample, thin, monitor, options,
    the path it must take, the oracle's error bound per log_post evaluation"""
    x = config2_data()
    if name == "A":             # config 2: resident column, working set in shared memory, gchain above 2^32, a ragged last CTA
        return dict(params=models.PARAMS_NORM, f=models.norm_post_readme(ld), data=x.tolist(), model="norm_readme", odata=x,
                    chains=1024 + 37, first=2 ** 32 + 5, seed=3, burn=70, sample=40, thin=1, monitor=None, opts={},
                    path={"JSTREAM": "0", "JWS_SMEM": "1", "JBLOCK": "-1"}, ragged=True, err=_norm_error(x))
    if name == "B_derived":     # a derived quantity, a monitored subset, thin 3
        xs = x[:300]
        return dict(params=models.PARAMS1, f=models.norm_post_test(ld), data=xs.tolist(), model="norm_test", odata=xs,
                    chains=517, first=77, seed=4, burn=60, sample=60, thin=3, monitor=["var", "mu"], opts={},
                    path={"JSTREAM": "0", "JBLOCK": "-1"}, ragged=True, err=_norm_error(xs))
    if name == "B_bounds":      # an int parameter (rounded proposals) and bounds that reject proposals without drawing a uniform
        P = {"mu": {"type": "int", "lower": 150, "upper": 200}, "sigma": {"type": "real", "lower": 0, "upper": 50}}
        return dict(params=P, f=models.norm_post_readme(ld), data=x.tolist(), model="norm_readme", odata=x,
                    chains=517, first=1000, seed=5, burn=60, sample=50, thin=1, monitor=None, opts={},
                    path={"JSTREAM": "0", "JBLOCK": "-1"}, ragged=True, err=_norm_error(x))
    if name == "C":             # hierarchical, 8 x 32 resident: the index-ordered block of group means, working set in global memory
        P, y, g = _hier(8, 32)
        return dict(params=P, f=models.hier_norm_post(ld), data={"y": y.tolist(), "g": g.astype(float).tolist()}, model="hier_norm",
                    odata={"y": y, "g": g}, chains=1024 + 37, first=9, seed=21, burn=70, sample=40, thin=1, monitor=None, opts={},
                    path={"JSTREAM": "0", "JWS_SMEM": "0", "JBLOCK": "0"}, ragged=True, err=_hier_error(y, g, 8))
    if name == "D":             # 12 x 1024 (96 KB): the ring, every plate ending on a tile end
        P, y, g = _hier(12, 1024)
        return dict(params=P, f=models.hier_norm_post(ld), data={"y": y.tolist(), "g": g.astype(float).tolist()}, model="hier_norm",
                    odata={"y": y, "g": g}, chains=200, first=3, seed=22, burn=15, sample=10, thin=1, monitor=None,
                    opts={"batch_size": 10}, path={"JSTREAM": "1", "JBLOCK": "0"}, ragged=True, err=_hier_error(y, g, 12))
    if name == "E":             # RAGGED: plates ending mid-tile, a group over more than two tiles, an odd total, 10 tiles per pass
        P, y, g = _hier(len(RAGGED), RAGGED)
        return dict(params=P, f=models.hier_norm_post(ld), data={"y": y.tolist(), "g": g.astype(float).tolist()}, model="hier_norm",
                    odata={"y": y, "g": g}, chains=200, first=2 ** 33 + 1, seed=23, burn=15, sample=10, thin=1, monitor=None,
                    opts={"batch_size": 10}, path={"JSTREAM": "1", "JBLOCK": "0"}, ragged=True, err=_hier_error(y, g, len(RAGGED)))
    raise KeyError(name)


CASES = ["A", "B_derived", "B_bounds", "C", "D", "E"]


def _components(s, d, names):
    """[rows, chains, D]: the recorded parameters of a sample() result, in the flat component order"""
    C = s.n_chains
    return np.concatenate([np.asarray(d[n], np.float64).reshape(len(d[n]), C, -1) for n in names], axis=2)


def _state_matrix(s):
    st = s.state
    return np.concatenate([np.asarray(st[n], np.float64).reshape(s.n_chains, -1) for n in s.params], axis=1)


def _make(pkg, monkeypatch, cs, jit):
    monkeypatch.setenv("AMWG_JIT", "1" if jit else "0")
    o = {"chains": cs["chains"], "seed": cs["seed"], "first_chain": cs["first"]}
    o.update(cs["opts"])
    s = pkg.mcmc.AmwgSampler(cs["params"], cs["f"], cs["data"], o)
    monkeypatch.delenv("AMWG_JIT")
    assert s.jit_status()[0] == jit, s.jit_status()
    assert s._program.stat_prog >= 0
    return s


def _check_cache(s, consts, tile, what, skip=()):
    cache = s._term_cache()                         # before anything else touches the cache
    return sc.check_term_cache(s._program, consts, cache, _state_matrix(s), tile, what, skip)


def _run(s, cs, consts, tile, what, skip=()):
    """burn, then (thin, monitor) sample, checking the term cache after each; -> (draws, worst err/bound per slot kind)"""
    worst = {"stat": 0.0, "term": 0.0}

    def take(w):
        for k in ("stat", "term"):
            worst[k] = max(worst[k], w[k])
    s.burn(cs["burn"])
    take(_check_cache(s, consts, tile, f"{what} burn", skip))
    if cs["thin"] != 1:
        s.thin(cs["thin"])
    if cs["monitor"] is not None:
        s.monitor(cs["monitor"])
    d = s.sample(cs["sample"])
    take(_check_cache(s, consts, tile, f"{what} sample", skip))
    return d, worst


def _report(line):
    print(line)
    out = os.environ.get("STAT_SWEEP_REPORT")
    if out:
        with open(out, "a") as fh:
            fh.write(line + "\n")


@pytest.mark.parametrize("name", CASES)
def test_specialised_statistics_sweep_chain_for_chain_against_the_oracle(gpu_pkg, orc, monkeypatch, name):
    """Oracle wall times measured on a 16-core host beside an H100 (orc_run_chains_mt, one thread per core): A 0.8 s, B_derived
    0.2 s, B_bounds 0.4 s, C 1.0 s, D 2.8 s, E 1.9 s; the whole file took 28 s there. No divergent chain was found in any case."""
    pr.require_extended()
    pkg = gpu_pkg
    cs = _case(name, pkg.ld)
    s = _make(pkg, monkeypatch, cs, True)
    C = cs["chains"]
    rc, msg, src = s.jit_compile_check(C)
    assert rc == 0, msg
    dfn = _defines(src)
    for k, v in cs["path"].items():
        assert dfn[k] == v, (name, k, dfn[k], v)
    if cs["ragged"]:
        assert C % int(dfn["JTHREADS"]) != 0, (C, dfn["JTHREADS"])
    tile = int(dfn["JRING_TILE"]) if dfn["JSTREAM"] == "1" else pr.JRING_TILE
    assert tile == pr.JRING_TILE
    consts = prog_eval.fold_constants(s._program, orc.lib())
    d, worst = _run(s, cs, consts, tile, f"{name} specialised")
    final = _state_matrix(s)

    names = list(cs["params"])
    comp_options = {k: dict(cs["opts"]) for k in names} if cs["opts"] else None
    t0 = time.perf_counter()
    ref, ofinal = orc.run_model(cs["model"], cs["odata"], cs["params"], chains=C, seed=cs["seed"], burn=cs["burn"], sample=cs["sample"],
                                thin=cs["thin"], first_chain=cs["first"], comp_options=comp_options, monitor=cs["monitor"],
                                threads=os.cpu_count() or 1, final_state=True)
    t_orc = time.perf_counter() - t0
    mon = cs["monitor"] or (names + list(s._derived_names))
    assert list(d.keys()) == mon
    same = np.ones(C, dtype=bool)
    for k in mon:
        a, b = np.asarray(d[k], np.float64), np.asarray(ref[k], np.float64)
        assert a.shape == b.shape, (k, a.shape, b.shape)
        same &= (a.view(np.uint64) == b.view(np.uint64)).reshape(a.shape[0], C, -1).all(axis=(0, 2))
    D = final.shape[1]
    same &= (final.view(np.uint64) == ofinal[:, :D].view(np.uint64)).all(axis=1)
    div = np.flatnonzero(~same)
    audited = 0
    for c in div:
        assert cs["thin"] == 1 and cs["monitor"] is None, f"chain {c} differs at thin {cs['thin']}: its decisions cannot be localised"
        g = _components(s, d, names)[:, c]
        o = np.concatenate([np.asarray(ref[n], np.float64).reshape(cs["sample"], C, -1)[:, c] for n in names], axis=1)
        g = np.vstack([g, final[c]])
        o = np.vstack([o, ofinal[c, :D]])
        r = int(np.flatnonzero((g.view(np.uint64) != o.view(np.uint64)).any(axis=1))[0])
        assert r > 0, f"chain {c} differs already in its first recorded row: the divergence lies in the burn and cannot be localised"
        orc_s = orc.OracleSampler(cs["model"], cs["odata"], cs["params"], seed=cs["seed"], chain=cs["first"] + int(c), comp_options=comp_options)
        orc_s.trace((cs["burn"] + cs["sample"]) * D)
        orc_s.burn(cs["burn"])
        orc_s.sample(cs["sample"])
        tr = orc_s.trace_rows()
        sweep = cs["burn"] + r - 1
        sc.audit_divergence(s._program, consts, tr[sweep * D:(sweep + 1) * D], g[r - 1], g[r], o[r], tile, cs["err"])
        audited += 1
    _report(f"{name}: {C} chains compared, {div.size} divergent, {audited} audited as ties; worst err/bound specialised: "
            f"stat {worst['stat']:.3g}, term {worst['term']:.3g}; oracle {t_orc:.1f} s on {os.cpu_count()} cores")

    # the interpreter's statistics sweep, the same schedule: its term cache (its ring's tiles hold 2048 points)
    si = _make(pkg, monkeypatch, cs, False)
    _, wi = _run(si, cs, consts, pr.RING_TILE, f"{name} interpreter")
    _report(f"{name}: worst err/bound interpreter statistics sweep: stat {wi['stat']:.3g}, term {wi['term']:.3g}")


# ---- a plate whose mean is an expression (jit_stat_extra): no oracle model, the term cache only ------------------------------
EXPR_PARAMS = {"a": {"type": "real"}, "k": {"type": "int", "lower": -20, "upper": 20}, "s": {"type": "real", "lower": 0, "upper": 50}}


def expr_data():
    return np.random.default_rng(9).normal(7.0, 2.0, 300)


def expr_post(ld):
    """test_gpu_jit.py's expression-mean model: mean 2a + 1 over 300 points, mean k over the first 100, an ld.gamma prior"""
    def lp(state, d):
        out = 0
        out += ld.norm(state.a, 0, 10)
        out += ld.unif(state.k, -20, 20)
        out += ld.gamma(state.s, 2, 0.5)
        for i in range(len(d)):
            out += ld.norm(d[i], state.a * 2 + 1, state.s)
        for i in range(100):
            out += ld.norm(d[i], state.k, 3.0)
        state.prec = 1 / (state.s * state.s)
        return out
    return lp


@pytest.mark.parametrize("jit", [True, False])
def test_expression_mean_statistics_in_the_term_cache(gpu_pkg, orc, monkeypatch, jit):
    """S at the mean 2a + 1 formed in fp64 from the chain's a, as the kernels form it (the program's MUL and ADD); the ld.gamma prior's
    slot has no reference here and is skipped by name."""
    pr.require_extended()
    cs = dict(params=EXPR_PARAMS, f=expr_post(gpu_pkg.ld), data=expr_data().tolist(), chains=4096 + 37, first=2 ** 32 + 1, seed=2,
              burn=70, sample=40, thin=1, monitor=None, opts={})
    s = _make(gpu_pkg, monkeypatch, cs, jit)
    if jit:
        rc, msg, src = s.jit_compile_check(cs["chains"])
        assert rc == 0, msg
        assert "sum_sq_dev(" in src.split("void jit_stat_extra")[1].split("\n}\n")[0]      # the 2a + 1 plate's S is formed there
        assert cs["chains"] % int(_defines(src)["JTHREADS"]) != 0
    consts = prog_eval.fold_constants(s._program, orc.lib())
    _, w = _run(s, cs, consts, pr.JRING_TILE, f"expression means jit={jit}", skip=("LD_GAMMA",))
    _report(f"expression means ({'specialised' if jit else 'interpreter'}): worst err/bound stat {w['stat']:.3g}, term {w['term']:.3g}")
