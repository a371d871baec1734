"""Self-checks of the statistics-sweep references (tests/plate_ref.py sum_sq, tests/stat_check.py) and of the oracle's step trace, on
the CPU: the GPU tests of tests/test_gpu_stat_sweep.py are only as strong as these."""
import math
from fractions import Fraction

import numpy as np
import pytest

import models
import plate_ref as pr
import prog_eval
import stat_check as sc
from conftest import config2_data


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))           # one rounding, as the device's DFMA


def _sum_sq_dev(x, mean, peel):
    """csrc amwg_tma.cuh sum_sq_dev, operation by operation in fp64 (fma exact via Fraction)"""
    s = [0.0, 0.0, 0.0, 0.0]
    i = 0
    if peel and len(x) > 0:
        d = float(x[0]) - mean
        s[3] = _fma(d, d, s[3])
        i = 1
    nb = (len(x) - i) >> 3
    for b in range(nb):
        d = [float(v) - mean for v in x[i + 8 * b:i + 8 * b + 8]]
        for k in range(8):
            s[k % 4] = _fma(d[k], d[k], s[k % 4])
    for v in x[i + 8 * nb:]:
        d = float(v) - mean
        s[0] = _fma(d, d, s[0])
    return (s[0] + s[1]) + (s[2] + s[3])


def _ring(x, mean, tile, offset):
    """the specialised sweep's ring: one sum_sq_dev per part of the plate inside a tile (tiles of `tile` points from `offset` points
    before the plate), peeling when the part starts at an odd point of its tile, partial sums added in order"""
    S, p0 = 0.0, 0
    while p0 < len(x):
        e = min(len(x), (offset + p0) // tile * tile + tile - offset)
        S = S + _sum_sq_dev(x[p0:e], mean, (offset + p0) % 2 == 1)
        p0 = e
    return S


@pytest.mark.parametrize("n,loc,scale", [(1, 184.5, 4.5), (7, 184.5, 4.5), (9, 184.5, 4.5), (1021, 184.5, 4.5), (1021, 1e6, 1.0),
                                         (2500, 100.0, 5.0)])
def test_sum_sq_against_exact_sums_and_the_kernels_arithmetic(n, loc, scale):
    """sum_sq's value against the exact rational sum, and the fp64 sums of the kernels' own structures (one partial, or tiles of
    1024 / 2048 points with the plate starting mid-tile) within its bound; a dropped or duplicated point is far outside it."""
    pr.require_extended()
    rng = np.random.default_rng(n)
    x = rng.normal(loc, scale, n)
    means = np.array([loc, loc + scale * 0.37, loc - scale * 1.9])
    for tile, offset in ((pr.JRING_TILE, 0), (pr.JRING_TILE, 613), (pr.JRING_TILE, 1023), (pr.RING_TILE, 0), (pr.RING_TILE, 1)):
        ref = pr.sum_sq(x, means, tile=tile)
        for k, m in enumerate(means):
            exact = sum((Fraction(float(v)) - Fraction(float(m))) ** 2 for v in x)
            assert abs(Fraction(*ref.value[k].as_integer_ratio()) - exact) <= Fraction(float(ref.bound[k])) * Fraction(1, 1000)
        got = np.array([_ring(x, m, tile, offset) for m in means])
        ref.check(got, f"n={n} tile={tile} offset={offset}")
        ref.check(np.array([_sum_sq_dev(x, m, offset % 2 == 1) for m in means]), "one partial")
        if n > 1:
            with pytest.raises(AssertionError):
                ref.check(np.array([_ring(x[:-1], m, tile, offset) for m in means]), "dropped")
        with pytest.raises(AssertionError):
            ref.check(np.array([_ring(np.append(x, x[n // 2]), m, tile, offset) for m in means]), "duplicated")


def _norm_model(pkg, orc, params):
    s = pkg.mcmc.AmwgSampler(params, models.norm_post_readme(pkg.ld), config2_data().tolist(), {"chains": 64, "_model_only": True})
    prog = s._program
    assert prog.stat_prog >= 0
    return prog, prog_eval.fold_constants(prog, orc.lib())


def _norm_oracle_error(x):
    def err(st):
        priors = [pr.norm_term([st[0]], 0.0, 100.0), pr.unif_term([st[1]], 0, 100)]
        return pr.oracle_norm_error(x, st[0], st[1], priors)
    return err


def _traced(orc, params, chain, sweeps, comp_options=None):
    o = orc.OracleSampler("norm_readme", config2_data(), params, seed=7, chain=chain, comp_options=comp_options)
    o.trace(2 * sweeps + 5)
    rows = o.sample(sweeps)
    return o, o.trace_rows(), np.column_stack([rows["mu"], rows["sigma"]])


def test_the_oracle_trace_replays_the_oracle(orc):
    """Replaying the traced decisions from the initial state gives the oracle's recorded draws, every traced proposal and uniform is
    the Philox stream's at its position (rnorm's trials re-drawn, one uniform per in-bounds proposal, one per sweep for the shuffle
    of the two substeppers), and the uniforms consumed are rng_position()."""
    params = {"mu": {"type": "int", "lower": 150, "upper": 200}, "sigma": {"type": "real", "lower": 0, "upper": 50}}
    opts = {k: {"is_adapting": False, "prop_log_scale": 1.5} for k in params}       # fixed proposal scales: rnorm can be re-drawn
    sweeps, chain = 300, 2 ** 32 + 5
    o, tr, rows = _traced(orc, params, chain, sweeps, opts)
    assert tr.shape == (2 * sweeps, 6)
    L = orc.lib()
    sd = L.orc_exp(1.5)
    state = rows[0].copy()
    n = 0
    import ctypes
    oob = 0
    for s in range(sweeps):
        assert np.array_equal(state, rows[s]), s
        n += 1                                                      # shuffle_array(substeppers): one uniform for two of them
        for c, cur, prop, u, lc, lp in tr[2 * s:2 * s + 2]:
            c = int(c)
            assert cur == state[c]
            pos = ctypes.c_uint64(n)
            p = L.orc_rnorm(7, chain, ctypes.byref(pos), cur, sd)
            n = pos.value
            assert prop == (L.orc_js_round(p) if c == 0 else p)
            if u < 0:
                assert prop < params[["mu", "sigma"][c]]["lower"] or prop > params[["mu", "sigma"][c]]["upper"]
                assert math.isnan(lc) and math.isnan(lp)
                oob += 1
                continue
            assert u == L.orc_stream_uniform(7, chain, n)
            n += 1
            if L.orc_exp(lp - lc) > u:
                state[c] = prop
    assert np.array_equal(state, o.state()[:2]) and n == o.rng_position()
    assert oob > 10                                                 # the int bounds and sigma's upper bound were hit


def test_the_audit_accepts_the_oracles_decisions_and_rejects_a_flip(pkg, orc):
    """Every traced decision of the oracle is what exp(delta*) > u says wherever |log u - delta*| exceeds the audit's bound; a
    decision flipped where that gap is large is reported as a wrong decision, not a tie."""
    pr.require_extended()
    params = models.PARAMS_NORM
    prog, consts = _norm_model(pkg, orc, params)
    err = _norm_oracle_error(config2_data())
    sweeps = 40
    o, tr, rows = _traced(orc, params, 11, sweeps)
    smallest = sc.oracle_decisions_agree(prog, consts, tr, rows[0], pr.JRING_TILE, err)
    assert smallest > 1.0                                          # no step of this run is anywhere near a tie
    after = np.vstack([rows[1:], o.state()[None, :2]])
    flipped = 0
    for s in range(5, sweeps):
        steps = tr[2 * s:2 * s + 2]
        c, cur, prop = int(steps[0][0]), steps[0][1], steps[0][2]
        if steps[0][3] < 0 or prop == cur:
            continue
        gpu = after[s].copy()
        gpu[c] = cur if after[s][c] == prop else prop              # the first step of the sweep decided the other way
        with pytest.raises(AssertionError, match="not a rounding tie"):
            sc.audit_divergence(prog, consts, steps, rows[s], gpu, after[s], pr.JRING_TILE, err)
        flipped += 1
    assert flipped >= 10
    with pytest.raises(AssertionError, match="every decision agrees"):
        sc.audit_divergence(prog, consts, tr[10:12], rows[5], after[5], after[5], pr.JRING_TILE, err)


def _hier_ragged():
    from test_jit_codegen_semantics import RAGGED
    sizes = np.asarray(RAGGED)
    rng = np.random.default_rng(4)
    g = np.repeat(np.arange(sizes.size), sizes)
    y = rng.normal(100, 5, g.size) + np.repeat(rng.normal(0, 3, sizes.size), sizes)
    P = {"mu": {"type": "real", "dim": [sizes.size], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    return P, {"y": y, "g": g.astype(float)}


def test_the_term_cache_check_has_teeth_on_the_emulated_statistics_sweep(pkg, orc, tmp_path):
    """The specialised statistics sweep compiled for the host (one thread per CTA, memcpy for TMA) on the ragged groups of
    test_gpu_stat_sweep.py's case E (9563 points streamed in tiles of 1024, plates ending mid-tile): its term cache passes
    check_term_cache; the same kernel text with one point dropped wherever a plate ends inside a tile fails it."""
    from test_jit_codegen_semantics import HostStatKernel
    pr.require_extended()
    P, data = _hier_ragged()
    good = tmp_path / "good"
    good.mkdir()
    hk = HostStatKernel(pkg, orc, good, P, models.hier_norm_post(pkg.ld), data)
    assert "#define JSTREAM 1" in hk.src and f"#define JRING_TILE {pr.JRING_TILE}\n" in hk.src
    hk.run(8, 77, 9, 20)
    worst = sc.check_term_cache(hk.prog, hk.consts, hk.work[:hk.NT], hk.state.T, pr.JRING_TILE, "host")
    assert worst["stat"] < 1.0 and worst["term"] < 1.0

    needle = "e - p0, mean);"

    def drop(text):
        assert text.count(needle) == 1
        return text.replace(needle, "e - p0 - ((e == pend && e < hi) ? 1 : 0), mean);")
    bad = tmp_path / "bad"
    bad.mkdir()
    hb = HostStatKernel(pkg, orc, bad, P, models.hier_norm_post(pkg.ld), data, edit=drop)
    hb.run(8, 77, 9, 20)
    with pytest.raises(AssertionError, match="of plate"):
        sc.check_term_cache(hb.prog, hb.consts, hb.work[:hb.NT], hb.state.T, pr.JRING_TILE, "host, a point dropped")


def test_the_slot_map_covers_every_slot_of_the_models_under_test(pkg, orc):
    """norm_readme, norm_test (a derived quantity), the int / bounded variant, the hierarchical model and the expression-mean model:
    every slot maps to a prior, a plate term or a statistic, the statistics after the terms of the sum; ld.gamma is the one op the
    map reports as having no reference."""
    ld, mcmc = pkg.ld, pkg.mcmc
    x = config2_data()
    P, data = _hier_ragged()
    cases = [(models.PARAMS_NORM, models.norm_post_readme(ld), x.tolist(), ["norm", "unif", "plate"]),
             (models.PARAMS1, models.norm_post_test(ld), x.tolist(), ["norm", "unif", "plate"]),
             (P, models.hier_norm_post(ld), data, ["norm"] * 9 + ["unif"] + ["plate"] * 9)]
    import test_gpu_stat_sweep as g
    cases.append((g.EXPR_PARAMS, g.expr_post(ld), g.expr_data().tolist(), ["norm", "unif", "other", "plate", "plate"]))
    for params, f, d, kinds in cases:
        s = mcmc.AmwgSampler(params, f, d, {"chains": 64, "_model_only": True})
        prog = s._program
        sl = sc.slots(prog, prog_eval.fold_constants(prog, orc.lib()))
        assert [t.kind for t in sl[:prog.n_sum_terms]] == kinds
        assert [t.kind for t in sl[prog.n_sum_terms:]] == ["stat"] * kinds.count("plate")
