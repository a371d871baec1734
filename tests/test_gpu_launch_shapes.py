"""The specialised sweeps at every launch shape the planner chooses, on the GPU.

choose_shape (csrc/amwg_jit.cuh) picks each handle's CTA size, CTAs per SM and where the working set lives from its chain count and
the device's SM count; each shape is a kernel of its own (__launch_bounds__, the JWS_SMEM / JWS_OFF layout). A chain's draws must
not depend on it: its stream is keyed by its global id, sum_sq_dev sums each lane's points in a fixed order, and nothing else a
chain computes reads its lane or its CTA. Per model, every shape reachable with LO to the model's `hi` chains (tests/launch_shape.py, at this
device's SM count) runs at its smallest ragged chain count (C % threads != 0: a last CTA with shadow threads), each handle starting
at its own offset into one range of global chains above 2^32, so the same chain sits on different lanes, warps and CTAs:

  invariance   every chain a shape handle shares with the reference handle (a 128-thread handle over the whole range) ends with the
               same checkpoint arrays (state, pls, perm / perm_ext, rng_n, acc), term cache, log_post() and recorded rows, bit for bit;
  interpreter  a full-program model's reference handle equals an AMWG_JIT=0 handle over the same chains, bit for bit;
  oracle       lanes 0, 31, 32, T - 1 and T, the last chain of the last full CTA and the first and last chain of the ragged CTA
               against the oracle: bit for bit, or (statistics sweep) a rounding tie that stat_check.audit_divergence accepts;
  restore      images of the reference handle, taken mid-run, restored into handles of the two shapes most unlike it, continue as
               the run that never stopped (once per skeleton).

To keep to about 40 compilations, each CTA size runs at its smallest and largest CTAs-per-SM count only; the report names the shapes
left out. On one H100 80GB HBM3 (132 SMs) the file ran 37 shape handles (51 handles in all) in 255 s, NVRTC builds included: a 13 s, b 34 s, c 11 s and
d 184 s, most of it d's oracle evaluating log_post through its Python callback. No chain differed from the reference or from the
interpreter, and no oracle chain needed the tie audit."""
import os
import time

import numpy as np
import pytest

import ckpt_ref
import launch_shape as ls
import models
import plate_ref as pr
import prog_eval
import stat_check as sc
from conftest import config2_data, config3_data

pytestmark = pytest.mark.gpu

BASE = 2 ** 32 + 11                                      # the first global chain of every model's range
RAGGED = (9, 2500, 37, 1111, 3001, 14, 777, 1500, 614)   # test_gpu_stat_sweep.py case E: 9563 points, streamed
LO = 40                                                  # the smallest chain count run: lanes 0, 31 and 32 exist
WIDE_T, WIDE_J = 17, 260                                 # model d: 19 named parameters, dim[0] = 260


def _hier(J, per, seed=5):
    sizes = np.broadcast_to(per, (J,))
    g = np.repeat(np.arange(J), sizes)
    mu = np.random.default_rng(seed).normal(100, 20, J)
    y = mu[g] + np.random.default_rng(seed + 1).normal(0, 5, g.size)
    P = {"mu": {"type": "real", "dim": [J], "init": 100.0}, "sigma": {"type": "real", "lower": 0, "init": 5.0}}
    return P, y, g


def _wide_params():
    P = {"t%d" % k: ({"type": "real"} if k % 3 else {"type": "int", "lower": -50, "upper": 50}) for k in range(WIDE_T)}
    P["x"] = {"type": "real", "dim": [WIDE_J]}
    P["s"] = {"type": "real", "lower": 0}
    return P


def _wide_post(ld):
    def lp(state, d=None):
        out = ld.gamma(state.s, 2, 1)
        for j in range(WIDE_J):
            out += ld.norm(state.x[j], 0.01 * j, state.s)
        for k in range(WIDE_T):
            out += ld.norm(state["t%d" % k], 0.5 * k, 1 + 0.1 * k)
        return out
    return lp


def _wide_oracle(O):
    def f(st):
        v = O.orc_ld_gamma(st[WIDE_T + WIDE_J], 2, 1)
        for j in range(WIDE_J):
            v += O.orc_ld_norm(st[WIDE_T + j], 0.01 * j, st[WIDE_T + WIDE_J])
        for k in range(WIDE_T):
            v += O.orc_ld_norm(st[k], 0.5 * k, 1 + 0.1 * k)
        return v
    return f


def _model(name, pkg, O):
    """-> dict: params, log_post, GPU data, oracle model + data, options, environment at create, range of chain counts, sweeps
    (burn before the mid-run image, burn after it, recorded rows), monitored names, oracle lanes, error bound per evaluation"""
    ld, mcmc = pkg.ld, pkg.mcmc
    if name == "a_config2":     # one resident column, the statistics sweep; its working set in shared memory up to 160 threads
        x = config2_data()
        return dict(params=models.PARAMS_NORM, f=models.norm_post_readme(ld), data=x.tolist(), omodel="norm_readme", odata=x,
                    opts={}, env={}, hi=300000, sweeps=(30, 30, 10), monitor=None, full=False,
                    err=lambda st: pr.oracle_norm_error(x, st[0], st[1], [pr.norm_term([st[0]], 0.0, 100.0), pr.unif_term([st[1]], 0, 100)]))
    if name == "b_ragged_ring":  # the streamed ring with plates ending mid-tile, the index-ordered block of group means (JBLOCK >= 0)
        P, y, g = _hier(len(RAGGED), RAGGED)
        J = len(RAGGED)

        def err(st):
            priors = [pr.norm_term([st[j]], 0.0, 100.0) for j in range(J)] + [pr.unif_term([st[J]], 0, 100)]
            return pr.oracle_norm_error(y, st[:J][g], st[J], priors)
        return dict(params=P, f=models.hier_norm_post(ld), data={"y": y.tolist(), "g": g.astype(float).tolist()}, omodel="hier_norm",
                    odata={"y": y, "g": g}, opts={"batch_size": 10}, env={}, hi=300000, sweeps=(15, 15, 8), monitor=None, full=False,
                    err=err)
    if name == "c_spike":       # the full-program sweep, Bernoulli plate as a bit mask built by a ballot
        x = config3_data()
        return dict(params=models.PARAMS_SPIKE, f=models.spike_bern(ld, mcmc), data={"x": x.tolist()}, omodel="spike_bern",
                    odata={"x": x}, opts={}, env={}, hi=300000, sweeps=(30, 30, 10), monitor=None, full=True)
    if name == "d_wide":        # the full-program sweep (term cache dropped) with perm_ext and order_ext in global rows
        # 278 components: its checkpoints take 5.6 KB per chain and the oracle evaluates log_post through a Python callback, so
        # this model runs the shapes of up to 40000 chains, four oracle chains per handle and fewer sweeps
        return dict(params=_wide_params(), f=_wide_post(ld), data=None, omodel=_wide_oracle(O), odata=None, opts={},
                    env={"AMWG_TERM_CACHE": "0"}, hi=40000, sweeps=(3, 3, 3), monitor=["t0", "t16", "s"], full=True, lanes="short")
    raise KeyError(name)


MODELS = ["a_config2", "b_ragged_ring", "c_spike", "d_wide"]


def _report(line):
    print(line)
    out = os.environ.get("LAUNCH_SHAPE_REPORT")
    if out:
        with open(out, "a") as fh:
            fh.write(line + "\n")


def _make(pkg, monkeypatch, m, first, chains, jit=True):
    for k, v in list(m["env"].items()) + [("AMWG_JIT", "1" if jit else "0")]:
        monkeypatch.setenv(k, v)
    o = {"chains": chains, "seed": 17, "first_chain": first}
    o.update(m["opts"])
    s = pkg.mcmc.AmwgSampler(m["params"], m["f"], m["data"], o)
    for k in list(m["env"]) + ["AMWG_JIT"]:
        monkeypatch.delenv(k)
    if m["monitor"] is not None:
        s.monitor(m["monitor"])
    on, note = s.jit_status()
    assert on == jit, note
    return s


def _assert_shape(s, shape, m):
    T, R, ws = shape
    note = s.jit_status()[1]
    assert f"{T} threads x {R} CTAs/SM" in note, (shape, note)
    assert ("working set in shared memory" in note) == bool(ws), (shape, note)
    assert ("full-program" in note) == m["full"], note


def _finish(s):
    """what a handle ends with: checkpoint arrays, term cache, log_post, per chain (chains on the last axis)"""
    ck = ckpt_ref.parse(s.checkpoint())
    out = {k: np.asarray(ck[k]) for k in ("state", "pls", "perm", "perm_ext", "rng_n", "acc") if k in ck}
    out["term_cache"] = s._term_cache()
    out["log_post"] = np.atleast_1d(np.asarray(s.log_post(), np.float64))
    return out


def _run(s, m, restore_from=None):
    """burn (with adaptation), a mid-run image, burn, sample -> (rows {name: [rows, C, ...]}, finish, mid-run image)"""
    b1, b2, n = m["sweeps"]
    img = None
    if restore_from is None:
        s.burn(b1)
        img = s.checkpoint()
    else:
        s.restore(restore_from)
    s.burn(b2)
    d = s.sample(n)
    return d, _finish(s), img


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _compare(got, ref, off, what):
    """every per-chain array of `got` against chains [off, off + C) of `ref` -> chains compared"""
    d, fin = got
    rd, rfin = ref
    C = fin["rng_n"].shape[-1]
    for k, v in fin.items():
        assert _same_bits(v, rfin[k][..., off:off + C]), (what, k)
    for k, v in d.items():
        assert _same_bits(np.asarray(v), np.asarray(rd[k])[:, off:off + C]), (what, "row", k)
    return C


def _select(all_shapes):
    """each CTA size at its smallest and largest CTAs-per-SM count -> (kept {shape: count}, left out [shape])"""
    keep = {}
    for t in sorted({k[0] for k in all_shapes}):
        rs = sorted(k for k in all_shapes if k[0] == t)
        for k in (rs[0], rs[-1]):
            keep[k] = all_shapes[k]
    return keep, sorted(set(all_shapes) - set(keep))


def _lanes(T, C, short=False):
    full_end = C // T * T
    want = (0, T - 1, T, C - 1) if short else (0, 31, 32, T - 1, T, full_end - 1, full_end, C - 1)
    return sorted({k for k in want if 0 <= k < C})


def _oracle_sampler(orc, m, gchain):
    comp = {k: dict(m["opts"]) for k in m["params"]} if m["opts"] else None
    return orc.OracleSampler(m["omodel"], m["odata"], m["params"], seed=17, chain=gchain, comp_options=comp)


def _oracle(orc, m, gchain):
    """one chain of the oracle over the same sweeps -> (rows {name: [rows, ...]}, final state [D])"""
    b1, b2, n = m["sweeps"]
    o = _oracle_sampler(orc, m, gchain)
    o.burn(b1 + b2)
    d = o.sample(n, monitor=m["monitor"])
    return d, o.state()[:o.D]


def _oracle_window(orc, s, m, d, fin, lanes, first, consts):
    """the chains at `lanes` of handle s against the oracle -> (compared, audited)"""
    b1, b2, n = m["sweeps"]
    names = list(m["monitor"] or list(m["params"]) + list(s._derived_names))
    got_rows, orc_rows, orc_final, same = [], [], [], []
    for k in lanes:
        od, ofin = _oracle(orc, m, first + k)
        eq = True
        for nm in names:
            a = np.asarray(d[nm], np.float64)[:, k]
            b = np.asarray(od[nm], np.float64).reshape(a.shape)
            eq &= _same_bits(a, b)
        same.append(eq)
        orc_final.append(ofin)
        if not m["full"]:
            got_rows.append(np.concatenate([np.asarray(d[nm], np.float64)[:, k].reshape(n, -1) for nm in m["params"]], axis=1))
            orc_rows.append(np.concatenate([np.asarray(od[nm], np.float64).reshape(n, -1) for nm in m["params"]], axis=1))
    gfin = np.ascontiguousarray(fin["state"][:, lanes].T)
    ofin = np.asarray(orc_final)
    if m["full"]:                                   # the full-program sweep is bit-faithful: no ties
        assert all(same), ("rows differ from the oracle", [k for k, e in zip(lanes, same) if not e])
        assert _same_bits(gfin, ofin), ("final states differ from the oracle", lanes)
        return len(lanes), 0

    def trace(j):
        o = _oracle_sampler(orc, m, first + lanes[j])
        o.trace((b1 + b2 + n) * gfin.shape[1])
        o.burn(b1 + b2)
        o.sample(n)
        return o.trace_rows()
    _, audited = sc.compare_and_audit(s._program, consts, np.asarray(same), np.stack(got_rows, axis=1), gfin,
                                      np.stack(orc_rows, axis=1), ofin, trace, b1 + b2, pr.JRING_TILE, m["err"])
    return len(lanes), audited


@pytest.mark.parametrize("name", MODELS)
def test_every_launch_shape_draws_what_the_others_draw(gpu_pkg, orc, monkeypatch, name):
    import torch
    pr.require_extended()
    t_start = time.perf_counter()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    m = _model(name, gpu_pkg, orc.lib())
    probe = _make(gpu_pkg, monkeypatch, m, BASE, 4096 + 1)
    if m["env"].get("AMWG_TERM_CACHE") == "0":
        probe._model_keepalive[-1].n_terms = 0          # what amwg_create did to the handle's model: the compile check plans that
    pi = ls.inputs(probe)
    assert pi.full == m["full"]
    dfn = ls.defines(probe.jit_compile_check(4096)[2])
    if name == "b_ragged_ring":
        assert dfn["JSTREAM"] == "1" and int(dfn["JBLOCK"]) >= 0, dfn
    if name == "d_wide":
        assert int(dfn["JP"]) > 16 and int(dfn["JMAX_DIM0"]) > 256, dfn
    consts = None if m["full"] else prog_eval.fold_constants(probe._program, orc.lib())
    del probe
    reach = ls.shapes(pi, sm, LO, m["hi"])
    keep, left_out = _select(reach)
    plan = [(shape, C, 13 * i + (i % 2) * 32) for i, (shape, C) in enumerate(sorted(keep.items()))]
    span = max(off + C for _, C, off in plan)
    n_ref = ls.count_with(pi, sm, 128, span)
    ref_s = _make(gpu_pkg, monkeypatch, m, BASE, n_ref)
    assert ls.plan(n_ref, sm, pi.off, pi.per_thread)[0] == 128 and "128 threads x" in ref_s.jit_status()[1]
    rd, rfin, img = _run(ref_s, m)
    ref_shape = ls.plan(n_ref, sm, pi.off, pi.per_thread)
    del ref_s
    _report(f"{name}: {sm} SMs, plan inputs {pi}; reachable shapes up to {m['hi']} chains: {len(reach)}; "
            f"left out (not the smallest or largest CTAs/SM of their size): {left_out}")
    _report(f"{name}: reference {ref_shape} at {n_ref} chains from {BASE}")
    if m["full"]:
        si = _make(gpu_pkg, monkeypatch, m, BASE, n_ref, jit=False)
        got = _run(si, m)
        c = _compare(got[:2], (rd, rfin), 0, "interpreter")
        del si, got
        _report(f"{name}: AMWG_JIT=0 handle equals the reference on all {c} chains")
    short = m.get("lanes") == "short"
    for shape, C, off in plan:
        t0 = time.perf_counter()
        s = _make(gpu_pkg, monkeypatch, m, BASE + off, C)
        _assert_shape(s, shape, m)
        assert C % shape[0] != 0
        d, fin, _ = _run(s, m)
        c = _compare((d, fin), (rd, rfin), off, shape)
        lanes = _lanes(shape[0], C, short)
        n_orc, audited = _oracle_window(orc, s, m, d, fin, lanes, BASE + off, consts)
        del s, d, fin
        _report(f"{name}: {shape[0]} threads x {shape[1]} CTAs/SM, working set in {'shared' if shape[2] else 'global'} memory: "
                f"{C} chains from {BASE + off}; {c} chains equal to the reference; oracle lanes {lanes}: {n_orc} compared, "
                f"{audited} audited as ties; {time.perf_counter() - t0:.1f} s")
    # restore across shapes, once per skeleton: the two kept shapes least like the reference's
    if name in ("a_config2", "c_spike"):
        far = sorted(keep, key=lambda k: (k[2] != ref_shape[2], abs(k[0] - 128), k[1]), reverse=True)[:2]
        for shape in far:
            C, off = keep[shape], dict((k, o) for k, _, o in plan)[shape]
            s = _make(gpu_pkg, monkeypatch, m, BASE + off, C)
            _assert_shape(s, shape, m)
            d, fin, _ = _run(s, m, restore_from=img)
            c = _compare((d, fin), (rd, rfin), off, ("restored", shape))
            del s
            _report(f"{name}: restored into {shape} at {C} chains: {c} chains continue as the run that never stopped")
    _report(f"{name}: {time.perf_counter() - t_start:.1f} s")
