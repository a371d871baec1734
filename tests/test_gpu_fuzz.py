"""Randomly composed models through every sweep kernel on the GPU, against the oracle chain for chain.

The models are those of tests/test_jit_codegen_fuzz.py's builders, and only the seeds listed there in GPU_SEEDS: each of them has first
run through the emulated specialised kernels under the strict shim (bulk copies, mbarrier accounting, declared shared memory,
device-shaped columns) and under AddressSanitizer. Each model runs on every path it is eligible for, each handle built under the
kernel switches that select the path, and asserts the path it took:

  interpreter, faithful        AMWG_JIT=0, options.faithful
  interpreter, defaults        AMWG_JIT=0: term cache, block steps, the statistics sweep where the tracer chose it
  specialised full program     AMWG_JIT=1, options.faithful (with AMWG_TERM_CACHE=0 where that lowering keeps a term cache)
  specialised statistics       AMWG_JIT=1, the production lowering of a statistics model

The reference is one OracleSampler per checked chain over prog_eval.logpost of the faithful program, on the same seed and global chain
id. A run: burn 30, sample 24, then thin 2 and a monitor subset, sample 16 -- 70 sweeps, so the adaptation batch boundary at 50 falls
inside it. Chain counts 37 and 4099 (not multiples of a warp or a CTA) at nonzero first chains; about 8 chains checked per handle.

  bit-exact paths     draws, derived quantities, final state, stream position, adaptation state (info()) and log_post(), bit for bit
  statistics sweeps   the same, except that a chain may differ when its first differing decision is a rounding tie
                      (tests/stat_check.audit_divergence); at most 1 chain in 16 may; log_post() within rounding of the reference"""
import numpy as np
import pytest

import ckpt_ref
import plate_ref as pr
import prog_eval
import stat_check as sc
from test_jit_codegen_fuzz import GPU_SEEDS, gpu_model
from bayes_js_b200._ffi import PLATE_BERN_IID, PLATE_GENERIC

pytestmark = pytest.mark.gpu

BURN, SAMPLE1, SAMPLE2, THIN2 = 30, 24, 16, 2
SHAPES = {("generic", 3): (37, 1000), ("generic", 7): (4099, 2 ** 32 + 3), ("stat", 4): (4099, 77), ("stat", 51): (37, 5),
          ("shapes", 2): (37, 9), ("shapes", 7): (4099, 123)}


def _sampler(pkg, monkeypatch, params, log_post, data, chains, first, seed, env, faithful):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    o = {"chains": chains, "first_chain": first, "seed": seed, "device": 0}
    if faithful:
        o["faithful"] = True
    s = pkg.mcmc.AmwgSampler(params, log_post, data, o)
    for k in env:
        monkeypatch.delenv(k)
    return s


def _flat(rows_by_name, names, c, n_chains):
    """[rows, entries] of chain c over `names`, from a sample() result ([rows, chains, *dim] per name)"""
    return np.concatenate([np.asarray(rows_by_name[n], np.float64).reshape(len(rows_by_name[n]), n_chains, -1)[:, c] for n in names], axis=1)


class Reference:
    """the oracle's run of one global chain: draws of both sample calls, final state, stream position, info(), derived quantities"""

    def __init__(self, orc, prog, consts, params, derived_names, seed, gchain):
        O = orc.lib()
        self.prog, self.consts, self.O = prog, consts, O
        o = orc.OracleSampler(lambda st: prog_eval.logpost(prog, consts, st, O), None, params, seed=seed, chain=gchain)
        o.burn(BURN)
        self.r1 = o.sample(SAMPLE1)
        o.set_thin(THIN2)
        self.r2 = o.sample(SAMPLE2)
        self.D = o.D
        self.final = o.state()[:o.D]
        self.rng = o.rng_position()
        self.info = o.info()
        self.names = list(params)
        self.derived_names = derived_names

    def rows(self, r):
        return np.concatenate([np.asarray(r[n], np.float64).reshape(len(r[n]), -1) for n in self.names], axis=1)

    def derived(self, states):
        out = np.empty((len(states), len(self.derived_names)))
        for i, st in enumerate(states):
            pc = self.prog.derived_prog
            if self.prog.variant_comps:
                v = sum((1 << k) for k, c in enumerate(self.prog.variant_comps) if st[c] != 0)
                pc = self.prog.variant_derived[v]
            der = [None] * len(self.derived_names)
            prog_eval.run(self.prog, self.consts, st, pc, self.O, der=der)
            out[i] = der
        return out

    def logpost(self, st):
        return prog_eval.logpost(self.prog, self.consts, st, self.O)


def _paths(pkg, params, log_post, data):
    """-> [(name, env, faithful, exact)] the paths this model is eligible for"""
    probe = lambda **o: pkg.mcmc.AmwgSampler(params, log_post, data, dict({"chains": 4096, "_model_only": True}, **o))._program
    pf, pd = probe(faithful=True), probe()
    stat = pd.stat_prog >= 0
    plain = all(p["kind"] in (PLATE_GENERIC, PLATE_BERN_IID) for p in pd.plates)       # no factorised plate: the defaults are bit-exact
    out = [("interpreter faithful", {"AMWG_JIT": "0"}, True, True),
           ("interpreter defaults", {"AMWG_JIT": "0"}, False, plain and not stat),
           ("specialised full program", dict({"AMWG_JIT": "1"}, **({"AMWG_TERM_CACHE": "0"} if pf.n_terms > 0 else {})), True, True)]
    if stat:
        out.append(("specialised statistics", {"AMWG_JIT": "1"}, False, False))
    return out


def _check_path(s, path, faithful, exact, stat):
    on, note = s.jit_status()
    prog = s._program
    if path.startswith("interpreter"):
        assert not on and "AMWG_JIT=0" in note, (path, note)
        assert len(s.plate_sources()) == len(prog.plates), (path, s.plate_sources())
        assert s._term_cache().shape[0] == (prog.n_terms if prog.n_terms > 0 else 0), path
        if faithful:
            assert all(p["kind"] in (PLATE_GENERIC, PLATE_BERN_IID) for p in prog.plates), path
            assert all(src in ("loop", "shared", "L2", "ring") for src in s.plate_sources())
        else:
            assert (prog.stat_prog >= 0) == stat, path
    elif path == "specialised full program":
        assert on and note.startswith("specialised full-program sweep"), (path, note)
    else:
        assert on and note.startswith("specialised sweep") and prog.stat_prog >= 0, (path, note)


def _info_rows(s, names, c):
    """[D, 4] of chain c: prop_log_scale, acceptance_count, iterations_since_adaption, batch_count (NaN rows for binary parameters)"""
    inf = s.info()["steppers"][0]
    rows = []
    for n in names:
        k = int(np.prod(s.params[n]["dim"]))
        q = inf[n]
        if not q:
            rows.append(np.full((k, 4), np.nan))
            continue
        pls = np.asarray(q["prop_log_scale"], np.float64)[..., c].reshape(-1)
        acc = np.asarray(q["acceptance_count"], np.float64)[..., c].reshape(-1)
        it = np.broadcast_to(np.asarray(q["iterations_since_adaption"], np.float64).reshape(-1), (k,))
        bc = np.broadcast_to(np.asarray(q["batch_count"], np.float64).reshape(-1), (k,))
        rows.append(np.stack([pls, acc, it, bc], axis=1))
    return np.concatenate(rows, axis=0)


@pytest.mark.parametrize("kind,seed", GPU_SEEDS)
def test_random_models_on_every_sweep_kernel_against_the_oracle(gpu_pkg, orc, monkeypatch, kind, seed):
    pr.require_extended()
    pkg = gpu_pkg
    params, log_post, data = gpu_model(pkg, kind, seed)
    chains, first = SHAPES[(kind, seed)]
    rseed = 100 + seed
    pf_s = pkg.mcmc.AmwgSampler(params, log_post, data, {"chains": chains, "faithful": True, "_model_only": True})
    prog_f, names, dnames = pf_s._program, list(params), list(pf_s._derived_names)
    consts_f = prog_eval.fold_constants(prog_f, orc.lib())
    rng = np.random.default_rng(seed)
    checked = sorted({0, 31, 32, chains - 1} | {int(v) for v in rng.integers(0, chains, 4)})
    refs = {c: Reference(orc, prog_f, consts_f, params, dnames, rseed, first + c) for c in checked}
    D = refs[0].D
    monitor = names[::-1][:max(1, len(names) - 1)] + dnames                 # a subset, in another order, with the derived quantities
    paths = _paths(pkg, params, log_post, data)
    stat = any(p[0] == "specialised statistics" for p in paths)
    assert len(paths) >= 3
    for path, env, faithful, exact in paths:
        s = _sampler(pkg, monkeypatch, params, log_post, data, chains, first, rseed, env, faithful)
        _check_path(s, path, faithful, exact, stat)
        s.burn(BURN)
        d1 = s.sample(SAMPLE1)
        s.thin(THIN2)
        s.monitor(monitor)
        d2 = s.sample(SAMPLE2)
        assert list(d2.keys()) == monitor
        st = s.state
        final = np.concatenate([np.asarray(st[n], np.float64).reshape(chains, -1) for n in names], axis=1)
        rng_n = ckpt_ref.parse(s.checkpoint())["rng_n"]
        lp = np.asarray(s.log_post(), np.float64).reshape(-1)
        prog, consts = s._program, prog_eval.fold_constants(s._program, orc.lib())
        diverged = []
        for c in checked:
            ref = refs[c]
            g1, o1 = _flat(d1, names, c, chains), ref.rows(ref.r1)
            mon_p = [n for n in monitor if n in params]
            g2 = _flat(d2, mon_p, c, chains)
            o2 = np.concatenate([np.asarray(ref.r2[n], np.float64).reshape(len(ref.r2[n]), -1) for n in mon_p], axis=1)
            same = (np.array_equal(g1.view(np.uint64), o1.view(np.uint64)) and np.array_equal(g2.view(np.uint64), o2.view(np.uint64))
                    and np.array_equal(final[c].view(np.uint64), ref.final.view(np.uint64)))
            if not same:
                assert not exact, (path, kind, seed, c, "draws differ on a bit-exact path")
                diverged.append((c, g1, o1))
                continue
            if dnames:                                      # derived quantities of the recorded rows, from the oracle's rows
                g_der = _flat(d1, dnames, c, chains)
                assert np.array_equal(g_der.view(np.uint64), ref.derived(o1).view(np.uint64)), (path, c, "derived, first sample")
                full2 = ref.rows(ref.r2)
                assert np.array_equal(_flat(d2, dnames, c, chains).view(np.uint64), ref.derived(full2).view(np.uint64)), (path, c, "derived")
            assert int(rng_n[c]) == ref.rng, (path, c, int(rng_n[c]), ref.rng)
            got_info, want = _info_rows(s, names, c), ref.info[:, [0, 2, 3, 4]]
            assert np.array_equal(got_info.view(np.uint64), want.view(np.uint64)) or \
                np.array_equal(np.isnan(got_info), np.isnan(want)) and np.array_equal(got_info[~np.isnan(got_info)], want[~np.isnan(want)]), \
                (path, c, got_info, want)
            want_lp = ref.logpost(final[c])
            if exact:
                assert np.float64(lp[c]).view(np.uint64) == np.float64(want_lp).view(np.uint64) or (lp[c] != lp[c] and want_lp != want_lp), \
                    (path, c, lp[c], want_lp)
            else:
                assert abs(lp[c] - want_lp) <= 1e-11 * (1.0 + abs(want_lp)), (path, c, lp[c], want_lp)
        assert len(diverged) * 16 <= len(checked), (path, [c for c, *_ in diverged])
        for c, g1, o1 in diverged:
            r = np.flatnonzero((g1.view(np.uint64) != o1.view(np.uint64)).any(axis=1))
            assert r.size and r[0] > 0, (path, c, "the divergence lies in the burn or the thinned sample and cannot be localised")
            r = int(r[0])
            o = orc.OracleSampler(lambda x: prog_eval.logpost(prog_f, consts_f, x, orc.lib()), None, params, seed=rseed, chain=first + c)
            o.trace((BURN + SAMPLE1) * D)
            o.burn(BURN)
            o.sample(SAMPLE1)
            tr = o.trace_rows()
            sweep = BURN + r - 1
            n_pts = sum(len(np.asarray(col).ravel()) for col in prog.columns)
            err = lambda x: pr.gamma(n_pts + 64) * (abs(float(refs[c].logpost(x))) + n_pts)
            sc.audit_divergence(prog, consts, tr[sweep * D:(sweep + 1) * D], g1[r - 1], g1[r], o1[r], pr.JRING_TILE, err)
        print(f"{kind} {seed} {path}: {chains} chains from {first}, {len(checked)} checked, {len(diverged)} audited as ties; {s.jit_status()[1]}")
        s.close()
