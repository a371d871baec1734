"""Checks of the statistics sweeps (csrc/amwg_jit_kernel.cuh amwg_jit_sweep, csrc/amwg_kernels.cu amwg_stat_sweep_kernel) at extended
precision -- test infrastructure, CPU only.

  slots()             what each slot of a statistics model's term cache holds, read from the lowered program (amwg.h stat_prog):
                      the log_post program stores every term of the sum into its slot (ld.norm / ld.unif priors, the Normal plates'
                      terms NORM_SS(S, sd)), and its PLATE_SS instructions name the slot of each plate's statistic S = sum (x_i - mean)^2.
  check_term_cache()  every slot of every chain against tests/plate_ref.py at the chain's own state.
  audit_divergence()  a chain whose draws differ from the oracle's: the first decision that differs must be a rounding tie.
"""
import math

import numpy as np

import plate_ref as pr
from plate_ref import LD, U, gamma
from bayes_js_b200._ffi import OP

INV = {v: k for k, v in OP.items()}
_BIN = {"ADD": np.add, "SUB": np.subtract, "MUL": np.multiply, "DIV": np.divide}


class Operand:
    """an operand of the program as a function of the states [C, D] (fp64, the program's own operations), and what it reads"""

    def __init__(self, f, comps=(), const=None):
        self.f, self.comps, self.const = f, frozenset(comps), const

    def __call__(self, st):
        return np.asarray(self.f(np.atleast_2d(st)), dtype=np.float64)


def _comp(c):
    return Operand(lambda st: st[:, c], {c})


def _const(v):
    return Operand(lambda st: np.full(st.shape[0], v), (), const=v)


class Slot:
    """kind: "norm" (ld.norm(x, mean, sd), sd a constant), "unif" (ld.unif(x, lo, hi)), "plate" (the term of NORM_IID plate q:
    n (c0 - log sd) - S / (2 sd sd)), "stat" (S of plate q), "other" (an ld.* this module has no reference for: `op`)"""

    def __init__(self, kind, **kw):
        self.kind = kind
        self.__dict__.update(kw)

    def reads(self):
        ops = [getattr(self, k) for k in ("x", "mean", "sd") if isinstance(getattr(self, k, None), Operand)]
        return frozenset().union(*[o.comps for o in ops]) | getattr(self, "extra", frozenset())

    def points(self, prog):
        pl = prog.plates[self.q]
        col = np.asarray(prog.columns[pl["col"][0]], dtype=np.float64)
        return col[pl["iparam"][2]:pl["iparam"][2] + pl["n"]]

    def reference(self, prog, st, tile):
        """-> (value [C] longdouble, bound [C], median per-point summand [C] or None) at the states st [C, D]"""
        if self.kind == "norm":
            v, b = pr.norm_term(self.x(st), self.mean(st), self.sd)
            return v, b, None
        if self.kind == "unif":
            v, b = pr.unif_term(self.x(st), self.lo, self.hi)
            return v, b, None
        if self.kind == "plate":
            return pr.norm_plate(self.points(prog), self.mean(st), self.sd(st), tile=tile)
        if self.kind == "stat":
            r = pr.sum_sq(self.points(prog), self.mean(st), tile=tile)
            return r.value, r.bound, r.row_median
        raise AssertionError(f"no reference for {self.kind}")


def slots(prog, consts):
    """[n_terms] Slot: decode the log_post program of a statistics model (stat_prog >= 0). consts: the constants with the device's
    folded values filled in (tests/prog_eval.fold_constants)."""
    assert prog.stat_prog >= 0, "not a statistics model"
    code, pc, stk = prog.code, prog.logpost_prog, []
    out = [None] * prog.n_terms

    def nxt():
        nonlocal pc
        pc += 1
        return code[pc - 1]

    def opnd(mode):
        if mode == 0:
            return stk.pop()
        ix = nxt()
        if mode == 1:
            return _const(float(consts[ix]))
        assert mode == 2, mode
        return _comp(ix)

    while True:
        w = nxt() & 0xffffffff
        op = INV[w & 0xff]
        m = [(w >> s) & 3 for s in (8, 10, 12, 14)]
        acc, store, a = (w >> 16) & 1, (w >> 17) & 1, w >> 18
        if op == "END":
            break
        val = term = None
        if op == "CONST":
            val = _const(float(consts[a]))
        elif op == "COMP":
            val = _comp(a)
        elif op in _BIN:
            y, x = opnd(m[1]), opnd(m[0])
            val = Operand(lambda st, x=x, y=y, f=_BIN[op]: f(x(st), y(st)), x.comps | y.comps)
        elif op == "NEG":
            x = opnd(m[0])
            val = Operand(lambda st, x=x: -x(st), x.comps)
        elif op in ("NORM_K", "UNIF_K"):
            k, z, y, x = opnd(m[3]), opnd(m[2]), opnd(m[1]), opnd(m[0])
            if op == "NORM_K":                       # (x, mean, K1, K2 = 2 sd sd)
                sd = math.sqrt(k.const / 2)
                assert 2 * sd * sd == k.const, k.const
                term = Slot("norm", x=x, mean=y, sd=sd)
            else:                                    # (x, min, max, K)
                term = Slot("unif", x=x, lo=y.const, hi=z.const)
        elif op.startswith("LD_"):
            n = {"LD_BERN": 2, "LD_POIS": 2, "LD_EXP": 2, "LD_T": 4, "LD_HYPER": 4}.get(op, 3)
            args = [opnd(mm) for mm in m[:n][::-1]]
            term = Slot("other", op=op, extra=frozenset().union(*[o.comps for o in args]))
        elif op == "PLATE_SS":
            mean = opnd(m[0])
            out[nxt()] = Slot("stat", q=a, mean=mean)
            val = ("S", a, mean)
        elif op == "NORM_SS":
            sd, S = opnd(m[1]), opnd(m[0])
            assert isinstance(S, tuple) and S[1] == a, (op, S)
            term = Slot("plate", q=a, mean=S[2], sd=sd)
        else:
            raise AssertionError(f"{op} in a statistics model's log_post: not mapped")
        if term is not None:
            assert acc and store, f"{op}: a term of the sum is accumulated and stored"
            out[nxt()] = term
        elif acc:
            raise AssertionError(f"{op} accumulated without a term slot")
        else:
            stk.append(val)
    return out


def check_term_cache(prog, consts, cache, states, tile, what, skip=()):
    """Every slot of every chain: cache [n_terms, C] against the reference at states [C, D] (the chains' components), within the
    bound of the kernel's fp64 operations (tile: the points per streamed tile of the kernel's ring). Plate terms and statistics also
    pass plate_ref's sensitivity test. A slot the map does not cover fails, unless its ld.* op is listed in `skip`.
    -> {"stat": worst err / bound of the statistic slots, "term": of the other slots, "skipped": ops skipped}"""
    sl = slots(prog, consts)
    cache = np.asarray(cache, dtype=np.float64)
    assert cache.shape == (len(sl), states.shape[0]), (what, cache.shape, len(sl), states.shape)
    worst = {"stat": 0.0, "term": 0.0, "skipped": []}
    n_stat = 0
    for t, s in enumerate(sl):
        assert s is not None, f"{what}: slot {t} is neither a term of the sum nor a statistic"
        if s.kind == "other":
            assert s.op in skip, f"{what}: slot {t} holds {s.op}, which has no reference here"
            worst["skipped"].append(s.op)
            continue
        assert (s.kind == "stat") == (t >= prog.n_sum_terms), (what, t, s.kind, prog.n_sum_terms)
        n_stat += s.kind == "stat"
        ref = pr.per_state(lambda u: pr.Value(*_with_med(s.reference(prog, u, tile))), states)
        value, bound = ref.value, ref.bound
        got = cache[t]
        if s.kind in ("plate", "stat"):
            ref.check(got, f"{what}: slot {t} ({s.kind} of plate {s.q})")
        else:
            err = np.abs(got.astype(LD) - value).astype(np.float64)
            assert np.all(err <= bound), (what, t, s.kind, int(np.sum(~(err <= bound))), float(np.max(err / bound)))
        r = float(np.max(np.abs(got.astype(LD) - value).astype(np.float64) / bound))
        key = "stat" if s.kind == "stat" else "term"
        worst[key] = max(worst[key], r)
    assert n_stat == prog.n_terms - prog.n_sum_terms
    return worst


def _with_med(r):
    v, b, m = r
    return v, b, (m if m is not None else np.full(np.shape(v), np.nan))


# ---- the audit of a chain whose decisions differ from the oracle's -----------------------------------------------------------
def delta_ref(prog, sl, state, c, prop, tile):
    """delta* = log_post(proposal) - log_post(state) at extended precision, as the specialised sweep forms it: the sum over the terms
    of the sum that read component c of (new value - cached value). -> (delta*, B_gpu), B_gpu the worst-case error of the kernel's
    delta: every new and cached term within its plate_ref bound, then one difference per term and the running sum over them."""
    s0 = np.asarray(state, dtype=np.float64)[None, :]
    s1 = s0.copy()
    s1[0, c] = prop
    d, b, mag, k = LD(0), 0.0, 0.0, 0
    for s in sl:
        if s.kind == "stat" or c not in s.reads():
            continue
        assert s.kind != "other", f"component {c} moves {s.op}, which has no reference here"
        v0, b0, _ = s.reference(prog, s0, tile)
        v1, b1, _ = s.reference(prog, s1, tile)
        d += v1[0] - v0[0]
        b += float(b0[0]) + float(b1[0])
        mag += abs(float(v0[0])) + abs(float(v1[0])) + float(b0[0]) + float(b1[0])
        k += 1
    return d, b + gamma(2 * k + 1) * mag


def audit_divergence(prog, consts, steps, before, gpu_after, orc_after, tile, oracle_error):
    """A chain whose recorded rows first differ from the oracle's at row r (thin 1): `before` is row r - 1 (equal on both sides),
    gpu_after / orc_after are row r (the D components), `steps` the oracle's trace rows (OracleSampler.trace) of the sweep between
    them. Within a sweep the proposals and accept uniforms do not depend on any decision (each component is stepped once, from its
    value at the start of the sweep, and draws one uniform when its proposal is in bounds): the oracle's trace is the GPU's too, and
    each side's decision on component c is `after[c] == proposal`. At the first step (in the oracle's order) where the decisions
    differ the state is the same on both sides, and it must be a rounding tie:

        |log u - delta*| <= B_gpu + B_oracle + 2^-51

    with delta* at extended precision (delta_ref), B_gpu the specialised sweep's error bound (delta_ref), B_oracle that of the oracle's
    two term-by-term evaluations of log_post (oracle_error(state), per evaluation) and 2^-51 for the rounding of exp.

    The group means of a hierarchical model (JBLOCK) are stepped by the GPU in index order, by the oracle in the chain's visiting
    order; their terms are disjoint (each reads one mean and the shared sd, which is stepped before or after the whole block on both
    sides), so every mean's delta is the same in either order and the first differing decision in the oracle's order is still taken
    at the same state. -> (component, |log u - delta*|, bound); raises AssertionError when the divergence is not a tie."""
    sl = slots(prog, consts)
    state = np.array(before, dtype=np.float64)
    for c, cur, prop, u, _lc, _lp in np.asarray(steps, dtype=np.float64):
        c = int(c)
        assert cur == state[c], ("the trace does not start from the row before", c, cur, state[c])
        assert gpu_after[c] in (cur, prop), ("the GPU's value is neither the current value nor the proposal", c, gpu_after[c], cur, prop)
        g_acc, o_acc = gpu_after[c] == prop != cur, orc_after[c] == prop != cur
        if g_acc != o_acc:
            assert u >= 0, ("a decision differs on an out-of-bounds proposal", c, prop)
            d, b_gpu = delta_ref(prog, sl, state, c, prop, tile)
            moved = state.copy()
            moved[c] = prop
            b_orc = oracle_error(state) + oracle_error(moved) + U * abs(float(d))
            gap = abs(math.log(u) - float(d)) if u > 0 else math.inf
            bound = b_gpu + b_orc + 2.0 ** -51
            assert gap <= bound, ("not a rounding tie: a wrong decision", c, float(d), math.log(u) if u > 0 else None, gap, bound)
            return c, gap, bound
        if o_acc:
            state[c] = prop
    raise AssertionError("the rows differ but every decision agrees: a wrong value, not a tie")


def oracle_decisions_agree(prog, consts, steps, start, tile, oracle_error):
    """Every traced step of the oracle, from state `start`: its decision is exp(delta*) > u unless |log u - delta*| is within the
    bound -- the audit accepts the oracle's own decisions. -> the smallest |log u - delta*| / bound seen."""
    sl = slots(prog, consts)
    state = np.array(start, dtype=np.float64)
    smallest = math.inf
    for c, cur, prop, u, lc, lp in np.asarray(steps, dtype=np.float64):
        c = int(c)
        assert cur == state[c]
        if u < 0:
            continue
        acc = lp - lc >= 0 or math.exp(lp - lc) > u
        d, b_gpu = delta_ref(prog, sl, state, c, prop, tile)
        moved = state.copy()
        moved[c] = prop
        bound = b_gpu + oracle_error(state) + oracle_error(moved) + U * abs(float(d)) + 2.0 ** -51
        gap = math.log(u) - float(d) if u > 0 else -math.inf
        if abs(gap) > bound:
            assert acc == (gap < 0), (c, cur, prop, u, float(d))
        smallest = min(smallest, abs(gap) / bound)
        if acc:
            state[c] = prop
    return smallest
