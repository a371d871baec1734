"""Turn a ``log_post(state, data)`` closure into the program the CUDA sampler runs.

The reference calls an opaque JS closure twice per parameter step (mcmc.js:958-960, 524-526).  A GPU
cannot call back into the host per step, so the closure is executed ONCE here with symbolic
parameter values and proxied data; what it computes is recorded as an expression, then lowered to
the postfix program of include/amwg.h:

* the returned value is split along its left spine of ``+`` into terms, preserving the order of the
  user's ``log_post += ...`` statements (so the device forms the sum in the JS order);
* runs of structurally identical terms that walk through the data (``for i: log_post +=
  ld.norm(data[i], mu, sigma)``) become *plates*; recognised plate bodies get a hand-written
  inner loop (AMWG_PLATE_*), anything else is interpreted per point;
* keys the closure adds to ``state`` (``par.var = sigma*sigma``, tests/test_data.js:89) become
  derived quantities.

Python control flow on a BINARY parameter (``if m == 0:``) is handled by recording the closure once per
configuration of the binary components (see trace()); control flow on a real / int parameter cannot be
recorded: use ``where(cond, a, b)``.  Such closures raise ``JsThrow`` -- there is no CPU fallback.
"""
from __future__ import annotations

import math
import numbers
from typing import Any, Dict, List, Optional, Sequence, Tuple

import os

import numpy as np

from ._ffi import (OP, PLATE_BERN_IID, PLATE_GENERIC, PLATE_NORM_GROUPED, PLATE_NORM_IID, PLATE_POIS_LOGLIN)


class JsThrow(Exception):
    """The reference throws bare strings (``throw "..."``); Python needs an exception type.
    ``str(e)`` / ``e.message`` is exactly the string the reference would throw."""

    def __init__(self, message: str):
        super().__init__(message)
        self.message = message


class NeedsConcrete(JsThrow):
    """log_post used a symbolic value where Python needs a concrete one (`if m == 0:`). When only binary parameters are
    involved the tracer retries with those parameters concrete, once per configuration (see trace())."""


# ------------------------------------------------------------------------------------------------
# symbolic values
# ------------------------------------------------------------------------------------------------
class Sym:
    """A node of the recorded expression. ``op`` is an opcode name of include/amwg.h."""
    __slots__ = ("op", "args", "val")

    def __init__(self, op: str, args: tuple = (), val: Any = None):
        self.op = op
        self.args = args
        self.val = val

    # arithmetic: one IEEE operation per node, like the JS operator it mirrors
    def __add__(self, o): return Sym("ADD", (self, lift(o)))
    def __radd__(self, o): return Sym("ADD", (lift(o), self))
    def __sub__(self, o): return Sym("SUB", (self, lift(o)))
    def __rsub__(self, o): return Sym("SUB", (lift(o), self))
    def __mul__(self, o): return Sym("MUL", (self, lift(o)))
    def __rmul__(self, o): return Sym("MUL", (lift(o), self))
    def __truediv__(self, o): return Sym("DIV", (self, lift(o)))
    def __rtruediv__(self, o): return Sym("DIV", (lift(o), self))
    def __pow__(self, o): return Sym("POW", (self, lift(o)))
    def __rpow__(self, o): return Sym("POW", (lift(o), self))
    def __neg__(self): return Sym("NEG", (self,))
    def __pos__(self): return self
    def __abs__(self): return Sym("ABS", (self,))
    def __lt__(self, o): return Sym("LT", (self, lift(o)))
    def __le__(self, o): return Sym("LE", (self, lift(o)))
    def __gt__(self, o): return Sym("GT", (self, lift(o)))
    def __ge__(self, o): return Sym("GE", (self, lift(o)))
    def __eq__(self, o): return Sym("EQ", (self, lift(o)))   # noqa: E721  (symbolic comparison)
    def __ne__(self, o): return Sym("NE", (self, lift(o)))
    __hash__ = object.__hash__

    def __bool__(self):
        raise NeedsConcrete("log_post branches on a parameter value, which cannot be traced for the device; "
                            "use mcmc.where(cond, a, b)")

    def __float__(self):
        raise NeedsConcrete("log_post converts a parameter to a Python float (e.g. math.log); use mcmc.Math.* / ld.*")

    def __index__(self):
        raise NeedsConcrete("log_post uses a parameter value as an index; only binary parameters can be used that way")

    def __repr__(self):
        if self.op == "CONST": return f"{self.val!r}"
        if self.op in ("COMP", "DATA", "DATA_I", "COMP_I"): return f"{self.op}{self.val}"
        return f"{self.op}({', '.join(map(repr, self.args))})"


def lift(x) -> Sym:
    if isinstance(x, Sym):
        return x
    if isinstance(x, (bool, np.bool_)):
        return Sym("CONST", (), 1.0 if x else 0.0)
    if isinstance(x, numbers.Real):
        return Sym("CONST", (), float(x))
    raise JsThrow(f"log_post produced a value of type {type(x).__name__} that is not a number")


def is_sym(x) -> bool:
    return isinstance(x, Sym)


def where(cond, a, b):
    """``cond ? a : b`` with both branches evaluated (device SELECT)."""
    if not is_sym(cond) and not is_sym(a) and not is_sym(b):
        return a if cond else b
    return Sym("SELECT", (lift(cond), lift(a), lift(b)))


def _unary(op):
    def f(x):
        return Sym(op, (lift(x),))
    return f


class _Math:
    """``Math.*`` for use inside log_post: symbolic in, symbolic out (evaluated on the device with JS semantics)."""
    PI = 3.141592653589793
    E = 2.718281828459045
    log = staticmethod(_unary("LOG"))
    exp = staticmethod(_unary("EXP"))
    sqrt = staticmethod(_unary("SQRT"))
    abs = staticmethod(_unary("ABS"))

    @staticmethod
    def pow(x, y): return Sym("POW", (lift(x), lift(y)))

    @staticmethod
    def max(a, b):
        """Math.max: NaN if either argument is NaN (x != x), like the engine's"""
        a, b = lift(a), lift(b)
        return where(Sym("OR", (a != a, b != b)), float("nan"), where(a > b, a, b))

    @staticmethod
    def min(a, b):
        a, b = lift(a), lift(b)
        return where(Sym("OR", (a != a, b != b)), float("nan"), where(a < b, a, b))


Math = _Math()


# ------------------------------------------------------------------------------------------------
# proxies handed to the closure
# ------------------------------------------------------------------------------------------------
class PlateIndex:
    """Symbolic loop index: ``for i in mcmc.points(n): log_post += ld.norm(data[i], mu, sigma)``
    records the body once for all n points (the concrete ``for i in range(n)`` form is traced point by
    point and compressed afterwards; both give the same program)."""
    __slots__ = ("n", "plate_id")

    def __init__(self, n: int, plate_id: int):
        self.n = int(n)
        self.plate_id = plate_id


class _Points:
    def __init__(self, tracer: "Tracer", n: int):
        self.tracer, self.n = tracer, int(n)

    def __iter__(self):
        if self.n > 0:
            yield self.tracer.new_plate_index(self.n)


class DataVec:
    """A 1-D or nested numeric array from ``data``. Elements stay symbolic references into a device column."""

    def __init__(self, tracer: "Tracer", col: int, shape: Tuple[int, ...], offset: int = 0):
        self._t, self._col, self._shape, self._off = tracer, col, tuple(shape), offset

    def __len__(self): return self._shape[0]

    @property
    def length(self): return self._shape[0]        # JS spelling

    def _inner(self) -> int:
        n = 1
        for d in self._shape[1:]: n *= d
        return n

    def __getitem__(self, i):
        inner = self._inner()
        if isinstance(i, PlateIndex):
            if i.n > self._shape[0]:
                raise JsThrow("plate index runs past the end of a data array")
            if len(self._shape) == 1:
                return Sym("DATA_I", (), (self._col, self._off, 1, i.plate_id))
            return _DataRowI(self._t, self._col, self._shape[1:], self._off, inner, i.plate_id)
        if isinstance(i, Sym):
            raise JsThrow("indexing data by a parameter value is not supported on the device")
        i = int(i)
        if i < 0: i += self._shape[0]
        if not 0 <= i < self._shape[0]:
            return Sym("CONST", (), float("nan"))          # JS: undefined -> NaN in arithmetic
        if len(self._shape) == 1:
            return Sym("DATA", (), (self._col, self._off + i))
        return DataVec(self._t, self._col, self._shape[1:], self._off + i * inner)

    def __iter__(self):
        for i in range(self._shape[0]):
            yield self[i]

    def value(self, i: int) -> float:
        return float(self._t.columns[self._col][self._off + i])


class _DataRowI:
    """``data.X[i]`` with a symbolic i: row of a 2-D array."""

    def __init__(self, tracer, col, shape, off, row_stride, plate_id):
        self._t, self._col, self._shape, self._off, self._rs, self._pid = tracer, col, tuple(shape), off, row_stride, plate_id

    def __len__(self): return self._shape[0]

    def __getitem__(self, k):
        if len(self._shape) != 1:
            raise JsThrow("data arrays deeper than 2 levels under a plate index are not supported")
        k = int(k)
        return Sym("DATA_I", (), (self._col, self._off + k, self._rs, self._pid))

    def __iter__(self):
        for k in range(self._shape[0]):
            yield self[k]


class ParamVec:
    """State of a multi-dim parameter: nested, indexable by ints, by data values and by plate-indexed data."""

    def __init__(self, tracer: "Tracer", comp0: int, shape: Tuple[int, ...]):
        self._t, self._c0, self._shape = tracer, comp0, tuple(shape)

    def __len__(self): return self._shape[0]

    @property
    def length(self): return self._shape[0]

    def __getitem__(self, i):
        inner = 1
        for d in self._shape[1:]: inner *= d
        if isinstance(i, Sym):
            if i.op == "DATA":                      # concrete data value used as an index (mu[g[i]])
                v = float(self._t.columns[i.val[0]][i.val[1]])
                if v != math.floor(v):
                    return Sym("CONST", (), float("nan"))          # JS: a[1.5] is undefined
                i = int(v)
            elif i.op == "DATA_I" and len(self._shape) == 1:
                col, off, stride, pid = i.val
                n = self._t.plate_sizes.get(pid, 0)
                idx = self._t.columns[col][off: off + stride * max(n, 1): stride]
                # JS reads `undefined` outside the array (-> NaN, the chain never moves); on the device the read would alias another
                # parameter or leave the state array, so such a model is refused
                if idx.size and (np.any(idx != np.floor(idx)) or idx.min() < 0 or idx.max() >= self._shape[0]):
                    raise JsThrow("log_post indexes a parameter array of length %d with data values outside its bounds [%g, %g]"
                                  % (self._shape[0], float(idx.min()), float(idx.max())))
                return Sym("COMP_I", (), (col, off, stride, self._c0, pid))
            else:
                raise JsThrow("a parameter array can only be indexed by numbers or by data values")
        i = int(i)
        if i < 0: i += self._shape[0]
        if not 0 <= i < self._shape[0]:
            return Sym("CONST", (), float("nan"))
        if len(self._shape) == 1:
            return self._t.comp(self._c0 + i)
        return ParamVec(self._t, self._c0 + i * inner, self._shape[1:])

    def __iter__(self):
        for i in range(self._shape[0]):
            yield self[i]


class State(dict):
    """``state``: parameters by name, attribute or item access (``state.mu`` / ``state["mu"]``).
    Keys the closure adds are derived quantities (mcmc.js:961-963)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


class DataObject(dict):
    """``data`` when it is an object: attribute and item access."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


# ------------------------------------------------------------------------------------------------
# tracing + lowering
# ------------------------------------------------------------------------------------------------
_MIN_PLATE = 8          # shorter runs stay unrolled scalar terms
MAX_IMMEDIATE = 16383
STORE_FLAG = 1 << 17
MODE_STACK, MODE_CONST, MODE_COMP, MODE_NONE = 0, 1, 2, 3
_ARITY = {"ADD": 2, "SUB": 2, "MUL": 2, "DIV": 2, "NEG": 1, "LOG": 1, "EXP": 1, "SQRT": 1, "ABS": 1, "POW": 2,
          "LT": 2, "LE": 2, "GT": 2, "GE": 2, "EQ": 2, "NE": 2, "AND": 2, "OR": 2, "NOT": 1, "SELECT": 3,
          "LGAMMA": 1, "LFACTORIAL": 1, "LCHOOSE": 2, "LBETA": 2,
          "LD_NORM": 3, "LD_UNIF": 3, "LD_BETA": 3, "LD_BERN": 2, "LD_POIS": 2, "LD_CAUCHY": 3, "LD_LAPLACE": 3,
          "LD_GAMMA": 3, "LD_INVGAMMA": 3, "LD_LNORM": 3, "LD_PARETO": 3, "LD_T": 4, "LD_WEIBULL": 3, "LD_LOGIS": 3,
          "LD_EXP": 2, "LD_BINOM": 3, "LD_NBINOM": 3, "LD_HYPER": 4, "NORM_K": 4, "UNIF_K": 4, "BETA_K": 4}
ACC_FLAG = 1 << 16
MIN_STAT_POINTS = 64    # pre-evaluated statistics pay for their bookkeeping from about this many plate points


class Program:
    """The lowered model: everything amwg_model needs."""

    def __init__(self):
        self.code: List[int] = []
        self.consts: List[float] = []
        self._const_index: Dict[bytes, int] = {}
        self.columns: List[np.ndarray] = []
        self.plates: List[dict] = []
        self.logpost_prog = 0
        self.derived_prog = -1
        self.derived_names: List[str] = []
        self.store_sites: List[Tuple[int, int]] = []
        self.n_terms = 0                       # dependency-aware evaluation (amwg.h comp_prog): 0 = not in use
        self.comp_prog: List[int] = []
        self.touch_off: List[int] = []
        self.touch_terms: List[int] = []
        self.stat_prog = -1                    # pre-evaluated plate statistics (amwg.h stat_prog): -1 = not in use
        self.n_sum_terms = 0                   # ... terms of the sum; slots n_sum_terms .. n_terms-1 of the term cache hold the statistics
        self.block_params: List[int] = []      # parameters stepped with one evaluation (amwg.h block_params) ...
        self.term_block_comp: List[int] = []   # ... and, per such parameter, the component of it each term reads (-1: none)
        self.variant_comps: List[int] = []     # binary components whose configuration selects the program (amwg.h variant_*)
        self.variant_logpost: List[int] = []
        self.variant_derived: List[int] = []
        self.fold_prog: List[int] = []         # word offsets of constant sub-expression programs (evaluated once on the device)
        self.fold_dst: List[int] = []          # ... and the consts[] slot each one fills
        self.summary: List[str] = []           # human-readable: what each term became

    def const(self, v: float) -> int:
        key = np.float64(v).tobytes()
        k = self._const_index.get(key)
        if k is None:
            k = len(self.consts)
            self.consts.append(float(v))
            self._const_index[key] = k
        return k

    def fold_slot(self) -> int:
        self.consts.append(float("nan"))       # filled by amwg_fold_kernel at create
        return len(self.consts) - 1

    def emit(self, op: str, operand: int = 0, *extra: int, modes=(), acc: bool = False, store: Optional[int] = None):
        """One instruction word (include/amwg.h): opcode | operand modes A..D | ACC | STORE | 14-bit immediate, + extra words
        (`store`: term id, written last)."""
        operand = int(operand)
        if not 0 <= operand <= MAX_IMMEDIATE:
            raise JsThrow("log_post is too large for the device program format (immediate > 16383)")
        m = list(modes) + [MODE_NONE] * (4 - len(modes))
        word = OP[op] | (m[0] << 8) | (m[1] << 10) | (m[2] << 12) | (m[3] << 14) | ((1 if acc else 0) << 16) | (operand << 18)
        if store is not None:
            word |= STORE_FLAG
        self.code.append(word)
        self.code.extend(int(e) for e in extra)
        if store is not None:
            self.store_sites.append((len(self.code) - 1 - len(extra), len(self.code)))    # (flagged word, its term-id word)
            self.code.append(int(store))


class Tracer:
    def __init__(self):
        self.columns: List[np.ndarray] = []
        self._n_plate_idx = 0
        self.plate_sizes: Dict[int, int] = {}
        self.concrete: Dict[int, float] = {}   # component -> value, for binary components traced per configuration

    def comp(self, c: int):
        """state component c as the closure sees it: symbolic, or a plain number when traced per configuration"""
        return self.concrete[c] if c in self.concrete else Sym("COMP", (), c)

    # -- data -----------------------------------------------------------------------------------
    def add_column(self, arr: np.ndarray) -> int:
        self.columns.append(np.ascontiguousarray(arr, dtype=np.float64).reshape(-1))
        return len(self.columns) - 1

    def wrap_data(self, data):
        """Proxy `data` (any nesting of dicts / lists / arrays / numbers; opaque to the reference, mcmc.js:942)."""
        if data is None or isinstance(data, (str, bytes)):
            return data
        if isinstance(data, (bool, numbers.Real)):
            return float(data)
        if isinstance(data, dict):
            return DataObject({k: self.wrap_data(v) for k, v in data.items()})
        if isinstance(data, (list, tuple, np.ndarray)):
            try:
                arr = np.asarray(data, dtype=np.float64)
            except (ValueError, TypeError):
                return [self.wrap_data(v) for v in data]          # ragged / mixed: recurse
            if arr.ndim == 0:
                return float(arr)
            if arr.size == 0:
                return []
            col = self.add_column(arr)
            return DataVec(self, col, arr.shape)
        return data

    def new_plate_index(self, n: int) -> PlateIndex:
        pid = self._n_plate_idx
        self._n_plate_idx += 1
        self.plate_sizes[pid] = int(n)
        return PlateIndex(n, pid)

    def points(self, n) -> _Points:
        return _Points(self, int(n))

    # -- state ----------------------------------------------------------------------------------
    def make_state(self, params: Dict[str, dict], offsets: Dict[str, int]) -> State:
        st = State()
        for name, p in params.items():
            dim = list(p["dim"])
            if dim == [1]:
                st[name] = self.comp(offsets[name])
            else:
                st[name] = ParamVec(self, offsets[name], tuple(dim))
        return st


# ---- ld.* as the JS source spells them (distributions.js), in device primitives ------------------------------------
# A recorded LD_* node keeps its identity for plate recognition; when it is emitted as a scalar term or inside a
# generic plate body it is first expanded into exactly the operations of the JS function, so that sub-expressions
# without parameters (log(2*pi), log(sd) of a constant sd, lbeta(2,2) ...) can be folded to constants. Same operations,
# same order => same bits as the native LD_* opcode.
_NEG_INF = float("-inf")


def _c(v) -> Sym:
    return Sym("CONST", (), float(v))


def _or(a: Sym, b: Sym) -> Sym:
    return Sym("OR", (a, b))


def _is_const(n: Sym) -> bool:
    stack = [n]
    while stack:
        m = stack.pop()
        if m.op in ("COMP", "DATA_I", "COMP_I"):
            return False
        stack.extend(m.args)
    return True


def _const_value(n: Sym):
    """numeric value of a literal leaf (CONST), else None"""
    return n.val if n.op == "CONST" else None


def _expand_ld(op: str, a: Tuple[Sym, ...]) -> Optional[Sym]:
    log = Math.log
    if op == "LD_NORM":                                   # distributions.js:119-121
        x, mean, sd = a
        k1 = _c(-0.5) * log(_c(2) * _c(Math.PI)) - log(sd)
        k2 = _c(2) * sd * sd
        if _is_const(sd):                                 # constant sd (a prior): one fused op, K1/K2 folded on the device
            return Sym("NORM_K", (x, mean, k1, k2))
        return k1 - Math.pow(x - mean, 2) / k2
    if op == "LD_UNIF":                                   # :221-223
        x, mn, mx = a
        k = log(_c(1) / (mx - mn))
        if _is_const(mn) and _is_const(mx):
            return Sym("UNIF_K", (x, mn, mx, k))
        return where(_or(x < mn, x > mx), _NEG_INF, k)
    if op == "LD_BETA":                                   # :104-113
        x, s1, s2 = a
        if _const_value(s1) is not None and _const_value(s2) is not None:
            if _const_value(s1) == 1 and _const_value(s2) == 1:
                return where(_or(x > 1, x < 0), _NEG_INF, 0.0)
            return Sym("BETA_K", (x, s1 - 1, s2 - 1, Sym("LBETA", (s1, s2))))
        body = (s1 - 1) * log(x) + (s2 - 1) * log(_c(1) - x) - Sym("LBETA", (s1, s2))
        return where(_or(x > 1, x < 0), _NEG_INF, where(Sym("AND", (s1 == 1, s2 == 1)), 0.0, body))
    if op == "LD_BERN":                                   # :228-230
        x, p = a
        return where(Sym("NOT", (_or(x == 0, x == 1),)), _NEG_INF, log(x * p + (_c(1) - x) * (_c(1) - p)))
    if op == "LD_POIS":                                   # :282-284
        x, lam = a
        return where(x < 0, _NEG_INF, log(lam) * x - lam - Sym("LFACTORIAL", (x,)))
    if op == "LD_EXP":                                    # :217-219
        x, rate = a
        return where(x < 0, _NEG_INF, log(rate) - rate * x)
    if op == "LD_LAPLACE":                                # :136-138
        x, loc, scale = a
        return (-abs(x - loc) / scale) - log(_c(2) * scale)
    if op == "LD_CAUCHY":                                 # :115-117
        x, loc, scale = a
        return log(scale) - log(Math.pow(x - loc, 2) + Math.pow(scale, 2)) - log(_c(Math.PI))
    return None                                           # the rest stay native opcodes


def expand(node: Sym) -> Sym:
    """Rewrite expandable LD_* nodes into primitives (iteratively bottom-up; trees are shallow)."""
    if not node.args:
        return node
    args = tuple(expand(a) for a in node.args)
    if node.op.startswith("LD_"):
        e = _expand_ld(node.op, args)
        if e is not None:
            return e
    return Sym(node.op, args, node.val)


def _spine_terms(expr: Sym) -> List[Sym]:
    """((0 + t1) + t2) + ...  ->  [t1, t2, ...] (iterative: spines can be 1e6 deep)."""
    terms: List[Sym] = []
    node = expr
    while node.op == "ADD":
        terms.append(node.args[1])
        node = node.args[0]
    if not (node.op == "CONST" and node.val == 0.0 and terms):
        terms.append(node)
    terms.reverse()
    return terms


def _signature(node: Sym, slots: list):
    """Structure of a term with data positions abstracted; collects (kind, col, index[, base]) per slot."""
    if node.op == "CONST": return ("K", node.val if node.val == node.val else "nan")
    if node.op == "COMP": return ("C", node.val)
    if node.op == "DATA":
        slots.append(("D", node.val[0], node.val[1]))
        return ("D", node.val[0])
    if node.op in ("DATA_I", "COMP_I"):
        return (node.op, node.val)
    return (node.op,) + tuple(_signature(a, slots) for a in node.args)


def _signature_loose(node: Sym, slots: list):
    """As _signature, but parameter components are slots too (mu[g[i]] varies from point to point)."""
    if node.op == "CONST": return ("K", node.val if node.val == node.val else "nan")
    if node.op == "COMP":
        slots.append(("C", -1, node.val))
        return ("C?",)
    if node.op == "DATA":
        slots.append(("D", node.val[0], node.val[1]))
        return ("D", node.val[0])
    if node.op in ("DATA_I", "COMP_I"):
        return (node.op, node.val)
    return (node.op,) + tuple(_signature_loose(a, slots) for a in node.args)


def _has_plate_ref(node: Sym) -> Optional[int]:
    """plate id referenced by a symbolic-index term, or None."""
    stack = [node]
    while stack:
        n = stack.pop()
        if n.op == "DATA_I": return n.val[3]
        if n.op == "COMP_I": return n.val[4]
        stack.extend(n.args)
    return None


def _index_free(node: Sym) -> bool:
    stack = [node]
    while stack:
        n = stack.pop()
        if n.op in ("DATA_I", "COMP_I"): return False
        stack.extend(n.args)
    return True


class Lowering:
    def __init__(self, tracer: Tracer, n_comp: int, faithful: bool = False, param_ranges: Optional[List[Tuple[int, int, str]]] = None):
        self.t = tracer
        self.n_comp = n_comp
        self.param_ranges = param_ranges or []   # (first component, number of components, type) per named parameter, in order
        self.faithful = faithful                 # True: no factorised plates -- every likelihood loop is added term by term like the JS loop
        self.prog = Program()
        self.prog.columns = tracer.columns       # shared list: synthesized columns are appended
        self._fold_memo: Dict[tuple, int] = {}
        self._fold_trees: List[Tuple[int, Sym]] = []
        self._terms: List[dict] = []             # top-level terms of the (single) log_post program: start, end, kind, deps, cost
        self._abs_words: List[int] = []          # positions of words that hold absolute program offsets (loop targets)
        self._record_terms = False
        self._stat_mode = False                  # second lowering pass: NORM_IID plates as PLATE_SS + NORM_SS (amwg.h stat_prog)

    # -- constant folding ---------------------------------------------------------------------------
    def _key(self, n: Sym):
        if n.op == "CONST": return ("K", np.float64(n.val).tobytes())
        if n.op in ("COMP", "DATA", "DATA_I", "COMP_I", "FOLD"): return (n.op, n.val)
        return (n.op,) + tuple(self._key(a) for a in n.args)

    def fold(self, node: Sym) -> Sym:
        """Replace every maximal parameter-free sub-expression that contains at least one operation by a FOLD(k) leaf;
        consts[k] is computed once on the device (amwg_fold_kernel) with the device's own log/exp."""
        def rec(n: Sym):
            if n.op in ("CONST", "DATA", "FOLD"):
                return n, True
            if n.op in ("COMP", "DATA_I", "COMP_I"):
                return n, False
            parts = [rec(a) for a in n.args]
            if all(c for _, c in parts):
                return Sym(n.op, tuple(x for x, _ in parts), n.val), True
            new_args = tuple(self._to_fold(x) if (c and x.args) else x for x, c in parts)
            return Sym(n.op, new_args, n.val), False
        out, is_const = rec(node)
        return self._to_fold(out) if (is_const and out.args) else out

    def _to_fold(self, tree: Sym) -> Sym:
        key = self._key(tree)
        k = self._fold_memo.get(key)
        if k is None:
            k = self.prog.fold_slot()
            self._fold_memo[key] = k
            self._fold_trees.append((k, tree))
        return Sym("FOLD", (), k)

    # -- expressions ------------------------------------------------------------------------------
    def _inline(self, n: Sym):
        """(mode, word) when the operand can ride inside the instruction: constants and state components."""
        if n.op == "CONST": return MODE_CONST, self.prog.const(n.val)
        if n.op == "FOLD": return MODE_CONST, n.val
        if n.op == "COMP": return MODE_COMP, n.val
        return None

    def _operands(self, args):
        """Emit the stack operands (left to right) and return (modes, inline words in consumption order: last operand first)."""
        modes, words = [], []
        for a in args:
            il = self._inline(a)
            if il is None:
                self._emit(a, False)
                modes.append(MODE_STACK)
            else:
                modes.append(il[0])
                words.append(il[1])
        return modes, list(reversed(words))

    def _emit(self, n: Sym, acc: bool, store: Optional[int] = None):
        p = self.prog
        if n.op in ("CONST", "FOLD", "COMP"):
            mode, idx = self._inline(n)
            p.emit("CONST" if mode == MODE_CONST else "COMP", idx, acc=acc, store=store)
        elif n.op == "DATA":
            p.emit("DATA", n.val[0], n.val[1], acc=acc, store=store)
        elif n.op == "DATA_I":
            p.emit("DATA_I", n.val[0], n.val[1], n.val[2], acc=acc, store=store)
        elif n.op == "COMP_I":
            p.emit("COMP_I", n.val[0], n.val[1], n.val[2], n.val[3], acc=acc, store=store)
        else:
            if n.op not in _ARITY:
                raise JsThrow(f"cannot lower operation {n.op}")
            modes, words = self._operands(n.args)
            p.emit(n.op, 0, *words, modes=modes, acc=acc, store=store)

    def emit_expr(self, node: Sym, prepare: bool = True, acc: bool = False, store: Optional[int] = None):
        """Postfix emission. `prepare`: expand LD_* into primitives and fold constants first. `acc`: the value is
        added to lp (a term of the sum) instead of being left on the stack; `store`: ... and kept in the term cache as term `store`."""
        if prepare:
            node = self.fold(expand(node))
        import sys
        if sys.getrecursionlimit() < 20000:
            sys.setrecursionlimit(20000)
        self._emit(node, acc, store)

    def _deps(self, node: Sym) -> set:
        """state components an (expanded) expression reads"""
        out, stack = set(), [node]
        while stack:
            n = stack.pop()
            if n.op == "COMP":
                out.add(n.val)
            elif n.op == "COMP_I":
                col, off, stride, base, pid = n.val
                cnt = self.t.plate_sizes.get(pid, 0)
                idx = self.t.columns[col][off: off + stride * max(cnt, 1): stride] if cnt else self.t.columns[col]
                out.update(int(base + v) for v in np.unique(idx))
            stack.extend(n.args)
        return out

    def prepared(self, node: Sym) -> Sym:
        return self.fold(expand(node))

    # -- plates -----------------------------------------------------------------------------------
    def _emit_plate(self, body: Sym, n: int):
        """Emit the code for a plate over n points whose per-point term is `body` (uses DATA_I/COMP_I)."""
        p = self.prog
        pl = dict(kind=PLATE_GENERIC, n=n, col=[-1] * 4, iparam=[0] * 4)

        def data_i(node, stride=1):
            return node.op == "DATA_I" and node.val[2] == stride

        q = len(p.plates)
        operands: List[Sym] = []
        if self.faithful and body.op in ("LD_NORM", "LD_POIS"):
            pass                                                  # bytecode loop below: bit-faithful to the reference's arithmetic
        elif body.op == "LD_NORM" and data_i(body.args[0]) and _index_free(body.args[2]):
            x, mean, sd = body.args
            if _index_free(mean):
                pl.update(kind=PLATE_NORM_IID)
                pl["col"][0] = x.val[0]; pl["iparam"][2] = x.val[1]
                operands = [mean, sd]
                p.summary.append(f"plate NORM_IID n={n}")
            elif mean.op == "COMP_I":
                grp = self._grouped(mean, n)
                if grp is not None:
                    base, J, start_col = grp
                    pl.update(kind=PLATE_NORM_GROUPED)
                    pl["col"][0] = x.val[0]; pl["col"][1] = start_col; pl["iparam"][2] = x.val[1]
                    pl["iparam"][0] = base; pl["iparam"][1] = J
                    operands = [sd]
                    p.summary.append(f"plate NORM_GROUPED n={n} groups={J}")
        elif body.op == "LD_BERN" and data_i(body.args[0]) and _index_free(body.args[1]):
            pl.update(kind=PLATE_BERN_IID)
            pl["col"][0] = body.args[0].val[0]; pl["iparam"][2] = body.args[0].val[1]
            operands = [body.args[1]]
            p.summary.append(f"plate BERN_IID n={n}")
        elif body.op == "LD_POIS" and data_i(body.args[0]) and body.args[1].op == "EXP":
            lin = self._loglinear(body.args[1].args[0])
            y = body.args[0]
            ycol = self.t.columns[y.val[0]][y.val[1]: y.val[1] + n]
            # ld.pois of a negative count is -Infinity (distributions.js:282-284), whatever the rate; the factorised sum has no place
            # for it (its lfactorial constant would be NaN), so such data keeps the term-by-term loop
            if lin is not None and not np.any(ycol < 0):
                xcol, K, base = lin
                # sum_i [y_i eta_i - exp(eta_i) - lfactorial(y_i)]: the first part is beta . (X^T y), the last a constant; both are
                # precomputed here (constant in the parameters), the device sums exp(eta_i) over the rows
                X = self.t.columns[xcol][: n * K].reshape(n, K)
                stats = np.concatenate([X.T @ ycol, [float(np.sum(_lfactorial_host_vec(ycol)))]])
                pl.update(kind=PLATE_POIS_LOGLIN)
                pl["col"][0] = y.val[0]; pl["iparam"][2] = y.val[1]
                pl["col"][1] = xcol; pl["col"][2] = self.t.add_column(stats)
                pl["iparam"][0] = base; pl["iparam"][1] = K
                p.summary.append(f"plate POIS_LOGLIN n={n} K={K}")
        p.plates.append(pl)
        start = len(p.code)
        if pl["kind"] == PLATE_NORM_IID and self._stat_mode:
            # the O(N) statistic S(mean) and the O(1) combination f(S, sd) as two instructions, S kept in its own cache slot
            mean_p, sd_p = self.prepared(operands[0]), self.prepared(operands[1])
            k = sum(1 for tr in self._terms if tr.get("stat") is not None)
            modes, words = self._operands([mean_p])
            ss_word = len(p.code)
            p.emit("PLATE_SS", q, *words, -1 - k, modes=modes)          # slot patched once the number of terms is known
            split = len(p.code)
            m_sd, w_sd = self._operands([sd_p])
            p.emit("NORM_SS", q, *w_sd, modes=[MODE_STACK] + m_sd, acc=True, store=len(self._terms))
            self._terms.append(dict(start=start, end=len(p.code), kind="value", deps=self._deps(mean_p) | self._deps(sd_p), cost=3 * n,
                                    stat=dict(k=k, ss_word=ss_word, slot_word=split - 1, split=split, mean_deps=self._deps(mean_p), n=n)))
            return
        if pl["kind"] != PLATE_GENERIC:
            prepared = [self.prepared(o) for o in operands]
            modes, words = self._operands(prepared)
            value_plate = pl["kind"] != PLATE_BERN_IID              # the Bernoulli plate adds term by term into lp: not a separable value
            tid = len(self._terms) if (self._record_terms and value_plate) else None
            p.emit("PLATE", q, *words, modes=modes, store=tid)
            if self._record_terms:
                deps = set()
                for o in prepared:
                    deps |= self._deps(o)
                if pl["kind"] == PLATE_NORM_GROUPED or pl["kind"] == PLATE_POIS_LOGLIN:
                    deps |= set(range(pl["iparam"][0], pl["iparam"][0] + pl["iparam"][1]))
                self._terms.append(dict(start=start, end=len(p.code), kind="value" if value_plate else "inorder", deps=deps, cost=3 * n,
                                        plate_kind=pl["kind"], mean_deps=self._deps(prepared[0]) if pl["kind"] == PLATE_NORM_IID else None, n=n))
            return
        # generic: a bytecode loop, lp += body(i) in order
        p.emit("LOOP_BEGIN", q, 0)
        fix = len(p.code) - 1
        self._abs_words.append(fix)
        body_start = len(p.code)
        self.emit_expr(body)
        p.emit("LOOP_END", 0, body_start)
        self._abs_words.append(len(p.code) - 1)
        p.code[fix] = len(p.code)
        if self._record_terms:
            self._terms.append(dict(start=start, end=len(p.code), kind="inorder", deps=set(), cost=12 * n * max(1, len(p.code) - body_start),
                                    plate_kind=PLATE_GENERIC))
        p.summary.append(f"plate GENERIC n={n} body={body.op}")

    def _grouped(self, mean: Sym, n: int):
        """mu[g_i] with points sorted by group and groups covering a contiguous component range."""
        col, off, stride, base, _pid = mean.val
        if stride != 1: return None
        g = self.t.columns[col][off: off + n]
        gi = g.astype(np.int64)
        if np.any(gi != g) or np.any(np.diff(gi) < 0): return None
        lo, hi = int(gi[0]), int(gi[-1])
        J = hi - lo + 1
        start = np.searchsorted(gi, np.arange(lo, hi + 2), side="left").astype(np.float64)
        return base + lo, J, self.t.add_column(start)

    def _loglinear(self, eta: Sym):
        """eta = sum_k X[i][k] * beta[k] (k ascending, optional leading 0), X row-major with row stride K."""
        terms = _spine_terms(eta)
        xcol = None
        base = None
        for k, tm in enumerate(terms):
            if tm.op != "MUL": return None
            a, b = tm.args
            if a.op == "COMP" and b.op == "DATA_I": a, b = b, a
            if not (a.op == "DATA_I" and b.op == "COMP"): return None
            c, off, stride, _pid = a.val
            if xcol is None: xcol, base = c, b.val
            if c != xcol or off != k or stride != len(terms) or b.val != base + k: return None
        if xcol is None or len(terms) not in POIS_LOGLIN_K: return None      # the device keeps the coefficients in registers: one kernel instance per K
        return xcol, len(terms), base

    # -- main -------------------------------------------------------------------------------------
    def add_logpost(self, result: Sym, derived: Dict[str, Sym]) -> Tuple[int, int]:
        """Emit one log_post program (and its derived-quantity program); returns their word offsets (derived: -1 if none)."""
        p = self.prog
        lp_off = len(p.code)
        terms = _spine_terms(result)
        i = 0
        n_terms = len(terms)
        while i < n_terms:
            tm = terms[i]
            pid = _has_plate_ref(tm)
            if pid is not None:                                   # symbolic-index term: a plate as written
                self._emit_plate(tm, self.t.plate_sizes[pid])
                i += 1
                continue
            run = self._find_run(terms, i)
            if run is not None:
                body, length = run
                self._emit_plate(body, length)
                i += length
                continue
            node = self.prepared(tm)
            start = len(p.code)
            tid = len(self._terms) if self._record_terms else None
            self.emit_expr(node, prepare=False, acc=True, store=tid)
            if self._record_terms:
                self._terms.append(dict(start=start, end=len(p.code), kind="value", deps=self._deps(node), cost=10 * (len(p.code) - start)))
            p.summary.append(f"term {tm.op}")
            i += 1
        p.emit("END")
        der_off = -1
        if derived:
            der_off = len(p.code)
            names = list(derived.keys())
            if p.derived_names and p.derived_names != names:
                raise JsThrow("log_post adds different derived quantities for different values of the binary parameters")
            p.derived_names = names
            for d, (name, expr) in enumerate(derived.items()):
                self.emit_expr(lift(expr))
                p.emit("STORE", d)
            p.emit("END")
        return lp_off, der_off

    def finish(self) -> Program:
        """constant sub-expression programs, in creation order (a later one may read an earlier slot)"""
        p = self.prog
        for k, tree in self._fold_trees:
            p.fold_prog.append(len(p.code))
            p.fold_dst.append(k)
            self.emit_expr(tree, prepare=False)
            p.emit("END")
        return p

    def _emit_component_programs(self):
        """Dependency-aware evaluation (amwg.h comp_prog): for every component c a program that recomputes only the terms that
        read c and adds the others from the chain's term cache, each in its original position. Only worth it when it removes
        a good part of the work (hierarchical models); models whose every step touches the big plate keep the full program."""
        p, terms = self.prog, self._terms
        full = sum(tr["cost"] for tr in terms)
        per_comp = self._per_component_cost()
        abs_words = sorted(self._abs_words)
        p.n_terms = len(terms)
        for c in range(self.n_comp):
            p.comp_prog.append(len(p.code))
            p.touch_off.append(len(p.touch_terms))
            run_start, run_len = None, 0

            def flush():
                nonlocal run_start, run_len
                if run_len:
                    p.emit("ACC_RANGE", run_start, run_len)
                run_start, run_len = None, 0
            for t, tr in enumerate(terms):
                if tr["kind"] == "value" and c not in tr["deps"]:
                    if run_len and run_start + run_len == t:
                        run_len += 1
                    else:
                        flush()
                        run_start, run_len = t, 1
                    continue
                flush()
                delta = len(p.code) - tr["start"]
                frag = list(p.code[tr["start"]:tr["end"]])
                for pos in abs_words:
                    if tr["start"] <= pos < tr["end"]:
                        frag[pos - tr["start"]] += delta
                p.code.extend(frag)
                if tr["kind"] == "value":
                    p.touch_terms.append(t)
            flush()
            p.emit("END")
        p.touch_off.append(len(p.touch_terms))
        p.summary.append(f"dependency-aware evaluation: {len(terms)} terms, cost {sum(per_comp) / (full * self.n_comp):.2f} of the full program")
        # block steps: multi-dim parameters whose components never share a term (amwg.h block_params)
        if all(tr["kind"] == "value" for tr in terms):
            for pidx, (off, n, ptype) in enumerate(self.param_ranges):
                if n <= 1 or ptype == "binary" or len(p.block_params) >= 4:
                    continue
                comps = set(range(off, off + n))
                row = []
                for tr in terms:
                    hit = tr["deps"] & comps
                    if len(hit) > 1:
                        row = None
                        break
                    row.append(next(iter(hit)) if hit else -1)
                if row is not None:
                    p.block_params.append(pidx)
                    p.term_block_comp.extend(row)
                    p.summary.append(f"block steps for parameter #{pidx}: {n} components with one evaluation")

    def _per_component_cost(self) -> List[int]:
        terms = self._terms
        return [sum(tr["cost"] for tr in terms if tr["kind"] == "inorder" or c in tr["deps"]) +
                3 * sum(1 for tr in terms if tr["kind"] == "value" and c not in tr["deps"]) + 40 for c in range(self.n_comp)]

    def _cache_worthwhile(self) -> bool:
        terms = self._terms
        if not any(tr["kind"] == "value" for tr in terms) or len(terms) > MAX_IMMEDIATE:
            return False
        full = sum(tr["cost"] for tr in terms)
        return sum(self._per_component_cost()) <= 0.6 * full * self.n_comp

    def _strip_stores(self, der_off: int) -> int:
        """The model keeps the full program for every step: remove the term-cache stores again (flag + term-id word), so that the
        hot program is exactly what it was without the feature. Returns the moved offset of the derived program."""
        p = self.prog
        removed = sorted(idw for _, idw in p.store_sites)
        for flagged, _ in p.store_sites:
            p.code[flagged] &= ~STORE_FLAG

        def shift(off: int) -> int:
            import bisect
            return off - bisect.bisect_left(removed, off)
        for pos in self._abs_words:
            p.code[pos] = shift(p.code[pos])
        self._abs_words = [shift(pos) for pos in self._abs_words]
        for idw in reversed(removed):
            del p.code[idw]
        p.store_sites = []
        return shift(der_off) if der_off >= 0 else der_off

    def _stat_mode_applies(self) -> bool:
        """amwg.h stat_prog: every O(N) piece of log_post is a NORM_IID plate whose mean reads exactly one component; no binary
        parameter; enough plate points for one data pass per sweep (instead of one per step) to matter."""
        terms = self._terms
        plates = [tr for tr in terms if "plate_kind" in tr]
        mode = os.environ.get("AMWG_STAT_LOWERING", "1")              # 0: never (A/B runs, tests); otherwise whenever eligible
        if mode == "0":
            return False
        # Round 1 kept two-component models on the full program (the interpreter's O(1) steps cost what the saved data pass gained:
        # 2.4e9 vs 2.5e9 draws/s on the headline model). The sweep is now specialised per model at run time (csrc/amwg_jit.cuh),
        # which removes that bookkeeping, so every eligible model is lowered this way.
        if not plates or any(ptype == "binary" for _, _, ptype in self.param_ranges) or not self.param_ranges:
            return False
        if any(tr["plate_kind"] != PLATE_NORM_IID or len(tr["mean_deps"]) != 1 for tr in plates):
            return False
        if any(tr["kind"] != "value" for tr in terms) or len(terms) + len(plates) > MAX_IMMEDIATE:
            return False
        return sum(tr["n"] for tr in plates) >= MIN_STAT_POINTS

    def _emit_stat_programs(self):
        """comp_prog[c] without O(N) work + stat_prog (amwg.h stat_prog). Called after the stat-mode pass over log_post."""
        p, terms = self.prog, self._terms
        n_sum = len(terms)
        stats = [tr["stat"] for tr in terms if tr.get("stat") is not None]
        for st in stats:                                             # statistics live behind the terms of the sum
            st["slot"] = n_sum + st["k"]
            p.code[st["slot_word"]] = st["slot"]
        p.n_sum_terms, p.n_terms = n_sum, n_sum + len(stats)
        for c in range(self.n_comp):
            p.comp_prog.append(len(p.code))
            p.touch_off.append(len(p.touch_terms))
            run_start, run_len = None, 0
            for t, tr in enumerate(terms):
                if c not in tr["deps"]:
                    if run_len and run_start + run_len == t:
                        run_len += 1
                    else:
                        if run_len:
                            p.emit("ACC_RANGE", run_start, run_len)
                        run_start, run_len = t, 1
                    continue
                if run_len:
                    p.emit("ACC_RANGE", run_start, run_len)
                run_start, run_len = None, 0
                st = tr.get("stat")
                if st is None:
                    p.code.extend(p.code[tr["start"]:tr["end"]])
                else:                                                # the plate's S: pre-evaluated at the proposal, or the committed one
                    moved_mean = c in st["mean_deps"]
                    p.emit("CAND" if moved_mean else "CACHED", st["slot"])
                    p.code.extend(p.code[st["split"]:tr["end"]])
                    if moved_mean:
                        p.touch_terms.append(st["slot"])
                p.touch_terms.append(t)
            if run_len:
                p.emit("ACC_RANGE", run_start, run_len)
            p.emit("END")
        p.touch_off.append(len(p.touch_terms))
        p.stat_prog = len(p.code)
        for tr in terms:
            st = tr.get("stat")
            if st is not None:
                frag = list(p.code[tr["start"]:st["split"]])
                frag[st["ss_word"] - tr["start"]] |= ACC_FLAG            # nothing consumes S here: do not leave it on the stack
                p.code.extend(frag)
        p.emit("END")
        p.summary.append(f"pre-evaluated statistics: {len(stats)} plate(s), {sum(st['n'] for st in stats)} points, one data pass per sweep")

    def lower(self, result: Sym, derived: Dict[str, Sym]) -> Program:
        self._record_terms = True
        p = self.prog
        mark = (len(p.code), len(p.plates), len(p.summary), len(p.store_sites), len(self._abs_words))
        lp_off, der_off = self.add_logpost(result, derived)
        if not self.faithful and self._stat_mode_applies():
            # lower log_post again with the plates split into statistic + combination (same plates, same fold slots and constants)
            del p.code[mark[0]:], p.plates[mark[1]:], p.summary[mark[2]:], p.store_sites[mark[3]:], self._abs_words[mark[4]:]
            self._terms = []
            self._stat_mode = True
            lp_off, der_off = self.add_logpost(result, derived)
            self._stat_mode = False
            self._record_terms = False
            self._emit_stat_programs()
            p.logpost_prog, p.derived_prog = lp_off, der_off
            return self.finish()
        self._record_terms = False
        if self._cache_worthwhile():
            self._emit_component_programs()
        else:
            der_off = self._strip_stores(der_off)
        self.prog.logpost_prog, self.prog.derived_prog = lp_off, der_off
        return self.finish()

    def _find_run(self, terms: List[Sym], i0: int):
        """Longest run starting at i0 of terms equal up to data positions that advance affinely. -> (body, length)."""
        slots0: list = []
        sig0 = _signature(terms[i0], slots0)
        loose = False
        if not slots0:
            return None
        # cheap pre-check with the next term
        if i0 + 1 >= len(terms):
            return None
        s1: list = []
        if _signature(terms[i0 + 1], s1) != sig0:
            slots0 = []
            sig0 = _signature_loose(terms[i0], slots0)
            s1 = []
            if _signature_loose(terms[i0 + 1], s1) != sig0:
                return None
            loose = True
        sigf = _signature_loose if loose else _signature
        seqs = [[s[2]] for s in slots0]
        j = i0 + 1
        while j < len(terms):
            sl: list = []
            if sigf(terms[j], sl) != sig0 or len(sl) != len(slots0):
                break
            if any(a[:2] != b[:2] for a, b in zip(sl, slots0)):
                break
            for k, s in enumerate(sl): seqs[k].append(s[2])
            j += 1
        length = j - i0
        if length < _MIN_PLATE:
            return None
        # every data slot must advance affinely; component slots may be arbitrary (-> synthesized index column)
        plan = []
        for (kind, col, first), seq in zip(slots0, seqs):
            arr = np.asarray(seq, dtype=np.int64)
            if kind == "D":
                stride = int(arr[1] - arr[0])
                if np.any(np.diff(arr) != stride):
                    # truncate the run at the first break
                    brk = int(np.argmax(np.diff(arr) != stride)) + 1
                    length = min(length, brk)
                plan.append(("D", col, int(arr[0]), stride))
            else:
                plan.append(("C", arr))
        if length < _MIN_PLATE:
            return None
        pid = self.t._n_plate_idx
        self.t._n_plate_idx += 1
        self.t.plate_sizes[pid] = length
        final_plan = []
        for item in plan:
            if item[0] == "D":
                final_plan.append(("DATA_I", (item[1], item[2], item[3], pid)))
            else:
                arr = item[1][:length]
                if np.all(arr == arr[0]):
                    final_plan.append(("COMP", int(arr[0])))
                else:
                    base = int(arr.min())
                    col = self.t.add_column((arr - base).astype(np.float64))
                    final_plan.append(("COMP_I", (col, 0, 1, base, pid)))
        it = iter(final_plan)
        body = self._rebuild(terms[i0], it, loose)
        return body, length

    def _rebuild(self, node: Sym, it, loose: bool) -> Sym:
        if node.op == "DATA":
            op, val = next(it)
            return Sym(op, (), val)
        if node.op == "COMP" and loose:
            op, val = next(it)
            return Sym(op, (), val)
        if not node.args:
            return node
        return Sym(node.op, tuple(self._rebuild(a, it, loose) for a in node.args), node.val)


def _lfactorial_host(y: float) -> float:
    """lfactorial(y) = Lanczos lgamma(y+1), distributions.js:63-82. Only used to PRECOMPUTE a data column for
    the Poisson plate (constant in the parameters). Plain fp64 ops in the JS order; math.log is within 1 ulp of
    the device log, which moves the constant offset of log_post by < 1e-15 relative (it cancels in every accept ratio)."""
    if y < 0: return float("nan")
    x = y + 1.0
    cof = [76.18009172947146, -86.50532032941677, 24.01409824083091, -1.231739572450155, 0.1208650973866179e-2, -0.5395239384953e-5]
    ser = 1.000000000190015
    xx = yy = x
    tmp = x + 5.5
    tmp -= (xx + 0.5) * math.log(tmp)
    for c in cof:
        yy += 1.0
        ser += c / yy
    return math.log(2.5066282746310005 * ser / xx) - tmp


def _lfactorial_host_vec(y: np.ndarray) -> np.ndarray:
    """_lfactorial_host over an array (the data column of a Poisson plate has up to millions of entries)."""
    y = np.asarray(y, dtype=np.float64)
    x = y + 1.0
    cof = [76.18009172947146, -86.50532032941677, 24.01409824083091, -1.231739572450155, 0.1208650973866179e-2, -0.5395239384953e-5]
    ser = np.full_like(x, 1.000000000190015)
    yy = x.copy()
    tmp = x + 5.5
    with np.errstate(invalid="ignore", divide="ignore"):
        tmp = tmp - (x + 0.5) * np.log(tmp)
        for c in cof:
            yy = yy + 1.0
            ser = ser + c / yy
        out = np.log(2.5066282746310005 * ser / x) - tmp
    return np.where(y < 0, np.nan, out)


POIS_LOGLIN_K = (1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 16)
MAX_VARIANT_COMPS = 4


def _run_closure(tr: Tracer, log_post, params, offsets, wrapped):
    state = tr.make_state(params, offsets)
    _ACTIVE.append(tr)
    try:
        result = log_post(state, wrapped)
    finally:
        _ACTIVE.pop()
    if result is None:
        raise JsThrow("log_post returned undefined")
    result = lift(result)
    derived = {k: v for k, v in state.items() if k not in params}
    for k, v in derived.items():
        if not isinstance(v, (Sym, numbers.Real)):
            raise JsThrow(f"derived quantity {k} must be a number")
    return result, derived


def trace(log_post, params: Dict[str, dict], offsets: Dict[str, int], n_comp: int, data, faithful: bool = False) -> Tuple[Program, List[str]]:
    """Run `log_post` symbolically and return the lowered program and the derived-quantity names.

    If the closure needs concrete values (Python `if` on a parameter) and the model has at most MAX_VARIANT_COMPS binary
    components, it is recorded once per configuration of those components instead (the device picks the program that matches the
    evaluated state, amwg.h variant_*): `if (m === 0) ... else ...` of tests/test_data.js:163-168 can be written as is."""
    tr = Tracer()
    wrapped = tr.wrap_data(data)
    ranges = [(offsets[name], int(np.prod(p["dim"])), p["type"]) for name, p in params.items()]
    low = Lowering(tr, n_comp, faithful, ranges)
    try:
        result, derived = _run_closure(tr, log_post, params, offsets, wrapped)
    except NeedsConcrete as exc:
        comps = [offsets[name] + c for name, p in params.items() if p["type"] == "binary" for c in range(int(np.prod(p["dim"])))]
        if not comps or len(comps) > MAX_VARIANT_COMPS:
            raise JsThrow(exc.message)
        prog = low.prog
        prog.variant_comps = comps
        for v in range(1 << len(comps)):
            tr.concrete = {c: float((v >> k) & 1) for k, c in enumerate(comps)}
            try:
                result, derived = _run_closure(tr, log_post, params, offsets, wrapped)
            except NeedsConcrete as exc2:
                raise JsThrow(exc2.message)                  # branches on a real / int parameter: cannot be recorded
            lp_off, der_off = low.add_logpost(result, derived)
            prog.variant_logpost.append(lp_off)
            prog.variant_derived.append(der_off)
        tr.concrete = {}
        prog.logpost_prog, prog.derived_prog = prog.variant_logpost[0], prog.variant_derived[0]
        low.finish()
        return prog, list(prog.derived_names)
    prog = low.lower(result, derived)
    return prog, list(derived.keys())


class LogLik:
    """A traced pointwise log-likelihood (sample_summary(..., loo=...)): the recorded expression of ``log_lik(state, data, i)``
    at a symbolic point index i of `points` points, and the parameters it reads (in the parameters' order)."""

    def __init__(self, tracer: Tracer, expr: Sym, reads: List[str], ranges: List[Tuple[str, int, int]]):
        self.tracer, self.expr, self.reads, self._ranges = tracer, expr, reads, ranges

    def lower(self, entry_start: Dict[str, int]) -> Program:
        """The body as an expression program addressing the sample block's ENTRIES: component c of parameter `name` (first
        component `off`) becomes entry entry_start[name] + c - off, for COMP and for the base of COMP_I alike (a parameter's
        entries are contiguous in the block). The body is at word 0 and leaves its value on the stack; its constant
        sub-expressions become fold programs (evaluated on the device, amwg_loo_pointwise) with their own constant bank."""
        prog, _ = self.lower_exprs([self.expr], entry_start)
        return prog

    def lower_exprs(self, exprs: Sequence[Sym], entry_start: Dict[str, int]) -> Tuple[Program, List[int]]:
        """Sub-expressions of the body (the parameters of its ld.* call, amwg_ppc_pointwise) lowered as `lower` lowers the body:
        one END-terminated program each, in order, sharing one constant bank and one set of fold programs. -> (program, the
        programs' offsets)."""
        def entry(c: int) -> int:
            for name, off, n in self._ranges:
                if off <= c < off + n:
                    return entry_start[name] + c - off
            raise JsThrow("log_lik reads component %d, which belongs to no parameter" % c)
        memo: Dict[int, Sym] = {}

        def remap(n: Sym) -> Sym:
            got = memo.get(id(n))
            if got is not None:
                return got
            if n.op == "COMP":
                out = Sym("COMP", (), entry(n.val))
            elif n.op == "COMP_I":
                col, off, stride, base, pid = n.val
                out = Sym("COMP_I", (), (col, off, stride, entry(base), pid))
            elif n.args:
                out = Sym(n.op, tuple(remap(a) for a in n.args), n.val)
            else:
                out = n
            memo[id(n)] = out
            return out
        low = Lowering(self.tracer, 0)
        offs = []
        for e in exprs:
            offs.append(len(low.prog.code))
            low.emit_expr(remap(e))
            low.prog.emit("END")
        low.prog.logpost_prog = 0
        return low.finish(), offs

    def observed_call(self, points: int):
        """The body as a posterior predictive check reads it (sample_summary(..., ppc=...)): one ld.* call whose first argument
        is a data value at the point index. -> (ld name, the observed values y_0 .. y_{points-1}, the call's other arguments).
        Raises ValueError for anything else: an expression around the call, or a first argument that is not data[i]."""
        e = self.expr
        if not e.op.startswith("LD_"):
            raise ValueError("ppc: log_lik must return one ld.* call (e.g. ld.norm(data.y[i], mu, sigma)), not %r" % (e,))
        family = e.op[3:].lower()
        obs = e.args[0]
        if obs.op != "DATA_I":
            raise ValueError("ppc: the first argument of ld.%s must be a data value at the point index (data.y[i]), not %r" % (family, obs))
        col, off, stride, _pid = obs.val
        column = np.asarray(self.tracer.columns[col], dtype=np.float64)
        y = column[off: off + stride * (points - 1) + 1: stride].copy()
        return family, y, list(e.args[1:])


def trace_log_lik(log_lik, params: Dict[str, dict], offsets: Dict[str, int], data, points: int, what: str = "loo") -> LogLik:
    """Run ``log_lik(state, data, i)`` once with symbolic parameters, proxied data and a symbolic point index i over `points`
    points (``data.y[i]`` -> DATA_I, ``mu[data.g[i]]`` -> COMP_I, as under mcmc.points), with the ld.* / Math rules of log_post.
    Raises ValueError when the closure cannot be traced for the device: it branches on a parameter, reads a data array past its
    end at some i < points, indexes a parameter with data values outside it, or returns something that is not a number. `what`
    names the argument in the message ("loo", "ppc")."""
    tr = Tracer()
    wrapped = tr.wrap_data(data)
    i = tr.new_plate_index(points)
    state = tr.make_state(params, offsets)
    _ACTIVE.append(tr)
    try:
        result = log_lik(state, wrapped, i)
        if result is None:
            raise JsThrow("log_lik returned undefined")
        expr = lift(result)
    except JsThrow as exc:
        raise ValueError(what + ": log_lik cannot be evaluated on the device: " + exc.message) from None
    finally:
        _ACTIVE.pop()
    ranges = [(name, offsets[name], int(np.prod(p["dim"]))) for name, p in params.items()]
    comps, stack, seen = set(), [expr], set()
    while stack:
        n = stack.pop()
        if id(n) in seen:
            continue
        seen.add(id(n))
        if n.op == "COMP":
            comps.add(n.val)
        elif n.op == "COMP_I":
            comps.add(n.val[3])
        stack.extend(n.args)
    reads = [name for name, off, n in ranges if any(off <= c < off + n for c in comps)]
    return LogLik(tr, expr, reads, ranges)


_ACTIVE: List[Tracer] = []


def points(n):
    """``for i in mcmc.points(n):`` -- a loop over n data points recorded once (see PlateIndex)."""
    if not _ACTIVE:
        return range(int(n))
    return _ACTIVE[-1].points(n)
