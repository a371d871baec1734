"""ctypes front-end of oracle/liboracle.so -- TEST INFRASTRUCTURE ONLY (see amwg_oracle.c header).

Nothing under bayes.js_b200/ imports this module. It shares no code with the product: parameter completion and
option defaults are restated here from /root/reference/mcmc.js (:313-403, :500-505), the sampler itself is the C
restatement in amwg_oracle.c.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
from typing import Callable, Dict, List, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None

LOGPOST_FN = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.c_void_p, C.c_void_p)


class OrcParam(C.Structure):
    _fields_ = [("type", C.c_int32), ("n_comp", C.c_int32), ("dim0", C.c_int32), ("comp_offset", C.c_int32),
                ("lower", C.c_double), ("upper", C.c_double)]


class OrcCompOptions(C.Structure):
    _fields_ = [("prop_log_scale", C.c_double), ("batch_size", C.c_double), ("max_adaptation", C.c_double),
                ("initial_adaptation", C.c_double), ("target_accept_rate", C.c_double), ("is_adapting", C.c_int32),
                ("_pad", C.c_int32)]


class OrcVec(C.Structure):
    _fields_ = [("x", C.POINTER(C.c_double)), ("n", C.c_int64)]


class OrcHier(C.Structure):
    _fields_ = [("y", C.POINTER(C.c_double)), ("g", C.POINTER(C.c_int32)), ("n", C.c_int64), ("J", C.c_int32)]


class OrcPoisReg(C.Structure):
    _fields_ = [("y", C.POINTER(C.c_double)), ("X", C.POINTER(C.c_double)), ("n", C.c_int64), ("K", C.c_int32)]


class OrcBinomData(C.Structure):
    _fields_ = [("x", C.POINTER(C.c_double)), ("n", C.POINTER(C.c_double)), ("len", C.c_int64)]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    src = os.path.join(_HERE, "amwg_oracle.c")
    if not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE], check=True, capture_output=True)
    L = C.CDLL(_LIB_PATH)
    d, u64, i64, vp = C.c_double, C.c_uint64, C.c_int64, C.c_void_p
    for name, n in (("orc_log", 1), ("orc_exp", 1), ("orc_js_round", 1), ("orc_ld_lgamma", 1), ("orc_ld_lfactorial", 1),
                    ("orc_ld_lchoose", 2), ("orc_ld_lbeta", 2), ("orc_ld_beta", 3), ("orc_ld_cauchy", 3), ("orc_ld_norm", 3),
                    ("orc_ld_laplace", 3), ("orc_ld_gamma", 3), ("orc_ld_invgamma", 3), ("orc_ld_lnorm", 3),
                    ("orc_ld_pareto", 3), ("orc_ld_t", 4), ("orc_ld_weibull", 3), ("orc_ld_logis", 3), ("orc_ld_exp", 2),
                    ("orc_ld_unif", 3), ("orc_ld_bern", 2), ("orc_ld_binom", 3), ("orc_ld_nbinom", 3), ("orc_ld_hyper", 4),
                    ("orc_ld_pois", 2)):
        f = getattr(L, name); f.restype = d; f.argtypes = [d] * n
    L.orc_ld_bivarnorm.restype = d; L.orc_ld_bivarnorm.argtypes = [vp, vp, vp, d]
    L.orc_ld_dirichlet.restype = d; L.orc_ld_dirichlet.argtypes = [vp, vp, C.c_int]
    L.orc_ld_cat.restype = d; L.orc_ld_cat.argtypes = [d, vp, C.c_int]
    L.orc_param_init_fixed.restype = d; L.orc_param_init_fixed.argtypes = [C.c_int, d, d]
    L.orc_philox4x32_10.restype = None; L.orc_philox4x32_10.argtypes = [vp, vp, vp]
    L.orc_stream_uniform.restype = d; L.orc_stream_uniform.argtypes = [u64, u64, u64]
    L.orc_runif.restype = d; L.orc_runif.argtypes = [u64, u64, C.POINTER(u64), d, d]
    L.orc_runif_discrete.restype = d; L.orc_runif_discrete.argtypes = [u64, u64, C.POINTER(u64), d, d]
    L.orc_rnorm.restype = d; L.orc_rnorm.argtypes = [u64, u64, C.POINTER(u64), d, d]
    L.orc_shuffle.restype = None; L.orc_shuffle.argtypes = [u64, u64, C.POINTER(u64), vp, C.c_int]
    L.orc_create.restype = vp
    L.orc_create.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, u64, u64]
    L.orc_destroy.restype = None; L.orc_destroy.argtypes = [vp]
    L.orc_step.restype = None; L.orc_step.argtypes = [vp]
    L.orc_burn.restype = None; L.orc_burn.argtypes = [vp, i64]
    L.orc_sample.restype = i64; L.orc_sample.argtypes = [vp, i64, vp, C.c_int, vp]
    L.orc_thin.restype = None; L.orc_thin.argtypes = [vp, i64]
    L.orc_set_adapting.restype = None; L.orc_set_adapting.argtypes = [vp, C.c_int]
    L.orc_info.restype = None; L.orc_info.argtypes = [vp, vp]
    L.orc_state.restype = C.POINTER(d); L.orc_state.argtypes = [vp]
    L.orc_rng_position.restype = u64; L.orc_rng_position.argtypes = [vp]
    L.orc_logpost_calls.restype = i64; L.orc_logpost_calls.argtypes = [vp]
    L.orc_set_replay.restype = None; L.orc_set_replay.argtypes = [vp, vp, u64]
    L.orc_substepper_order.restype = None; L.orc_substepper_order.argtypes = [vp, vp]
    L.orc_run_chains.restype = None
    L.orc_run_chains.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, vp, u64, u64, i64, i64, i64, i64, vp, C.c_int, vp, vp]
    L.orc_run_chains_mt.restype = C.c_int
    L.orc_run_chains_mt.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, vp, u64, u64, i64, i64, i64, i64, vp, C.c_int, vp, vp, C.c_int]
    L.orc_trace.restype = i64; L.orc_trace.argtypes = [vp, vp, i64]
    L.orc_trace_len.restype = i64; L.orc_trace_len.argtypes = [vp]
    _lib = L
    return L


# ---- parameter completion restated from mcmc.js:313-403 (independent of bayes.js_b200/mcmc.py) -----------------
_TYPES = {"real": 0, "int": 1, "binary": 2}
INF = float("inf")


def js_round(x):
    r = math.ceil(x)
    return float(r - 1.0 if r - 0.5 > x else r)


def param_init_fixed(ptype: str, lower: float, upper: float) -> float:
    v = lib().orc_param_init_fixed(_TYPES.get(ptype, -1), float(lower), float(upper))
    if v != v:
        raise ValueError("param_init_fixed throws")
    return v


def complete_params(params: Dict[str, dict]) -> Dict[str, dict]:
    out = {}
    for name, p in params.items():
        q = dict(p)
        q.setdefault("type", "real")
        dim = q.get("dim", [1])
        q["dim"] = [dim] if isinstance(dim, (int, float)) else list(dim)
        if q["type"] == "binary":
            q["upper"], q["lower"] = 1, 0
        q.setdefault("upper", INF)
        q.setdefault("lower", -INF)
        n = int(np.prod(q["dim"]))
        if "init" in q:
            init = q["init"]
            if q["dim"] == [1] and callable(init):
                init = init()
            if q["dim"] != [1] and not isinstance(init, (list, tuple, np.ndarray)):
                init = [init() if callable(init) else init for _ in range(n)]
        else:
            v = param_init_fixed(q["type"], q["lower"], q["upper"])
            init = v if q["dim"] == [1] else [v] * n
        q["init_flat"] = [float(v) for v in np.asarray(init, dtype=float).reshape(-1)]
        out[name] = q
    return out


DEFAULT_OPTIONS = dict(prop_log_scale=0.0, batch_size=50.0, max_adaptation=0.33, initial_adaptation=1.0,
                       target_accept_rate=0.44, is_adapting=True)         # mcmc.js:500-505


def _layout(params: Dict[str, dict], comp_options: Optional[Dict[str, dict]]):
    cp = complete_params(params)
    P = len(cp)
    prm = (OrcParam * P)()
    init: List[float] = []
    opts_list = []
    off = 0
    for k, (name, q) in enumerate(cp.items()):
        n = int(np.prod(q["dim"]))
        prm[k] = OrcParam(_TYPES[q["type"]], n, int(q["dim"][0]), off, float(q["lower"]), float(q["upper"]))
        init.extend(q["init_flat"])
        o = dict(DEFAULT_OPTIONS)
        o.update((comp_options or {}).get(name, {}))
        for c in range(n):
            oc = {key: (val[c] if isinstance(val, (list, tuple, np.ndarray)) else val) for key, val in o.items()}
            opts_list.append(oc)
        off += n
    opts = (OrcCompOptions * off)()
    for c, oc in enumerate(opts_list):
        opts[c] = OrcCompOptions(float(oc["prop_log_scale"]), float(oc["batch_size"]), float(oc["max_adaptation"]),
                                 float(oc["initial_adaptation"]), float(oc["target_accept_rate"]), 1 if oc["is_adapting"] else 0, 0)
    return cp, prm, np.asarray(init, dtype=np.float64), opts, off


# ---- built-in models (amwg_oracle.c "Models") ------------------------------------------------------------------------
def _vec(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, OrcVec(a.ctypes.data_as(C.POINTER(C.c_double)), a.size)


def _model(name: str, data):
    """-> (C function pointer, data struct, keepalive, derived names)"""
    L = lib()
    fn = getattr(L, "orc_model_" + name)
    keep = []
    derived: List[str] = []
    if name in ("norm_readme", "norm_test", "beta_bern", "spike_bern", "complex"):
        a, v = _vec(data["x"] if isinstance(data, dict) else data)
        keep += [a]
        st = v
        if name == "norm_test":
            derived = ["var"]
    elif name == "hier_norm":
        y = np.ascontiguousarray(data["y"], dtype=np.float64)
        g = np.ascontiguousarray(data["g"], dtype=np.int32)
        keep += [y, g]
        st = OrcHier(y.ctypes.data_as(C.POINTER(C.c_double)), g.ctypes.data_as(C.POINTER(C.c_int32)), y.size, int(g.max()) + 1)
    elif name == "pois_reg":
        y = np.ascontiguousarray(data["y"], dtype=np.float64)
        X = np.ascontiguousarray(data["X"], dtype=np.float64)
        keep += [y, X]
        st = OrcPoisReg(y.ctypes.data_as(C.POINTER(C.c_double)), X.ctypes.data_as(C.POINTER(C.c_double)), y.size, X.shape[1])
    elif name == "hier_binom":
        x = np.ascontiguousarray(data["x"], dtype=np.float64)
        n = np.ascontiguousarray(data["n"], dtype=np.float64)
        keep += [x, n]
        st = OrcBinomData(x.ctypes.data_as(C.POINTER(C.c_double)), n.ctypes.data_as(C.POINTER(C.c_double)), x.size)
    else:
        st = None
    return fn, st, keep, derived


class OracleSampler:
    """One chain of the reference sampler (mcmc.AmwgSampler) with Math.random() := Philox stream (seed, chain)."""

    def __init__(self, model, data, params: Dict[str, dict], seed: int = 0, chain: int = 0,
                 comp_options: Optional[Dict[str, dict]] = None, thin: int = 1, n_derived: int = 0,
                 derived_names: Optional[List[str]] = None):
        L = lib()
        self.params, prm, init, opts, D = _layout(params, comp_options)
        self.D = D
        if callable(model) and not isinstance(model, str):
            # arbitrary Python closure f(state_array) -> float; state_array has D + n_derived slots
            self._n_derived = n_derived
            self.derived_names = list(derived_names or [])

            def cb(state_ptr, _d, _u, f=model, n=D + n_derived):
                arr = np.ctypeslib.as_array(state_ptr, shape=(n,))
                return float(f(arr))
            self._cb = LOGPOST_FN(cb)
            fn, dptr, self._keep = self._cb, None, []
        else:
            cfn, st, keep, self.derived_names = _model(model, data)
            self._n_derived = len(self.derived_names)
            self._keep = keep + [st]
            fn = C.cast(cfn, C.c_void_p)
            dptr = C.cast(C.pointer(st), C.c_void_p) if st is not None else None
        self._prm, self._init, self._opts = prm, init, opts
        self.h = L.orc_create(len(self.params), C.cast(prm, C.c_void_p), init.ctypes.data, C.cast(opts, C.c_void_p),
                              self._n_derived, fn, dptr, None, seed, chain)
        L.orc_thin(self.h, thin)
        self.thin = thin

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_destroy(self.h)
            self.h = None

    def names(self) -> List[str]:
        return list(self.params.keys()) + list(self.derived_names)

    def entries(self, name: str) -> List[int]:
        off = 0
        for nm, q in self.params.items():
            n = int(np.prod(q["dim"]))
            if nm == name:
                return list(range(off, off + n))
            off += n
        return [self.D + self.derived_names.index(name)]

    def burn(self, n: int):
        lib().orc_burn(self.h, n)

    def set_thin(self, k: int):
        lib().orc_thin(self.h, k)
        self.thin = k

    def step(self):
        lib().orc_step(self.h)

    def state(self) -> np.ndarray:
        return np.ctypeslib.as_array(lib().orc_state(self.h), shape=(self.D + self._n_derived,)).copy()

    def sample(self, n: int, monitor: Optional[List[str]] = None) -> Dict[str, np.ndarray]:
        names = self.names() if monitor is None else monitor
        ent: List[int] = []
        spans = {}
        for nm in names:
            e = self.entries(nm)
            spans[nm] = (len(ent), len(e))
            ent.extend(e)
        mon = np.asarray(ent, dtype=np.int32)
        rows = (n + self.thin - 1) // self.thin if n > 0 else 0
        out = np.empty((max(rows, 1), len(ent)))
        got = lib().orc_sample(self.h, n, mon.ctypes.data, len(ent), out.ctypes.data)
        assert got == rows
        out = out[:rows]
        res = {}
        for nm in names:
            s, ln = spans[nm]
            dim = self.params[nm]["dim"] if nm in self.params else [1]
            a = out[:, s:s + ln]
            res[nm] = a[:, 0] if list(dim) == [1] else a.reshape(rows, *dim)
        return res

    def set_adapting(self, flag: bool):
        lib().orc_set_adapting(self.h, 1 if flag else 0)

    def info(self) -> np.ndarray:
        out = np.empty((self.D, 5))
        lib().orc_info(self.h, out.ctypes.data)
        return out

    def rng_position(self) -> int:
        return int(lib().orc_rng_position(self.h))

    def logpost_calls(self) -> int:
        return int(lib().orc_logpost_calls(self.h))

    TRACE_FIELDS = ("comp", "current", "proposal", "u", "curr_log_dens", "prop_log_dens")

    def trace(self, cap: int):
        """Record every Metropolis step from now on (orc_trace), up to `cap` steps: one row per step of TRACE_FIELDS -- the
        component, its current value, the proposal, the accept uniform (-1: the proposal is out of bounds, no uniform drawn) and
        log_post at the current state and at the proposal (NaN when not evaluated)."""
        self._trace = np.full((int(cap), 6), np.nan)
        lib().orc_trace(self.h, self._trace.ctypes.data, int(cap))

    def trace_rows(self) -> np.ndarray:
        """the rows recorded since trace(); fails if more steps were taken than it has room for"""
        n = int(lib().orc_trace_len(self.h))
        assert n <= self._trace.shape[0], f"{n} steps traced, room for {self._trace.shape[0]}"
        return self._trace[:n].copy()

    def substepper_order(self) -> List[int]:
        out = np.empty(len(self.params), dtype=np.int32)
        lib().orc_substepper_order(self.h, out.ctypes.data)
        return out.tolist()


def run_model(model: str, data, params: Dict[str, dict], chains: int = 1, seed: int = 0, burn: int = 0, sample: int = 0,
              thin: int = 1, first_chain: int = 0, comp_options: Optional[Dict[str, dict]] = None,
              monitor: Optional[List[str]] = None, threads: int = 1, final_state: bool = False):
    """`chains` independent oracle chains of a built-in model; output shaped like mcmc.AmwgSampler.sample():
    [rows, *dim] for one chain, [rows, chains, *dim] otherwise. With final_state, returns (that, [chains, D + n_derived] the state
    each chain ends in)."""
    L = lib()
    cp, prm, init, opts, D = _layout(params, comp_options)
    cfn, st, keep, derived = _model(model, data)
    names = (list(cp.keys()) + derived) if monitor is None else monitor
    ent: List[int] = []
    spans = {}
    for nm in names:
        if nm in cp:
            off = 0
            for k, q in cp.items():
                n = int(np.prod(q["dim"]))
                if k == nm:
                    e = list(range(off, off + n))
                off += n
        else:
            e = [D + derived.index(nm)]
        spans[nm] = (len(ent), len(e))
        ent.extend(e)
    mon = np.asarray(ent, dtype=np.int32)
    rows = (sample + thin - 1) // thin if sample > 0 else 0
    out = np.empty((chains, max(rows, 1), len(ent)))
    final = np.empty((chains, D + len(derived))) if final_state else None
    args = (len(cp), C.cast(prm, C.c_void_p), init.ctypes.data, C.cast(opts, C.c_void_p), len(derived),
            C.cast(cfn, C.c_void_p), C.cast(C.pointer(st), C.c_void_p) if st is not None else None,
            seed, first_chain, chains, burn, sample, thin, mon.ctypes.data, len(ent), out.ctypes.data,
            final.ctypes.data if final is not None else None)
    if threads > 1:
        L.orc_run_chains_mt(*args, int(threads))          # the C call releases the GIL; chains are dealt out to pthreads inside
    else:
        L.orc_run_chains(*args)
    out = out[:, :rows, :]
    res = {}
    for nm in names:
        s, ln = spans[nm]
        dim = cp[nm]["dim"] if nm in cp else [1]
        a = np.moveaxis(out[:, :, s:s + ln], 0, 1)        # [rows, chains, entries]
        a = a.reshape(rows, chains) if list(dim) == [1] else a.reshape(rows, chains, *dim)
        res[nm] = a[:, 0] if chains == 1 else a
    return (res, final) if final_state else res


def time_model(model: str, data, params, chains: int, burn: int, sample: int, seed: int = 0, threads: int = 1) -> float:
    """Wall seconds of `chains` oracle chains on `threads` host threads (bench.py's CPU baseline / reference arm)."""
    import time
    t0 = time.perf_counter()
    run_model(model, data, params, chains=chains, seed=seed, burn=burn, sample=sample, threads=threads)
    return time.perf_counter() - t0
