"""``mcmc`` -- host-side mirror of /root/reference/mcmc.js for the one path this package accelerates:

    sampler = mcmc.AmwgSampler(params, log_post, data, options)     # mcmc.js:1090-1092, 940-966
    sampler.burn(1000); samples = sampler.sample(5000)              # mcmc.js:1035-1039, 1005-1030

Same names, argument meaning and error strings as the reference; the stepping itself happens in
libamwg_b200.so (CUDA, sm_90a) for ``options["chains"]`` independent chains at once.  The host
language is Python because no JavaScript engine exists in this image; INTEGRATION.md shows the N-API
binding a Node host would put under the same `mcmc` / `ld` module names.

New, non-reference options (the many-chain setting needs them): ``chains`` (default 1: output is
shaped exactly like the reference's), ``seed``, ``device``, ``distributed``, ``first_chain`` (global id of
the first chain, default 0), ``faithful`` (no factorised likelihood plates: bit-faithful, slower),
``init_radius`` (over-dispersed starting points drawn on the device, DESIGN.md §2; default: every chain
starts at the params' init), ``superchain_size`` (chains per superchain: with ``init_radius`` the chains of a
superchain start at one point, and ``sample_summary(n, nested=True)`` uses it; DESIGN.md §4.6), ``temperatures`` (parallel
tempering: ladders of K neighbouring chains at temperatures T_0 = 1 < ... < T_{K-1} that swap states after every sweep, so that
multimodal posteriors are sampled; sample() and sample_summary() return the T = 1 chains; DESIGN.md §2). ``sampler.set_state(values)``
places the chains anywhere; ``sampler.checkpoint()`` and ``sampler.restore(images)`` stop and resume a run bit for bit.
"""
from __future__ import annotations

import copy
import ctypes as C
import math
import os
from typing import Any, Dict, List, Optional

import numpy as np

from . import _ffi
from ._ffi import AmwgColumn, AmwgCompOptions, AmwgModel, AmwgParam, AmwgPlate, BINARY, INT, REAL
from .tracer import JsThrow, Math, Sym, points, trace, where  # noqa: F401  (re-exported)

Infinity = float("inf")
_TYPE_CODE = {"real": REAL, "int": INT, "binary": BINARY}


# ------------------------------------------------------------------------------------------------
# helpers -- mcmc.js:131-303
# ------------------------------------------------------------------------------------------------
def is_number(x) -> bool:
    """mcmc.js:131-133"""
    return isinstance(x, (int, float, np.integer, np.floating)) and not isinstance(x, bool)


def create_array(dim, init):
    """mcmc.js:147-168 -- nested list of shape `dim`; `init` is a value or a zero-arg function."""
    dim = list(dim)
    if len(dim) == 1:
        return [init() if callable(init) else init for _ in range(int(dim[0]))]
    if len(dim) > 1:
        return [create_array(dim[1:], init) for _ in range(int(dim[0]))]
    raise JsThrow("create_array can't create a dimensionless array")


def array_dim(a) -> List[int]:
    """mcmc.js:178-184"""
    if len(a) > 0 and isinstance(a[0], (list, tuple, np.ndarray)):
        return [len(a)] + array_dim(a[0])
    return [len(a)]


def array_equal(a1, a2) -> bool:
    """mcmc.js:191-205"""
    if len(a1) != len(a2):
        return False
    for x, y in zip(a1, a2):
        if isinstance(x, (list, tuple)) and isinstance(y, (list, tuple)):
            if not array_equal(x, y):
                return False
        elif x != y:
            return False
    return True


def _flatten(a) -> List[Any]:
    if isinstance(a, (list, tuple, np.ndarray)):
        out: List[Any] = []
        for v in a:
            out.extend(_flatten(v))
        return out
    return [a]


def _js_truthy(v) -> bool:
    """JS truthiness for the `a || b` option merge (mcmc.js:873-878): undefined/null/0/NaN/false/"" are falsy, arrays are truthy."""
    if v is None or v is False:
        return False
    if isinstance(v, str):
        return v != ""
    if is_number(v):
        return not (v == 0 or v != v)
    return True


def _js_join(a) -> str:
    """Array -> string as JS string concatenation does it ("" + [1,[2,3]] === "1,2,3")."""
    return ",".join(_js_join(v) if isinstance(v, (list, tuple)) else _js_num(v) for v in a)


def _js_num(v) -> str:
    if isinstance(v, float):
        if v == Infinity: return "Infinity"
        if v == -Infinity: return "-Infinity"
        if v != v: return "NaN"
        if v == int(v) and abs(v) < 1e21: return str(int(v))
    return str(v)


def get_option(option_name: str, options: Optional[dict], defaul_value):
    """mcmc.js:280-285 -- undefined and null fall back to the default; 0 / false do not."""
    options = options or {}
    v = options.get(option_name) if option_name in options else None
    return v if v is not None else defaul_value


def get_multidim_option(option_name: str, options: Optional[dict], dim, defaul_value):
    """mcmc.js:293-303"""
    value = get_option(option_name, options, defaul_value)
    if not isinstance(value, (list, tuple)):
        value = create_array(dim, value)
    if not array_equal(array_dim(value), list(dim)):
        raise JsThrow("The option " + option_name + " is of dimension [" + _js_join(array_dim(value)) +
                      "] but should be [" + _js_join(list(dim)) + "].")
    return value


def js_round(x: float) -> float:
    """Math.round: halves toward +infinity."""
    r = math.ceil(x)
    if r - 0.5 > x:
        r -= 1.0
    return float(r)


# ------------------------------------------------------------------------------------------------
# parameter handling -- mcmc.js:313-403
# ------------------------------------------------------------------------------------------------
def param_init_fixed(type, lower, upper):
    """mcmc.js:313-341"""
    if lower > upper:
        raise JsThrow("Can not initialize parameter where lower bound > upper bound")
    if type == "real":
        if lower == -Infinity and upper == Infinity: return 0.5
        if lower == -Infinity: return upper - 0.5
        if upper == Infinity: return lower + 0.5
        if lower <= upper: return (lower + upper) / 2
    elif type == "int":
        if lower == -Infinity and upper == Infinity: return 1
        if lower == -Infinity: return upper - 1
        if upper == Infinity: return lower + 1
        if lower <= upper: return js_round((lower + upper) / 2)
    elif type == "binary":
        return 1
    raise JsThrow("Could not initialize parameter of type " + str(type) + "[" + _js_num(lower) + ", " + _js_num(upper) + "]")


def complete_params(params_to_complete: Dict[str, dict], param_init=param_init_fixed) -> Dict[str, dict]:
    """mcmc.js:357-403 -- returns a completed deep copy; the input is not modified."""
    params = copy.deepcopy(params_to_complete)
    for param_name, param in params.items():
        if "type" not in param:
            param["type"] = "real"
        if "dim" not in param:
            param["dim"] = [1]
        if is_number(param["dim"]):
            param["dim"] = [param["dim"]]
        param["dim"] = list(param["dim"])
        if param["type"] == "binary":
            param["upper"] = 1
            param["lower"] = 0
        if "upper" not in param:
            param["upper"] = Infinity
        if "lower" not in param:
            param["lower"] = -Infinity
        if "init" in param:
            if array_equal(param["dim"], [1]) and callable(param["init"]):
                param["init"] = param["init"]()
            elif not array_equal(param["dim"], [1]) and not isinstance(param["init"], (list, tuple, np.ndarray)):
                param["init"] = create_array(param["dim"], param["init"])
        else:
            if array_equal(param["dim"], [1]):
                param["init"] = param_init(param["type"], param["lower"], param["upper"])
            else:
                param["init"] = create_array(
                    param["dim"], lambda p=param: param_init(p["type"], p["lower"], p["upper"]))
    return params


# ------------------------------------------------------------------------------------------------
# exported RNG helpers -- mcmc.js:31-54 (kept for the export list; the sampler does not use them)
# ------------------------------------------------------------------------------------------------
class _HostStream:
    """`Math.random()` for the exported helpers: the Philox stream definition of the sampler, drawn on the device."""
    seed = 0x6d636d63
    chain = 0xFFFFFFFF
    n = 0
    _block = np.empty(0)
    _block0 = 0

    @classmethod
    def random(cls) -> float:
        k = cls.n - cls._block0
        if not (0 <= k < cls._block.size):
            want = cls.n + 1024
            buf = np.empty(want)
            _ffi.check(_ffi.lib().amwg_primitive_eval(2, np.zeros(want).ctypes.data, want, cls.seed, cls.chain,
                                                      buf.ctypes.data, _default_device()))
            cls._block, cls._block0 = buf[cls.n:], cls.n
            k = 0
        cls.n += 1
        return float(cls._block[k])


def set_random_stream(seed: int, chain: int = 0, position: int = 0):
    """Not in the reference (its helpers use the engine's unseedable Math.random): choose the Philox stream (seed, chain) the
    exported helpers runif / runif_discrete / rnorm draw from, and the position in it."""
    _HostStream.seed, _HostStream.chain, _HostStream.n = int(seed) & 0xFFFFFFFFFFFFFFFF, int(chain) & 0xFFFFFFFFFFFFFFFF, int(position)
    _HostStream._block, _HostStream._block0 = np.empty(0), 0


def _device_log(x: float) -> float:
    """Math.log as the device computes it (fdlibm e_log, csrc/amwg_math.cuh): the helpers agree with the sampler bit for bit."""
    a, out = np.array([float(x)]), np.empty(1)
    _ffi.check(_ffi.lib().amwg_primitive_eval(0, a.ctypes.data, 1, 0, 0, out.ctypes.data, _default_device()))
    return float(out[0])


def runif(min, max):
    """mcmc.js:31-33"""
    return _HostStream.random() * (max - min) + min


def runif_discrete(min, max):
    """mcmc.js:36-38"""
    return math.floor(_HostStream.random() * (max - min + 1)) + min


def rnorm(mean, sd):
    """mcmc.js:43-54"""
    while True:
        u = _HostStream.random()
        v = 1.7156 * (_HostStream.random() - 0.5)
        x = u - 0.449871
        y = abs(v) + 0.386595
        q = x * x + y * (0.19600 * y - 0.25472 * x)
        if not (q > 0.27597 and (q > 0.27846 or v * v > -4 * _device_log(u) * u * u)):
            break
    return (v / u) * sd + mean


DISPERSE_ATTEMPTS = 100         # csrc/amwg_init.cuh kDisperseAttempts
MAX_RUNGS = 256                 # csrc/amwg_temper.cuh kMaxRungs


def ladder_betas(temperatures, n_chains: int) -> List[float]:
    """options.temperatures -> [beta_r = 1.0 / T_r], one IEEE division each: the doubles the device and the reference use. Raises
    unless there are 2..256 finite temperatures, T_0 = 1, strictly increasing, whose count K divides options.chains (global chain
    g is rung g mod K of ladder g // K, DESIGN.md §2 "Tempered ladders")."""
    if isinstance(temperatures, (str, bytes, dict)) or not hasattr(temperatures, "__len__"):
        raise JsThrow("options.temperatures must be a list of numbers")
    temps = list(np.asarray(temperatures, dtype=object).reshape(-1)) if isinstance(temperatures, np.ndarray) else list(temperatures)
    if not all(is_number(t) for t in temps):
        raise JsThrow("options.temperatures must be a list of numbers")
    temps = [float(t) for t in temps]
    if not 2 <= len(temps) <= MAX_RUNGS:
        raise JsThrow("options.temperatures must have between 2 and %d entries" % MAX_RUNGS)
    if not all(math.isfinite(t) for t in temps):
        raise JsThrow("options.temperatures must be finite")
    if temps[0] != 1.0:
        raise JsThrow("options.temperatures must start at 1")
    if not all(a < b for a, b in zip(temps, temps[1:])):
        raise JsThrow("options.temperatures must be strictly increasing")
    if n_chains % len(temps):
        raise JsThrow("options.temperatures: their number must divide options.chains")
    return [1.0 / t for t in temps]


def dispersal_failure_message(n_failed: int, n_chains: int, distributed: bool = False, device: int = 0) -> Optional[str]:
    """What options.init_radius raises when chains found no starting point (None: every chain found one). `n_failed` counts this
    handle's chains; with `distributed` it is summed over all ranks first, so that every rank takes the same decision."""
    if distributed:
        from .parallel import total_over_ranks
        n_failed = total_over_ranks(n_failed, device)
    if n_failed <= 0:
        return None
    return "options.init_radius: %d of %d chains found no starting point with a finite log_post in %d attempts" % (
        n_failed, n_chains, DISPERSE_ATTEMPTS)


RESTORE_REFUSED_ELSEWHERE = "restore: refused on another rank; no rank was changed"


def restore_images(images) -> List[np.ndarray]:
    """restore()'s argument -> one uint8 array per image, without copying: bytes, bytearray and memoryview are images, as is a
    non-empty list or tuple of them. Anything else raises."""
    kinds = (bytes, bytearray, memoryview)
    if isinstance(images, kinds):
        images = [images]
    if not isinstance(images, (list, tuple)) or not images or not all(isinstance(x, kinds) for x in images):
        raise JsThrow("restore expects a checkpoint image (bytes, bytearray or memoryview) or a list of them")
    out = []
    for x in images:
        try:
            out.append(np.frombuffer(x, dtype=np.uint8))
        except (ValueError, BufferError):                      # a non-contiguous memoryview
            out.append(np.frombuffer(memoryview(x).tobytes(), dtype=np.uint8))
    return out


def restore_with(load, distributed: bool = False, device: int = 0):
    """The decision of a restore. load(dry_run) runs amwg_checkpoint_load and returns "" or its refusal. With `distributed` every rank
    validates first and the refusals are counted over all ranks: if any rank refuses, no rank commits, the refusing ranks raise their
    own message and the others RESTORE_REFUSED_ELSEWHERE."""
    if distributed:
        err = load(True)
        from .parallel import total_over_ranks
        if total_over_ranks(1 if err else 0, device) > 0:
            raise JsThrow(err or RESTORE_REFUSED_ELSEWHERE)
    err = load(False)
    if err:
        raise JsThrow(err)


def _default_device() -> int:
    return int(os.environ.get("LOCAL_RANK", "0")) if os.environ.get("AMWG_DEVICE") is None else int(os.environ["AMWG_DEVICE"])


# ------------------------------------------------------------------------------------------------
# option resolution -- AmwgStepper ctor (mcmc.js:837-881) + stepper ctors (:500-505, :644-649)
# ------------------------------------------------------------------------------------------------
_STEPPER_OPTIONS = (("prop_log_scale", 0), ("batch_size", 50), ("max_adaptation", 0.33), ("initial_adaptation", 1.0),
                    ("target_accept_rate", 0.44), ("is_adapting", True))


def resolve_stepper_options(params: Dict[str, dict], options: Optional[dict]) -> Dict[str, Dict[str, list]]:
    """Per parameter, per option: the flat list (one entry per component) the reference's steppers end up with.

    Reproduces the `a || b` merge of mcmc.js:871-878, including its quirks: falsy per-parameter and global values
    (0, false) fall through to the next level, and options.params[name] is mutated in place."""
    out: Dict[str, Dict[str, list]] = {}
    for name, param in params.items():
        if param["type"] not in _TYPE_CODE:
            raise JsThrow("AmwgStepper can't handle parameter " + name + " with type " + str(param["type"]))
        options = options or {}
        po = (options.get("params") or {}).get(name) if _js_truthy(options.get("params")) else None
        param_options = po if _js_truthy(po) else {}
        for key, _ in _STEPPER_OPTIONS:
            mine = param_options.get(key)
            param_options[key] = mine if _js_truthy(mine) else options.get(key)
        resolved: Dict[str, list] = {}
        if param["type"] != "binary":
            for key, default in _STEPPER_OPTIONS:
                if array_equal(param["dim"], [1]):
                    resolved[key] = [get_option(key, param_options, default)]
                else:
                    resolved[key] = _flatten(get_multidim_option(key, param_options, param["dim"], default))
        out[name] = resolved
    return out


# ------------------------------------------------------------------------------------------------
# Sampler / AmwgSampler -- mcmc.js:940-1099
# ------------------------------------------------------------------------------------------------
class Sampler:
    """mcmc.js:940-1073.  `create_stepper_ensamble` is the subclass hook, as in the reference."""

    def __init__(self, params, log_post, data=None, options=None):
        self.data = data
        self.param_names = list(params.keys())
        self.param_init_fun = get_option("param_init_fun", options, param_init_fixed)
        thinning_interval = get_option("thin", options, 1)
        params_to_monitor = get_option("monitor", options, None)
        self.thin(thinning_interval)
        self.monitor(params_to_monitor)
        self.options = options
        self.params = complete_params(params, self.param_init_fun)
        self._user_log_post = log_post
        self._handle = None
        self.steppers = self.create_stepper_ensamble(self.params, None, log_post, self.options)

    def create_stepper_ensamble(self, params, state, log_post, options):
        raise JsThrow("Every Sampler needs to implement create_stepper_ensamble()")

    def thin(self, thinning_interval):
        """mcmc.js:1053-1055"""
        self.thinning_interval = thinning_interval

    def monitor(self, params_to_monitor):
        """mcmc.js:1045-1047"""
        self.monitored_params = params_to_monitor


class AmwgSampler(Sampler):
    """mcmc.js:1090-1099 -- the AMWG sampler, `options["chains"]` chains at once on one H100."""

    # -- construction ---------------------------------------------------------------------------
    def _resolve_options(self, params, options):
        """AmwgStepper's per-parameter option merge (mcmc.js:871-878); the stand-alone steppers read `options` directly."""
        return resolve_stepper_options(params, options)

    def create_stepper_ensamble(self, params, state, log_post, options):
        options = options if options is not None else {}
        self.n_chains = int(get_option("chains", options, 1))
        if self.n_chains < 1:
            raise JsThrow("options.chains must be >= 1")
        seed = get_option("seed", options, None)
        self.seed = int.from_bytes(os.urandom(8), "little") if seed is None else int(seed) & 0xFFFFFFFFFFFFFFFF
        self.device = int(get_option("device", options, _default_device()))
        self.distributed = bool(get_option("distributed", options, False))
        self.gather = get_option("gather", options, "all")                # distributed sample(): "all" | "root" | "none"
        if self.gather not in ("all", "root", "none"):
            raise JsThrow("options.gather must be \"all\", \"root\" or \"none\"")
        self.faithful = bool(get_option("faithful", options, False))      # no factorised plates: bit-faithful sums, slower
        radius = get_option("init_radius", options, None)                  # over-dispersed starting points (DESIGN.md §2)
        if radius is not None and not (is_number(radius) and math.isfinite(radius) and radius > 0):
            raise JsThrow("options.init_radius must be a finite number > 0")
        self.init_radius = None if radius is None else float(radius)
        size = get_option("superchain_size", options, None)               # chains per superchain (nested R-hat, DESIGN.md §4.6)
        if size is not None:
            if not (is_number(size) and math.isfinite(size) and size >= 1 and size == math.floor(size)):
                raise JsThrow("options.superchain_size must be an integer >= 1")
            if self.n_chains % int(size):
                raise JsThrow("options.superchain_size must divide options.chains")
        self.superchain_size = None if size is None else int(size)
        temps = get_option("temperatures", options, None)                 # parallel tempering (DESIGN.md §2 "Tempered ladders")
        self.betas = None if temps is None else ladder_betas(temps, self.n_chains)
        self.temperatures = None if temps is None else [float(t) for t in temps]
        if self.betas is not None and self.superchain_size is not None:
            raise JsThrow("options.superchain_size cannot be combined with options.temperatures: superchains of tempered chains are not defined")
        K = 1 if self.betas is None else len(self.betas)

        # flat component layout: Object.keys(params) order, row-major inside a parameter
        self._offsets: Dict[str, int] = {}
        n_comp = 0
        for name in self.param_names:
            self._offsets[name] = n_comp
            n_comp += int(np.prod(self.params[name]["dim"]))
        self.n_comp = n_comp

        resolved = self._resolve_options(self.params, options)
        self._program, self._derived_names = trace(self._user_log_post, self.params, self._offsets, n_comp, self.data, self.faithful)

        # shard the chains when running one process per GPU (torch.distributed, see parallel.py)
        self.first_chain, self.local_chains = int(get_option("first_chain", options, 0)), self.n_chains
        if self.distributed:
            from .parallel import check_ladder_shards, shard_chains
            self.first_chain, self.local_chains = shard_chains(self.n_chains)
            if self.betas is not None:
                check_ladder_shards(self.n_chains, K)
        elif self.betas is not None and self.first_chain % K:
            raise JsThrow("options.first_chain must be a multiple of the number of temperatures")
        # the chains sample() and sample_summary() return: all of them, or the T = 1 rung of every ladder
        self.cold_chains, self.local_cold = self.n_chains // K, self.local_chains // K

        self._build_model(resolved)
        return ["AmwgStepper"]

    def _build_model(self, resolved):
        P = len(self.param_names)
        prm = (AmwgParam * P)()
        init = np.empty(self.n_comp)
        opts = (AmwgCompOptions * self.n_comp)()
        for k, name in enumerate(self.param_names):
            p = self.params[name]
            ncomp = int(np.prod(p["dim"]))
            off = self._offsets[name]
            prm[k] = AmwgParam(_TYPE_CODE[p["type"]], ncomp, int(p["dim"][0]), off, float(p["lower"]), float(p["upper"]))
            flat = _flatten(p["init"])
            if len(flat) != ncomp:
                raise JsThrow("The init of parameter " + name + " does not match its dim")
            init[off:off + ncomp] = [float(v) for v in flat]
            for c in range(ncomp):
                o = opts[off + c]
                if p["type"] == "binary":
                    o.prop_log_scale, o.batch_size, o.max_adaptation = 0.0, 50.0, 0.33
                    o.initial_adaptation, o.target_accept_rate, o.is_adapting = 1.0, 0.44, 0
                else:
                    r = resolved[name]
                    o.prop_log_scale = float(r["prop_log_scale"][c]); o.batch_size = float(r["batch_size"][c])
                    o.max_adaptation = float(r["max_adaptation"][c]); o.initial_adaptation = float(r["initial_adaptation"][c])
                    o.target_accept_rate = float(r["target_accept_rate"][c]); o.is_adapting = 1 if r["is_adapting"][c] else 0
        prog = self._program
        code = np.asarray(prog.code, dtype=np.int32)
        consts = np.asarray(prog.consts if prog.consts else [0.0], dtype=np.float64)
        cols = (AmwgColumn * max(len(prog.columns), 1))()
        self._col_keepalive = [np.ascontiguousarray(c, dtype=np.float64) for c in prog.columns]
        for k, c in enumerate(self._col_keepalive):
            cols[k] = AmwgColumn(c.ctypes.data_as(C.POINTER(C.c_double)), c.size)
        plates = (AmwgPlate * max(len(prog.plates), 1))()
        for k, pl in enumerate(prog.plates):
            q = AmwgPlate()
            q.kind, q.n = pl["kind"], pl["n"]
            for j in range(4):
                q.col[j] = pl["col"][j]; q.iparam[j] = pl["iparam"][j]
            plates[k] = q
        m = AmwgModel()
        m.abi_version = _ffi.ABI_VERSION
        m.n_params, m.params = P, prm
        m.n_comp, m.init = self.n_comp, init.ctypes.data_as(C.POINTER(C.c_double))
        m.comp_options = opts
        m.n_code, m.code = code.size, code.ctypes.data_as(C.POINTER(C.c_int32))
        m.logpost_prog, m.derived_prog, m.n_derived = prog.logpost_prog, prog.derived_prog, len(self._derived_names)
        m.n_consts, m.consts = consts.size, consts.ctypes.data_as(C.POINTER(C.c_double))
        m.n_columns, m.columns = len(prog.columns), cols
        m.n_plates, m.plates = len(prog.plates), plates
        fold_prog = np.asarray(prog.fold_prog if prog.fold_prog else [0], dtype=np.int32)
        fold_dst = np.asarray(prog.fold_dst if prog.fold_dst else [0], dtype=np.int32)
        m.n_fold = len(prog.fold_prog)
        m.fold_prog = fold_prog.ctypes.data_as(C.POINTER(C.c_int32))
        m.fold_dst = fold_dst.ctypes.data_as(C.POINTER(C.c_int32))
        comp_prog = np.asarray(prog.comp_prog if prog.n_terms else [0], dtype=np.int32)
        touch_off = np.asarray(prog.touch_off if prog.n_terms else [0], dtype=np.int32)
        touch_terms = np.asarray(prog.touch_terms if prog.touch_terms else [0], dtype=np.int32)
        m.n_terms = prog.n_terms
        m.comp_prog = comp_prog.ctypes.data_as(C.POINTER(C.c_int32)) if prog.n_terms else None
        m.touch_off = touch_off.ctypes.data_as(C.POINTER(C.c_int32)) if prog.n_terms else None
        m.touch_terms = touch_terms.ctypes.data_as(C.POINTER(C.c_int32)) if prog.n_terms else None
        block_params = np.asarray(prog.block_params if prog.block_params else [0], dtype=np.int32)
        tbc = np.asarray(prog.term_block_comp if prog.term_block_comp else [0], dtype=np.int32)
        m.n_block_params = len(prog.block_params)
        m.block_params = block_params.ctypes.data_as(C.POINTER(C.c_int32)) if prog.block_params else None
        m.term_block_comp = tbc.ctypes.data_as(C.POINTER(C.c_int32)) if prog.block_params else None
        m.stat_prog = prog.stat_prog
        m.n_sum_terms = prog.n_sum_terms if prog.stat_prog >= 0 else prog.n_terms
        self._cache_keepalive = (comp_prog, touch_off, touch_terms, block_params, tbc)
        vcomps = np.asarray(prog.variant_comps if prog.variant_comps else [0], dtype=np.int32)
        vlp = np.asarray(prog.variant_logpost if prog.variant_logpost else [0], dtype=np.int32)
        vder = np.asarray(prog.variant_derived if prog.variant_derived else [-1], dtype=np.int32)
        m.n_variant_comps = len(prog.variant_comps)
        m.variant_comps = vcomps.ctypes.data_as(C.POINTER(C.c_int32))
        m.variant_logpost = vlp.ctypes.data_as(C.POINTER(C.c_int32))
        m.variant_derived = vder.ctypes.data_as(C.POINTER(C.c_int32))
        self._model_keepalive = (prm, init, opts, code, consts, cols, plates, fold_prog, fold_dst, vcomps, vlp, vder, m)
        L = _ffi.lib()
        if get_option("_model_only", self.options, False):       # tests: lower the model, do not touch a device
            self._model = m
            return
        h = C.c_void_p()
        rc = L.amwg_create(C.byref(m), self.local_chains, self.first_chain, self.seed, self.device, C.byref(h))
        if rc != 0:
            raise JsThrow(L.amwg_last_error().decode())
        self._handle = h
        if self.betas is not None:
            b = np.asarray(self.betas, dtype=np.float64)
            if L.amwg_set_ladder(h, b.ctypes.data_as(C.POINTER(C.c_double)), b.size) != 0:
                err = L.amwg_last_error().decode()
                self.close()
                raise JsThrow(err)
        if self.init_radius is not None:
            self._disperse(self.init_radius)

    def _disperse(self, radius: float):
        """options.init_radius: every chain to its first valid point of the device's dispersal (amwg_disperse_state_superchains; with
        options.superchain_size the chains of a superchain share one point). With options.distributed the failed chains are counted
        over all ranks, so that every rank raises the same message or none."""
        L = _ffi.lib()
        failed = C.c_int64(0)
        rc = L.amwg_disperse_state_superchains(self._handle, float(radius), self.superchain_size or 1, C.byref(failed))
        err = L.amwg_last_error().decode() if rc != 0 else ""
        msg = dispersal_failure_message(failed.value, self.n_chains, self.distributed, self.device)
        if rc != 0 or msg:
            self.close()
            raise JsThrow(msg or err)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_handle", None):
            _ffi.lib().amwg_destroy(self._handle)
            self._handle = None

    # -- layout helpers -------------------------------------------------------------------------
    def _state_keys(self) -> List[str]:
        """Object.keys(state): the parameters, then the derived quantities in creation order (mcmc.js:1010)."""
        return self.param_names + self._derived_names

    def _entries(self, name: str) -> List[int]:
        if name in self._offsets:
            n = int(np.prod(self.params[name]["dim"]))
            return list(range(self._offsets[name], self._offsets[name] + n))
        if name in self._derived_names:
            return [self.n_comp + self._derived_names.index(name)]
        return []          # JS: state[name] is undefined -> the column is filled with undefined

    def _shape_out(self, name: str, arr: np.ndarray, chains_total: Optional[int] = None) -> np.ndarray:
        """arr: [rows, entries, chains] -> reference-shaped array ([rows, *dim] for one chain, else [rows, chains, *dim]); one chain
        means `chains_total` chains in all (default options.chains; sample() passes the cold chains of a tempered sampler)."""
        rows, _, chains = arr.shape
        dim = self.params[name]["dim"] if name in self.params else [1]
        a = np.moveaxis(arr, 1, 2)                        # [rows, chains, entries]
        a = a.reshape(rows, chains) if list(dim) == [1] else a.reshape(rows, chains, *dim)
        return a[:, 0] if (self.n_chains if chains_total is None else chains_total) == 1 else a

    # -- the reference's methods -----------------------------------------------------------------
    def step(self):
        """mcmc.js:985-997 -- one sweep; returns the live state."""
        self.burn(1)
        return self.state

    @property
    def state(self) -> Dict[str, Any]:
        L = _ffi.lib()
        n_entries = self.n_comp + len(self._derived_names)
        buf = np.empty((n_entries, self.local_chains))
        _ffi.check(L.amwg_get_state(self._handle, buf.ctypes.data))
        out = {}
        for name in self._state_keys():
            e = self._entries(name)
            out[name] = self._shape_out(name, buf[e][None, :, :])[0]
        return out

    def set_state(self, values: Dict[str, Any]):
        """Not in the reference: place the chains, e.g. where a previous run, prior draws or an optimiser left them. `values` is keyed
        by parameter name; each value is shaped like `state[name]` ([chains, *dim], [chains] for a scalar parameter; the reference's
        shape for one chain), or like one chain's value (`dim`, a number for a scalar parameter), which every chain receives.
        Parameters not named keep their values. log_post and its cached terms are evaluated afresh; proposal scales, adaptation and
        the random streams carry on untouched, so each chain continues as the reference chain would from that point. With
        options.distributed the arrays cover all `chains` global chains and every rank takes its own."""
        if not isinstance(values, dict):
            raise JsThrow("set_state expects an object keyed by parameter name")
        L = _ffi.lib()
        cur = np.empty((self.n_comp + len(self._derived_names), self.local_chains))
        _ffi.check(L.amwg_get_state(self._handle, cur.ctypes.data))
        block = np.ascontiguousarray(self._set_state_block(values, cur[:self.n_comp]))
        if L.amwg_set_state(self._handle, block.ctypes.data) != 0:
            raise JsThrow(L.amwg_last_error().decode())

    def _set_state_block(self, values: Dict[str, Any], current: np.ndarray) -> np.ndarray:
        """set_state's argument over `current` ([n_comp, local_chains]: the state now) -> the [n_comp, local_chains] block of
        amwg_set_state. Host-side shaping only: checked without a device."""
        from .parallel import local_chain_rows
        out = np.array(current, dtype=np.float64, copy=True)
        first = self.first_chain if self.distributed else 0
        for name, v in values.items():
            if name in self._derived_names:
                raise JsThrow("set_state: " + name + " is a derived quantity, not a parameter")
            if name not in self._offsets:
                raise JsThrow("set_state: " + name + " is not a parameter of this sampler")
            dim = list(self.params[name]["dim"])
            n, off = int(np.prod(dim)), self._offsets[name]
            try:
                a = np.asarray(v, dtype=np.float64)
            except (TypeError, ValueError):
                raise JsThrow("set_state: the value of " + name + " is not numeric") from None
            one = [] if dim == [1] else dim                       # one chain's value: a number for a scalar parameter
            per_chain = [self.n_chains] + one
            if list(a.shape) in (one, dim):
                out[off:off + n, :] = a.reshape(n, 1)
            elif list(a.shape) == per_chain:
                out[off:off + n, :] = local_chain_rows(a.reshape(self.n_chains, n), first, self.local_chains).T
            else:
                raise JsThrow("set_state: " + name + " is of dimension [" + _js_join(list(a.shape)) + "] but should be [" + _js_join(dim) +
                              "] or [" + _js_join(per_chain) + "]")
        return out

    def checkpoint(self) -> bytes:
        """Not in the reference: the image of this handle's chains (with options.distributed: this rank's shard), from which `restore`
        resumes the run bit for bit, in this or another process, on any sharding (DESIGN.md §2 "Checkpoints"). thin and monitor are
        not part of it."""
        L = _ffi.lib()
        n = C.c_int64(0)
        _ffi.check(L.amwg_checkpoint_size(self._handle, C.byref(n)))
        buf = np.empty(n.value, dtype=np.uint8)
        if L.amwg_checkpoint_save(self._handle, buf.ctypes.data, n.value) != 0:
            raise JsThrow(L.amwg_last_error().decode())
        return buf.tobytes()

    def restore(self, images):
        """Not in the reference: resume the run `images` were taken from (one bytes-like image, or a list of them, e.g. every rank's
        file of an earlier run). The sampler must have the same model, data and options; the images together must cover its chains
        (more is fine). Afterwards every chain continues exactly as it would have without the interruption, and `self.seed` is the
        images' seed. A refused restore raises "restore: ..." and changes nothing. With options.distributed every rank checks its
        images first and no rank changes unless all of them can."""
        imgs = restore_images(images)
        L = _ffi.lib()
        ptrs = (C.c_void_p * len(imgs))(*[a.ctypes.data for a in imgs])
        sizes = (C.c_int64 * len(imgs))(*[a.size for a in imgs])

        def load(dry_run: bool) -> str:
            rc = L.amwg_checkpoint_load(self._handle, ptrs, sizes, len(imgs), 1 if dry_run else 0)
            return L.amwg_last_error().decode() if rc != 0 else ""
        restore_with(load, self.distributed, self.device)
        self.seed = int.from_bytes(imgs[0][32:40].tobytes(), "little")

    def model_fingerprint(self) -> int:
        """amwg_model_fingerprint of this sampler's lowered model (no device needed): what checkpoint images are matched against."""
        out = C.c_uint64(0)
        _ffi.check(_ffi.lib().amwg_model_fingerprint(C.byref(self._model_keepalive[-1]), C.byref(out)))
        return int(out.value)

    def log_post(self):
        """mcmc.js:958-960 -- `sampler.log_post()`: log_post at the current state (one number, or one per chain)."""
        buf = np.empty(self.local_chains)
        _ffi.check(_ffi.lib().amwg_get_log_post(self._handle, buf.ctypes.data))
        return float(buf[0]) if self.n_chains == 1 else buf

    def burn(self, n_iterations):
        """mcmc.js:1035-1039"""
        L = _ffi.lib()
        rc = L.amwg_burn(self._handle, int(n_iterations))
        if rc != 0:
            raise JsThrow(L.amwg_last_error().decode())

    def sample(self, n_iterations):
        """mcmc.js:1005-1030 -- {name: draws}; rows = ceil(n/thin); row r is the state before sweep r*thin."""
        from .summary import entry_spans
        monitored = self._state_keys() if self.monitored_params is None else list(self.monitored_params)
        entries = [i for name in monitored for i in self._entries(name)]
        spans = entry_spans(monitored, {name: [len(self._entries(name))] for name in monitored})
        n = int(n_iterations)
        thin = abs(int(self.thinning_interval))                 # `i % thin === 0` (mcmc.js:1021): the sign of thin does not matter ...
        if thin == 0:                                           # ... and i % 0 is NaN: nothing is ever recorded, the chains still step
            self.burn(max(n, 0))
            return {name: np.empty((0,)) for name in monitored}
        rows = 0 if n <= 0 else (n + thin - 1) // thin
        raw = self._sample_raw(n, thin, entries, rows)          # [rows, n_entries, chains]
        out = {}
        for name in monitored:
            s, ln = spans[name]
            if ln == 0:
                out[name] = np.full((rows,), np.nan)
            else:
                out[name] = self._shape_out(name, raw[:, s:s + ln, :], self.cold_chains)
        return out

    def _sample_raw(self, n: int, thin: int, entries: List[int], rows: int) -> np.ndarray:
        L = _ffi.lib()
        mon = np.asarray(entries, dtype=np.int32)
        if self.distributed:
            from .parallel import sample_and_gather
            return sample_and_gather(self, n, thin, mon, rows)
        buf = _pinned_empty((rows, len(entries), self.local_cold))
        rc = L.amwg_sample(self._handle, n, thin, mon.ctypes.data_as(C.POINTER(C.c_int32)), len(entries), buf.ctypes.data)
        if rc != 0:
            raise JsThrow(L.amwg_last_error().decode())
        return buf

    def sample_summary(self, n_iterations, probs=(0.025, 0.25, 0.5, 0.75, 0.975), diagnostics=False, histogram=None, covariance=None,
                       nested=None, loo=None, ppc=None, mcse=False):
        """Not in the reference (SURVEY 8(f).3): the same sweeps and the same kept rows as `sample(n)` (thin / monitor apply), but the
        draws stay in HBM and only their summary comes back: {name: {"mean", "sd", "rhat", "quantiles", "n_draws"}}, pooled over
        all chains and kept rows; multi-dim parameters give arrays of their `dim` ("quantiles": [len(probs), *dim], exact order
        statistics with numpy.quantile's linear rule; a long grid such as numpy.linspace(0, 1, 41) gives an equal-mass histogram and
        runs as several radix selects of 16 probabilities each). With options.distributed every rank returns the all-GPU summary
        (two small collectives, summary.py). Advances the chains exactly as sample(n) does. A NaN or +-inf draw (a derived quantity
        such as Math.log(mu) or 1/x) is summarised as numpy summarises it: a NaN draw makes the entry's mean and every quantile NaN;
        +inf draws alone make the mean +inf, -inf draws alone -inf, both NaN; sd and rhat are NaN. Only an entry whose finite
        draws overflow the sum can differ from numpy.mean (summary.nonfinite_as_numpy).
        diagnostics=True adds, per parameter and shaped like "mean": "ess_mean" and "ess_tail" (split-chain effective sample
        sizes of the draws and of the 5 % / 95 % tail indicators, Vehtari et al. 2021), "mcse_mean" (sd / sqrt(ess_mean)) and
        "rhat_split" (split-chain R-hat, not rank-normalised); the other keys keep their values bit for bit. Fewer than 10 kept
        rows give NaN; see summary.split_chain_diagnostics for the estimator and its edge cases. The R-hats compare chains, so they
        can only flag what the chains' starting points let them see: by default every chain starts at the same init, and chains
        that all stay in one mode report R-hat near 1. options.init_radius draws over-dispersed starting points (DESIGN.md §2);
        set_state places the chains anywhere.
        diagnostics="rank" returns everything diagnostics=True does, bit for bit, plus "ess_bulk" (ESS of the rank-normalised
        split chains) and "rhat_rank" (the larger split R-hat of the rank-normalised draws and of the rank-normalised folded draws
        |x - median|), ranked over the pooled draws of all chains on all GPUs (Vehtari et al. 2021, §4; the numbers Stan and
        ArviZ print). They stay finite with +-inf draws and catch chains that differ in scale only; see summary.rank_diagnostics.
        Ranking needs 56 bytes of device scratch per ranked draw for one parameter entry at a time. Any other value raises.
        histogram=k (or {"bins": k}) adds equal-width posterior histograms, counted on the device and equal to numpy's on the raw
        draws count for count. A dict may hold "bins" (1..4096 per entry; may be left out when only pairs are wanted), "range"
        ({name: (lo, hi)}, finite lo < hi, for every component of that name), "pairs" (at most 64 (a, b), each selector a scalar's
        name or (name, flat_index) for one component, row-major) and "pair_bins" (1..128 per axis, default 50). Each monitored
        name gains, shaped like "quantiles" with the bins last ([k] or [*dim, k]): "hist" (int64 counts), "hist_edges" (k + 1
        edges) and "hist_outside" (int64 [3]: draws < lo, > hi and NaN; infinities count as below or above), so hist.sum() +
        hist_outside.sum() == n_draws. The range is range[name] when given, else the smallest and largest finite draw over all
        chains, rows and GPUs (numpy.histogram's default on the finite draws), widened to (lo - 0.5, hi + 0.5) when lo == hi, and
        (0, 1) when there is no finite draw. The edges are numpy.linspace(lo, hi, k + 1), and a draw lo <= x <= hi goes to the bin
        numpy.histogram gives it (its equal-width arithmetic, in the same fp64 operations). Each pair adds a top-level entry keyed by
        the pair as given: {"hist": int64 [pair_bins, pair_bins] (a on axis 0), "xedges", "yedges"}, the edges being linspace(lo,
        hi, pair_bins + 1) of each selector's range; a draw counts when both values lie inside, binned as numpy.histogram2d bins
        it. Every other key keeps its bits. A refused histogram raises ValueError before the chains move (summary.resolve_histogram).
        covariance=True adds the posterior covariance of every monitored entry, formed on the device (the cross-products of the
        draws on the fp64 tensor core); a list of selectors (each a scalar's name or (name, flat_index), as for the histogram
        pairs; at most 128 entries) covers those only, in the order given. The result gains the top-level key "covariance":
        {"labels" (the selectors in matrix order; with True, every monitored name in order, a multi-dim one as (name, flat_index)
        row-major), "mean" [k], "cov" [k, k] (ddof 1, over all rows and chains: numpy.cov of the pooled draws; its diagonal is
        "sd" squared), "corr" [k, k] (numpy.corrcoef's), "within" (mean within-chain covariance, ddof 1), "between" (covariance
        of the chain means, ddof 1), "rhat_multivariate" (Brooks & Gelman 1998: (n - 1)/n + (C + 1)/C lambda_max(within^-1
        between), n kept rows, C chains; it flags chains that disagree on a combination of entries while every univariate R-hat
        passes) and "n_draws"}. A NaN or +-inf draw makes its entry's rows and columns NaN, as numpy.cov does; rhat_multivariate
        is NaN with fewer than 2 rows or chains, any non-finite entry, or a within matrix that is not positive definite (a
        constant entry, or a derived quantity linear in others). The device scratch (summary.comoments_scratch_bytes) is counted
        in the memory check. Every other key keeps its bits. A refused covariance (an unknown name, a component out of range,
        more than 128 entries, anything but None / False / True / a list, or a monitored name "covariance") raises ValueError
        before the chains move (summary.resolve_covariance); see summary.finalize_comoments for the arithmetic.
        nested=M adds "rhat_nested" to every monitored name, shaped like "mean": the nested R-hat of Margossian et al. (Bayesian
        Analysis 2024) for superchains of M chains, superchain k being the global chains [kM, (k + 1)M). It is built for many
        short chains: it compares the superchain means with the variance inside the superchains, is defined for one kept row, and
        tends to 1 once the ensemble of chains is stationary, whether or not each chain is long. nested=True takes M from
        options.superchain_size, which with options.init_radius also starts the chains of each superchain at one point; nested=M
        sets it for this call (for chains placed with set_state). With N kept rows, K superchains, chain means xbar_km,
        superchain means xbar_k and xbar their mean: B^ = sum_k (xbar_k - xbar)^2 / (K - 1), B~_k = sum_m (xbar_km - xbar_k)^2 /
        (M - 1) (0 when M = 1), W-_k = (1/M) sum_m sum_n (x_nmk - xbar_km)^2 / (N - 1) (0 when N = 1), W^ = (1/K) sum_k (B~_k +
        W-_k), rhat_nested = sqrt(1 + B^ / W^); NaN when K < 2, W^ = 0 or any draw of the entry is not finite. The chains
        summarised (this handle's, or all of them with options.distributed) must be whole superchains. The device scratch
        (summary.nested_scratch_bytes) is counted in the memory check. Every other key keeps its bits. A refused nested (True
        without options.superchain_size, anything but None / False / True / an int >= 1, or chains that are not whole
        superchains) raises ValueError before the chains move (summary.resolve_nested); see summary.finalize_nested.
        loo={"log_lik": f, "points": N} (optional "r_eff": a finite float > 0, default 1.0) adds the top-level key "loo": PSIS-LOO
        and WAIC (Vehtari, Gelman & Gabry 2017; Vehtari et al. 2024) in ArviZ's conventions, from the pointwise log-likelihood
        ll[s, i] = f(state, data, i) at every kept draw s (S = kept rows x chains, on all GPUs with options.distributed) and point
        i < N, formed on the device and never moved to the host. f is traced once with a symbolic point index i, as a body under
        mcmc.points(n) is (data.y[i], mu[data.g[i]], ld.*, Math.*), and evaluated with the model's arithmetic; components it reads
        that are not monitored are sampled alongside and not returned. The dict holds "elpd_loo", "se_elpd_loo", "p_loo", "looic",
        "elpd_waic", "se_elpd_waic", "p_waic", "waic", "pointwise" ({"elpd_loo", "lppd", "p_loo", "elpd_waic", "p_waic",
        "pareto_k"}, each [N]), "pareto_k_threshold" (min(1 - 1/log10 S, 0.7)), "n_high_k", "r_eff", "n_draws" and "points"; see
        summary.loo_block for the estimator. A point with a non-finite ll is NaN throughout, and so are the totals. r_eff = 1 is exact
        for one row of independent chains; pass the relative efficiency for long chains. The points run in chunks sized to the
        free device memory. Every other key keeps its bits. A refused loo (not a dict, unknown keys, points not an int >= 1, r_eff
        not finite and > 0, a log_lik that branches on a parameter or indexes past a data array for some i < N, fewer than 2
        draws, or a monitored name "loo") raises ValueError before the chains move (summary.resolve_loo, tracer.trace_log_lik).
        ppc={"log_lik": f, "points": N} adds the top-level key "ppc": posterior predictive checks (BDA3 ch. 6; ArviZ's plot_ppc /
        plot_bpv). f is the kind of function loo= takes (often the same one), traced the same way; its value must be one ld.* call
        whose first argument is a data value at the point index, e.g. ld.norm(data.y[i], mu[data.g[i]], sigma): that names the
        observation y_i and the family, and the other arguments are the family's parameters at point i. At every kept draw (S =
        kept rows x chains, all GPUs with options.distributed) the device draws a replicated dataset y_rep_0 .. y_rep_{N-1} from
        that family (csrc/amwg_ppc.cuh: every family but hyper, with the samplers and domains listed there; parameters outside the
        domain give NaN), from the chain's own Math.random() stream at positions reserved for (kept row, point) (DESIGN.md §4.8:
        repeated calls reuse those positions for new posterior draws), and nothing of it moves to the host. The dict holds
        "family" (the ld name), "points", "n_draws", "pointwise" ({"mean", "sd" (pooled, ddof 1), "n_below", "n_equal", "n_nan"
        (int64: y_rep_i < y_i, == y_i, NaN), "pit" = (n_below + n_equal) / S}, each [N]) and "stats": for each T in "mean", "sd",
        "min", "max" of a dataset (points in index order; sequential Welford, sd ddof 1, NaN-propagating min / max) {"observed"
        T(y), "mean", "sd", "quantiles" (probs) of T(y_rep), "n_greater", "n_equal", "n_nan", "p_value" = (n_greater + n_equal)
        / S: Pr(T(y_rep) >= T(y)), a NaN draw counting as not >=}; see summary.ppc_block. With loo= it shares the sample block.
        The points run in chunks sized to the free device memory. Every other key keeps its bits. A refused ppc (not a dict,
        unknown keys, points not an int >= 1, anything loo refuses in f, a value that is not one ld.* call with data[i] first, a
        family without a sampler, kept rows x points >= 2^46, or a monitored name "ppc") raises ValueError before the chains move
        (summary.resolve_ppc, summary.check_ppc_call, tracer.LogLik.observed_call).
        ppc={..., "loo_pit": True} (or {"r_eff": r}, r a finite float > 0; True means r = 1.0, as in loo=) adds "loo_pit" to the
        "ppc" dict: the PIT of each observation under its leave-one-out predictive (LOO-PIT; Gabry et al. 2019, Säilynoja, Bürkner &
        Vehtari 2022; ArviZ's loo_pit), which the in-sample "pit" cannot give: there y_i shapes the posterior that predicts it. It
        holds {"pit", "pit_equal", "pareto_k" (float64 [N] each), "pareto_k_threshold", "n_high_k", "r_eff"}. The log-likelihood is
        ppc's own f, the ld.* call y_rep is drawn from, evaluated on the device as loo= evaluates its body (loo= is not needed).
        Definition, per point i over the S draws: ll_s, lw_s = llmin - ll_s, M, cut, the tail T = {s : lw_s > cut}, k^, sigma^ and
        the smoothed weights are those of loo= (DESIGN.md §4.7). The tail sorted by ascending lw has ranks j = 0..n-1; its smoothed
        weight is w'_j = exp(min(0, log(gpinv((j + 0.5)/n; k^, sigma^) + exp(cut)))) when k^ is finite, and exp(lw) otherwise.
        Ties: the sorted tail splits into maximal runs of equal ll, and every draw of run R gets the run's mean weight
        (sum_{j in R} w'_j) / |R|; a draw outside the tail gets exp(lw_s). D is the sum of all weights (elpd_loo's normaliser: a run's
        mean keeps its total), LE the sum of the weights of draws with y_rep_s <= y_i and EQ of those with y_rep_s == y_i (a NaN
        y_rep counts in D only); pit_i = min(1, LE / D) and pit_equal_i = min(1, EQ / D), so pit - U pit_equal (U uniform) is the
        randomised PIT of a count family. pareto_k is loo='s k^ (+inf for a tail of <= 4 draws or when no candidate of the fit
        has a finite profile value); the threshold and n_high_k are loo='s. A point with any non-finite ll gets NaN in pit,
        pit_equal and pareto_k. Without ties this is ArviZ's min(1, exp(logsumexp(lw_norm[y_rep <= y]))); the run means make it
        independent of the order of tied draws (a rejected step repeats its ll), and so of sharding, chunking and the sort. See
        summary.loo_pit_chunk. Every other key, and the chains' state, keep their bits. A refused loo_pit (anything but True or
        {"r_eff": ...}, an r_eff not finite and > 0, fewer than 2 draws, a tail of more than 2^20 draws) raises ValueError before
        the chains move.
        mcse=True adds Monte Carlo standard errors of the quantiles and of the sd (Vehtari et al. 2021, §4.3; posterior's
        mcse_quantile / mcse_sd, ArviZ's mcse), with any diagnostics= and every other option. Per monitored name, "ess_quantile"
        and "mcse_quantile" are shaped like "quantiles": the split-chain ESS of the indicator 1[x <= q_p] for each p in probs,
        formed on the device from exact integer autocovariance sums (so it does not depend on the number of GPUs or the chain
        order), and the standard error of each returned quantile, half the distance between the two exact order statistics at
        the ranks of ArviZ's beta rule. "mcse_sd", shaped like "mean", is the delta-method standard error of "sd" from the ESS of
        the squared deviations (x - mean)^2. Fewer than 10 kept rows or a NaN draw give NaN; +-inf draws give mcse_sd NaN; a
        constant entry gives M h, 0 and 0. See summary.mcse_block for the definitions and edge cases. It needs scipy
        (scipy.special.betaincinv). Every other key, and the chains' state, keep their bits. Anything but a bool, mcse=True
        without scipy, or 2 M h^2 >= 2^63 (M = 2 x chains, h = kept rows // 2) raises ValueError before the chains move."""
        import torch
        from .summary import (CudaBlockReducer, CudaPointwise, CudaPpc, check_diagnostics, check_loo_size, check_ppc_call, comoments_scratch_bytes,
                              covariance_block, entry_spans, histogram_block, loo_block, loo_pit_point_bytes, loo_point_bytes, loo_tail_cap,
                              nested_block, nested_scratch_bytes, ppc_block, ppc_fixed_bytes, ppc_point_bytes, resolve_covariance,
                              resolve_histogram, resolve_loo, resolve_nested, resolve_ppc, summarise_block)
        from .summary import check_mcse, check_mcse_size, mcse_block, mcse_scratch_bytes
        check_diagnostics(diagnostics)
        check_mcse(mcse)
        monitored = self._state_keys() if self.monitored_params is None else list(self.monitored_params)
        entries = [i for name in monitored for i in self._entries(name)]
        spans = entry_spans(monitored, {name: [len(self._entries(name))] for name in monitored})
        named = [name for name in monitored if spans[name][1] > 0]
        dims = {name: list(self.params[name]["dim"]) if name in self.params else [1] for name in named}
        plan = resolve_histogram(histogram, named, dims)
        cov_plan = resolve_covariance(covariance, named, dims)
        first, held = (0, self.n_chains) if self.distributed else (self.first_chain, self.local_chains)
        superchain = resolve_nested(nested, self.superchain_size, first, held)
        loo_plan = resolve_loo(loo, named)
        ppc_plan = resolve_ppc(ppc, named)
        if self.betas is not None and superchain is not None:
            raise ValueError("nested= is not available with options.temperatures: superchains of tempered chains are not defined")
        if self.betas is not None and ppc_plan is not None:
            raise ValueError("ppc= is not available with options.temperatures: its stream positions are defined per chain id")
        n_chains, local_chains = self.cold_chains, self.local_cold      # the block's chain axis: the T = 1 chains
        n = int(n_iterations)
        thin = abs(int(self.thinning_interval))
        rows = 0 if (n <= 0 or thin == 0) else (n + thin - 1) // thin
        if rows == 0 or not entries:
            raise JsThrow("sample_summary needs at least one kept iteration and one monitored entry")
        if mcse:
            check_mcse_size(rows, n_chains)
        sampled = list(entries)                                 # the block's entries: the monitored ones, then what log_lik reads besides
        start = {}

        def block_entries(reads):
            for name in reads:
                if name in start:
                    continue
                if name in spans and spans[name][1] > 0:
                    start[name] = spans[name][0]
                else:
                    start[name] = len(sampled)
                    sampled.extend(self._entries(name))
        if loo_plan is not None:
            from .tracer import trace_log_lik
            loo_m = check_loo_size(rows * n_chains, loo_plan.r_eff)
            lik = trace_log_lik(loo_plan.log_lik, self.params, self._offsets, self.data, loo_plan.points)
        if ppc_plan is not None:
            from .tracer import trace_log_lik
            if ppc_plan.loo_pit is not None:
                pit_m = check_loo_size(rows * n_chains, ppc_plan.loo_pit, "ppc loo_pit")
            ppc_lik = trace_log_lik(ppc_plan.log_lik, self.params, self._offsets, self.data, ppc_plan.points, what="ppc")
            ppc_family, ppc_y, ppc_args = ppc_lik.observed_call(ppc_plan.points)
            ppc_code = check_ppc_call(ppc_family, rows, ppc_plan.points)
        if loo_plan is not None:
            block_entries(lik.reads)
            loo_prog = lik.lower(start)
        if ppc_plan is not None:
            block_entries(ppc_lik.reads)
            ppc_prog, ppc_offs = ppc_lik.lower_exprs(ppc_args, start)
            if ppc_plan.loo_pit is not None:
                pit_prog = ppc_lik.lower(start)                   # the log-likelihood of the same ld.* call, as loo= lowers its body
        L = _ffi.lib()
        dev = torch.device("cuda", self.device)
        need = rows * len(sampled) * local_chains * 8
        if len(sampled) > len(entries):
            need += rows * len(entries) * local_chains * 8         # the monitored entries' block, copied out after the loo / ppc pass
        if ppc_plan is not None:
            need += ppc_fixed_bytes(rows, local_chains)
        if plan is not None:
            # edges and counts of the histograms, and the extremes (8 B each)
            nb, pb = plan.bins or 0, plan.pair_bins
            need += 8 * (len(entries) * (2 * nb + 4 + pb + 1 + 5) + len(plan.pairs) * pb * pb)
        if cov_plan is not None:
            need += comoments_scratch_bytes(len(cov_plan.entries), local_chains)
        if superchain is not None:
            need += nested_scratch_bytes(len(entries), local_chains, self.first_chain, superchain)
        if mcse:
            need += mcse_scratch_bytes(len(entries), len(probs))
        free, _total = torch.cuda.mem_get_info(dev)
        base = need + 2 * len(entries) * local_chains * 8      # and the base summary's scratch: two doubles per entry and chain
        if base > 0.9 * free:
            raise JsThrow("sample_summary: the sample block (%.1f GB) does not fit in device memory; raise thin() or lower n" % (need / 1e9))
        if diagnostics == "rank" and rows >= 10:
            # rank_diagnostics, per entry: keys 2 x 8 B, indices 2 x 4 B, rank sums 8 B, a ring buffer 8 B and two z-blocks 2 x 8 B per
            # ranked draw (the ring buffers hold the largest shard, at most one chain more than this one), and the sort's tile
            # tables (2 x 256 x 4 B per 2048 keys)
            ranked = 2 * (rows // 2) * (local_chains + (1 if self.distributed else 0))
            scratch = 56 * ranked + 2 * 256 * 4 * (-(-ranked // 2048))
            if base + scratch > 0.9 * free:
                raise JsThrow("sample_summary: the sample block (%.1f GB) and the scratch of diagnostics=\"rank\" (%.1f GB) do not fit in "
                              "device memory; raise thin() or lower n" % (need / 1e9, scratch / 1e9))
        def chunk_size(per_point, points, what):
            chunk_points = int((0.9 * free - base) // per_point)
            if chunk_points < 1:
                raise JsThrow("sample_summary: the sample block (%.1f GB) and one point of the %s (%.1f GB) do not fit "
                              "in device memory; raise thin() or lower n" % (need / 1e9, what, per_point / 1e9))
            chunk_points = min(chunk_points, points, 65535)
            if self.distributed:                                  # every rank takes the same chunks: the collectives pair up
                t = torch.tensor([chunk_points], dtype=torch.int64, device=dev)
                torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MIN)
                chunk_points = int(t.item())
            return chunk_points
        world = torch.distributed.get_world_size() if self.distributed else 1
        if loo_plan is not None:
            chunk_points = chunk_size(loo_point_bytes(rows, local_chains, loo_tail_cap(loo_m), world), loo_plan.points,
                                      "pointwise log-likelihood")
        if ppc_plan is not None:
            per_point = ppc_point_bytes(rows, local_chains)
            if ppc_plan.loo_pit is not None:                      # LOO-PIT holds a chunk of ll beside the chunk of y_rep
                per_point += loo_pit_point_bytes(rows, local_chains, loo_tail_cap(pit_m), world)
            ppc_chunk = chunk_size(per_point, ppc_plan.points, "replicated data")
        block = torch.empty((rows, len(sampled), local_chains), dtype=torch.float64, device=dev)
        mon = np.asarray(sampled, dtype=np.int32)
        torch.cuda.current_stream(dev).synchronize()   # the library writes `block` on its own stream: torch's queued work goes first
        rc = L.amwg_sample_device(self._handle, n, thin, mon.ctypes.data_as(C.POINTER(C.c_int32)), len(sampled), block.data_ptr())
        if rc != 0:
            raise JsThrow(L.amwg_last_error().decode())
        reducer = CudaBlockReducer(self.device)
        loo_out = None
        if loo_plan is not None:
            loo_out = loo_block(reducer, CudaPointwise(self._handle, loo_prog, block, self.device), rows, n_chains, loo_plan.points,
                                loo_plan.r_eff, chunk_points, self.distributed)
        ppc_out = None
        if ppc_plan is not None:
            pit = None
            if ppc_plan.loo_pit is not None:
                pit = (CudaPointwise(self._handle, pit_prog, block, self.device), ppc_plan.loo_pit)
            ppc_out = ppc_block(reducer, CudaPpc(self._handle, ppc_prog, ppc_offs, ppc_code, block, ppc_plan.points), rows, n_chains,
                                ppc_plan.points, ppc_family, ppc_y, probs, ppc_chunk, self.distributed, loo_pit=pit)
        if len(sampled) > len(entries):
            block = block[:, :len(entries)].contiguous()
        res = summarise_block(reducer, block, rows, n_chains, probs, self.distributed, diagnostics)
        mean, sd, rhat, q = res[:4]
        hist = None if plan is None else histogram_block(reducer, block, rows, plan, self.distributed)
        cov = None if cov_plan is None else covariance_block(reducer, block, rows, cov_plan, self.distributed)
        rn = None if superchain is None else nested_block(reducer, block, rows, self.first_chain, superchain, self.distributed)
        mc = mcse_block(reducer, block, rows, n_chains, probs, mean, sd, q, self.distributed) if mcse else None
        del block
        out = {}
        for name in monitored:
            s0, ln = spans[name]
            if ln == 0:
                continue
            dim = list(self.params[name]["dim"]) if name in self.params else [1]
            shape = (lambda a: float(a[0])) if dim == [1] else (lambda a, dim=dim: np.asarray(a).reshape(*dim))
            out[name] = {"mean": shape(mean[s0:s0 + ln]), "sd": shape(sd[s0:s0 + ln]), "rhat": shape(rhat[s0:s0 + ln]),
                         "quantiles": q[:, s0] if dim == [1] else q[:, s0:s0 + ln].reshape(len(q), *dim),
                         "n_draws": rows * n_chains}
            if diagnostics:
                for key, val in res[4][0].items():
                    out[name][key] = shape(val[s0:s0 + ln])
            if hist is not None and plan.bins is not None:
                for key in ("hist", "hist_edges", "hist_outside"):
                    val = hist[key][s0:s0 + ln]
                    out[name][key] = val[0] if dim == [1] else val.reshape(*dim, val.shape[-1])
            if rn is not None:
                out[name]["rhat_nested"] = shape(rn[s0:s0 + ln])
            if mc is not None:
                for key in ("ess_quantile", "mcse_quantile"):
                    out[name][key] = mc[key][:, s0] if dim == [1] else mc[key][:, s0:s0 + ln].reshape(len(q), *dim)
                out[name]["mcse_sd"] = shape(mc["mcse_sd"][s0:s0 + ln])
        if hist is not None:
            out.update(hist["pairs"])
        if cov is not None:
            out["covariance"] = cov
        if loo_out is not None:
            out["loo"] = loo_out
        if ppc_out is not None:
            out["ppc"] = ppc_out
        return out

    def start_adaptation(self):
        """mcmc.js:1060-1064"""
        _ffi.check(_ffi.lib().amwg_set_adapting(self._handle, 1))

    def stop_adaptation(self):
        """mcmc.js:1069-1073"""
        _ffi.check(_ffi.lib().amwg_set_adapting(self._handle, 0))

    def info(self):
        """mcmc.js:977-980 + AmwgStepper.info (:906-912) + OnedimMetropolisStepper.info (:563-571).
        (The reference returns the thin/monitor *methods* under those keys -- a bug; the values are returned here.)"""
        L = _ffi.lib()
        scal = np.empty(self.n_comp * 3)
        pls = np.empty((self.n_comp, self.local_chains))
        acc = np.empty((self.n_comp, self.local_chains), dtype=np.int32)
        _ffi.check(L.amwg_info(self._handle, scal.ctypes.data, pls.ctypes.data, acc.ctypes.data))
        per_param = {}
        for name in self.param_names:
            p = self.params[name]
            if p["type"] == "binary":
                per_param[name] = {}                       # BinaryStepper inherits Stepper.info -> {} (mcmc.js:465-468)
                continue
            e = self._entries(name)
            dim = list(p["dim"])

            def per_chain(a, dim=dim):                     # a: [entries, chains]
                a = a[0] if dim == [1] else a.reshape(*dim, a.shape[-1])
                return a[..., 0] if self.n_chains == 1 else a

            def invariant(vals, dim=dim):
                return vals[0] if dim == [1] else np.asarray(vals).reshape(*dim)

            per_param[name] = {
                "prop_log_scale": per_chain(pls[e]),
                "is_adapting": invariant([bool(scal[c * 3]) for c in e]),
                "acceptance_count": per_chain(acc[e]),
                "iterations_since_adaption": invariant([scal[c * 3 + 1] for c in e]),
                "batch_count": invariant([scal[c * 3 + 2] for c in e]),
            }
        out = {"state": self.state, "thin": self.thinning_interval, "monitor": self.monitored_params,
               "steppers": [per_param]}
        if self.betas is not None:
            out["tempering"] = self._tempering_info()
        return out

    def _tempering_info(self) -> Dict[str, Any]:
        """options.temperatures: the swap rounds so far and, per rung pair (r, r + 1), the swaps accepted and attempted over this
        handle's ladders (round k attempts the pairs r = k mod 2)."""
        K = len(self.betas)
        rounds = C.c_uint64(0)
        acc = np.zeros(K - 1, dtype=np.int64)
        L = _ffi.lib()
        if L.amwg_ladder_info(self._handle, C.byref(rounds), acc.ctypes.data_as(C.POINTER(C.c_int64))) < 0:
            raise JsThrow(L.amwg_last_error().decode())
        k = int(rounds.value)
        ladders = self.local_chains // K
        att = np.asarray([ladders * ((k + 1 - (r & 1)) // 2) for r in range(K - 1)], dtype=np.int64)
        with np.errstate(invalid="ignore", divide="ignore"):
            rate = np.where(att > 0, acc / np.maximum(att, 1), np.nan)
        return {"temperatures": list(self.temperatures), "rounds": k, "swap_accepts": acc, "swap_attempts": att, "swap_rate": rate}

    # -- instrumentation (not in the reference) -------------------------------------------------------
    def kernel_launches(self) -> int:
        return int(_ffi.lib().amwg_kernel_launches(self._handle))

    def last_sweep_kernel_ms(self) -> float:
        return float(_ffi.lib().amwg_last_sweep_kernel_ms(self._handle))

    def program_summary(self) -> List[str]:
        return list(self._program.summary)

    def jit_status(self):
        """(active, note): does this handle step with a kernel specialised for its model at run time (csrc/amwg_jit.cuh)?"""
        if not getattr(self, "_handle", None):
            return False, "no device handle"
        buf = C.create_string_buffer(4096)
        on = _ffi.lib().amwg_jit_status(self._handle, buf, len(buf))
        return bool(on), buf.value.decode("utf-8", "replace")

    def plate_sources(self) -> List[str]:
        """Where the interpreter kernels (init, sweeps, the log_post() re-evaluation) read each plate's column, in plate order:
        "shared", "ring", "L2", or "loop" for a bytecode plate."""
        buf = C.create_string_buffer(4096)
        n = _ffi.lib().amwg_plate_sources(self._handle, buf, len(buf))
        return buf.value.decode().split(",") if n > 0 else []

    def _term_cache(self) -> np.ndarray:
        """The term cache as the sweep kernels left it, [n_terms, chains] (amwg_get_term_cache; [0, chains] without one). Slots below
        the program's n_sum_terms are terms of the sum, the rest plate statistics S, all at each chain's current state."""
        nt = int(self._program.n_terms)
        buf = np.empty((max(nt, 1), self.local_chains))
        L = _ffi.lib()
        got = L.amwg_get_term_cache(self._handle, buf.ctypes.data, buf.size)
        if got < 0:
            raise _ffi.AmwgError(L.amwg_last_error().decode("utf-8", "replace"))
        return buf[:got]

    def jit_compile_check(self, n_chains=None):
        """Generate and compile the specialised sweep of this model without running it (works without a GPU).
        -> (rc, message, source): rc 0 compiled, 1 model not eligible, -1 error."""
        log = C.create_string_buffer(1 << 16)
        src = C.create_string_buffer(1 << 20)
        m = self._model_keepalive[-1]
        rc = _ffi.lib().amwg_jit_compile_check(C.byref(m), int(n_chains or self.n_chains), log, len(log), src, len(src))
        return rc, log.value.decode("utf-8", "replace"), src.value.decode("utf-8", "replace")


class _PinnedPool:
    """Page-locked host buffers for sample(): pinning GBs costs more than the copy itself, so buffers are recycled once
    every array handed to the user (all views of the buffer) has been garbage collected."""

    def __init__(self):
        self._free: Dict[tuple, list] = {}

    def get(self, shape) -> np.ndarray:
        shape = tuple(int(v) for v in shape)
        try:
            import torch
            if not torch.cuda.is_available():
                raise RuntimeError
        except Exception:
            return np.empty(shape, dtype=np.float64)
        import weakref
        lst = self._free.get(shape)
        t = lst.pop() if lst else torch.empty(shape, dtype=torch.float64, pin_memory=True)
        a = t.numpy()
        weakref.finalize(a, self._put, shape, t)
        return a

    def _put(self, shape, t):
        lst = self._free.setdefault(shape, [])
        if len(lst) < 2:
            lst.append(t)


_PINNED = _PinnedPool()


def _pinned_empty(shape) -> np.ndarray:
    return _PINNED.get(shape)


# ------------------------------------------------------------------------------------------------
# stand-alone steppers -- mcmc.js:433-912 (the export list of mcmc.js:1103-1117)
# ------------------------------------------------------------------------------------------------
def _resolve_direct(params: Dict[str, dict], options: Optional[dict]) -> Dict[str, Dict[str, list]]:
    """Option handling of the stepper constructors themselves: get_option / get_multidim_option on `options`
    (mcmc.js:500-505, 644-649) -- no AmwgStepper merge."""
    out: Dict[str, Dict[str, list]] = {}
    for name, param in params.items():
        r: Dict[str, list] = {}
        if param["type"] != "binary":
            for key, default in _STEPPER_OPTIONS:
                if array_equal(param["dim"], [1]):
                    r[key] = [get_option(key, options, default)]
                else:
                    r[key] = _flatten(get_multidim_option(key, options, param["dim"], default))
        out[name] = r
    return out


def _set_nested(dst, src):
    """copy a nested array into an existing nested list IN PLACE (the reference's steppers mutate state[name][i]...)"""
    for i, v in enumerate(src):
        if isinstance(v, (list, np.ndarray)) and isinstance(dst[i], list):
            _set_nested(dst[i], v)
        else:
            dst[i] = float(v)


class _SteppedModel(AmwgSampler):
    """The device machinery of AmwgSampler behind a zero-argument `log_post` that closes over the caller's `state` object:
    the closure is recorded by temporarily putting symbolic values into `state`."""

    def __init__(self, params, state, log_post, options, direct_options: bool):
        self._user_state, self._zero_arg_log_post, self._direct = state, log_post, direct_options
        names = list(params.keys())

        def foreign(v, key):
            """numeric entries of `state` that belong to OTHER steppers: marked, so that a log_post that reads them is noticed"""
            if is_number(v):
                return Sym("FOREIGN", (), key)
            if isinstance(v, list):
                return [foreign(x, key) for x in v]
            return v

        def recorded(sym_state, _data):
            others = [k for k in list(state.keys()) if k not in names]
            saved = {n: state[n] for n in names + others}
            try:
                for n in names:
                    state[n] = sym_state[n]
                for k in others:
                    state[k] = foreign(saved[k], k)
                result = log_post()
            finally:
                for n in saved:
                    state[n] = saved[n]
            # The reference's steppers close over the LIVE state object (mcmc.js:433-437): a second stepper's updates are seen by
            # this one's log_post. Here log_post is recorded once, so a value owned by another stepper would be frozen into the
            # device program -- refuse instead of silently sampling the wrong conditional.
            stack, seen = [result] if isinstance(result, Sym) else [], 0
            while stack:
                node = stack.pop()
                if node.op == "FOREIGN":
                    raise JsThrow("log_post reads state." + str(node.val) + ", which this stepper does not step: composing several "
                                  "stand-alone steppers over one state object is not supported on the device; give one "
                                  "AmwgStepper / AmwgSampler all the parameters")
                stack.extend(node.args)
                seen += 1
            return result
        p = copy.deepcopy(params)
        for n in names:
            p[n]["init"] = copy.deepcopy(state[n])          # a stepper starts from the state it is given, not from params.init
        sampler_options = {k: v for k, v in (options or {}).items()}
        Sampler.__init__(self, p, recorded, None, sampler_options)

    def _resolve_options(self, params, options):
        stepper_options = {k: v for k, v in (options or {}).items() if k not in ("chains", "seed", "device", "first_chain", "faithful")}
        return _resolve_direct(params, stepper_options) if self._direct else resolve_stepper_options(params, stepper_options)

    def advance(self):
        """one step; writes the new values into the caller's state object (in place for arrays) and returns them by name"""
        self.burn(1)
        new = self.state
        for n in self.param_names:
            v = new[n]
            if isinstance(self._user_state[n], list):
                _set_nested(self._user_state[n], np.asarray(v).tolist())
            else:
                self._user_state[n] = v.tolist() if isinstance(v, np.ndarray) else float(v)
        return new


class Stepper:
    """mcmc.js:433-468 -- the Stepper "interface"."""

    def __init__(self, params, state, log_post):
        self.params, self.state, self.log_post = params, state, log_post

    def step(self):
        raise JsThrow("Every Stepper need to implement step()")

    def start_adaptation(self):
        pass

    def stop_adaptation(self):
        pass

    def info(self):
        return {}


class _DeviceStepper(Stepper):
    _type: Optional[str] = None        # proposal kind forced by the class (the reference's Real/Int steppers ignore params.type)
    _onedim = True
    _who = "Stepper"

    def __init__(self, params, state, log_post, options=None):
        super().__init__(params, state, log_post)
        names = list(params.keys())
        self._check(names, params)
        self.param_name = names[0] if len(names) == 1 else None
        p = complete_params(copy.deepcopy(params))
        if self._type is not None:
            for n in names:
                p[n]["type"] = self._type
                if self._type == "binary":
                    p[n]["lower"], p[n]["upper"] = 0, 1
        self._model = _SteppedModel(p, state, log_post, options, direct_options=self._who != "AmwgStepper")

    def _check(self, names, params):
        pass

    def step(self):
        new = self._model.advance()
        return self.state[self.param_name] if self.param_name is not None else self.state

    def start_adaptation(self):
        self._model.start_adaptation()

    def stop_adaptation(self):
        self._model.stop_adaptation()

    def _info_of(self, name):
        per = self._model.info()["steppers"][0][name]
        if not per:
            return {}
        dim = list(self._model.params[name]["dim"])
        if dim == [1]:
            return per
        keys = list(per.keys())                          # nested arrays of info objects (mcmc.js:698-702)
        flat = {k: np.asarray(per[k]).reshape(-1) for k in keys}
        objs = [{k: flat[k][c].item() for k in keys} for c in range(int(np.prod(dim)))]

        def nest(lst, d):
            if len(d) == 1:
                return lst
            step = len(lst) // d[0]
            return [nest(lst[i * step:(i + 1) * step], d[1:]) for i in range(d[0])]
        return nest(objs, dim)

    def info(self):
        return self._info_of(self.param_name)


class OnedimMetropolisStepper(_DeviceStepper):
    """mcmc.js:485-571"""
    _who = "OnedimMetropolisStepper"

    def _check(self, names, params):
        if len(names) != 1:
            raise JsThrow("OnedimMetropolisStepper can only handle one parameter.")
        dim = params[names[0]].get("dim", [1])
        if not array_equal([dim] if is_number(dim) else list(dim), [1]):
            raise JsThrow("OnedimMetropolisStepper can only handle one one-dimensional parameter.")


class RealMetropolisStepper(OnedimMetropolisStepper):
    """mcmc.js:586-591"""
    _type = "real"


class IntMetropolisStepper(OnedimMetropolisStepper):
    """mcmc.js:605-610"""
    _type = "int"


class MultidimComponentMetropolisStepper(_DeviceStepper):
    """mcmc.js:631-702"""
    _who = "MultidimComponentMetropolisStepper"

    def _check(self, names, params):
        if len(names) != 1:
            raise JsThrow("MultidimComponentMetropolisStepper can't handle more than one parameter.")


class MultiRealComponentMetropolisStepper(MultidimComponentMetropolisStepper):
    """mcmc.js:709-714"""
    _type = "real"


class MultiIntComponentMetropolisStepper(MultidimComponentMetropolisStepper):
    """mcmc.js:721-726"""
    _type = "int"


class BinaryStepper(_DeviceStepper):
    """mcmc.js:740-767"""
    _type = "binary"
    _who = "BinaryStepper"

    def _check(self, names, params):
        if len(names) != 1:
            raise JsThrow("BinaryStepper can't handle more than one parameter.")


class BinaryComponentStepper(_DeviceStepper):
    """mcmc.js:781-820"""
    _type = "binary"
    _who = "BinaryComponentStepper"

    def _check(self, names, params):
        if len(names) != 1:
            raise JsThrow("BinaryComponentStepper can't handle more than one parameter.")


class AmwgStepper(_DeviceStepper):
    """mcmc.js:837-912 -- any number of parameters; per-parameter option merge as in AmwgSampler."""
    _who = "AmwgStepper"

    def info(self):
        return {n: self._info_of(n) for n in self._model.param_names}
