"""Restatement of the over-dispersed starting points of amwg_disperse_state (DESIGN.md §2 "Dispersed starting points") over the
oracle's primitives: its Philox stream (orc_stream_uniform), Math.log / Math.exp (orc_log, orc_exp) and Math.round (orc_js_round).
Python floats are IEEE-754 doubles and every operation below is one rounding, as on the device."""
import math

import numpy as np

ATTEMPTS = 100
STREAM_BASE = 1 << 63
REAL, INT, BINARY = 0, 1, 2


def uniform(O, seed, chain, attempt, n_comp, c):
    """uniform #(2^63 + attempt*n_comp + c) of global chain `chain`"""
    return O.orc_stream_uniform(seed, chain, STREAM_BASE + attempt * n_comp + c)


def component(O, typ, lower, upper, init, radius, U):
    """(value, valid) of one component for the uniform U"""
    if typ == BINARY:
        return (0.0 if U < 0.5 else 1.0), True
    lo, hi = lower != -math.inf, upper != math.inf
    if lo and hi:
        z0 = O.orc_log(init - lower) - O.orc_log(upper - init)
    elif lo:
        z0 = O.orc_log(init - lower)
    elif hi:
        z0 = O.orc_log(upper - init)
    else:
        z0 = init
    if not math.isfinite(z0):
        z0 = 0.0
    z = z0 + (2.0 * U - 1.0) * radius
    if lo and hi:
        x = lower + (upper - lower) / (1.0 + O.orc_exp(-z))
    elif lo:
        x = lower + O.orc_exp(z)
    elif hi:
        x = upper - O.orc_exp(z)
    else:
        x = z
    if typ == INT:
        x = O.orc_js_round(x)
    return x, lower <= x <= upper


def comps_of(sampler):
    """[(type, lower, upper, init)] per flat component of an AmwgSampler, in the device's order"""
    code = {"real": REAL, "int": INT, "binary": BINARY}
    out = []
    for name in sampler.param_names:
        p = sampler.params[name]
        flat = np.asarray(p["init"], dtype=np.float64).reshape(-1)
        out += [(code[p["type"]], float(p["lower"]), float(p["upper"]), float(v)) for v in flat]
    return out


def disperse_chain(O, seed, chain, comps, radius, finite_log_post):
    """The point chain `chain` keeps and the attempt it came from; (None, ATTEMPTS) when no attempt succeeds.
    finite_log_post(x) says whether log_post is finite at the flat state x."""
    for a in range(ATTEMPTS):
        xs, ok = [], True
        for c, (t, lo, hi, init) in enumerate(comps):
            x, v = component(O, t, lo, hi, init, radius, uniform(O, seed, chain, a, len(comps), c))
            xs.append(x)
            ok = ok and v
        if ok and finite_log_post(xs):
            return xs, a
    return None, ATTEMPTS
