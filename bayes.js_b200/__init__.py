"""bayes.js_b200 -- H100-native many-chain AMWG sampler behind the bayes.js API.

    from bayes_js_b200 import mcmc, ld          (see __graft_entry__.load_package for the import shim:
                                                 the directory name `bayes.js_b200` is not a Python identifier)
    sampler = mcmc.AmwgSampler(params, log_post, data, {"chains": 1 << 20, "seed": 0})
    sampler.burn(1000); draws = sampler.sample(1000)

`mcmc` mirrors /root/reference/mcmc.js, `ld` mirrors /root/reference/distributions.js; the hot path runs in
libamwg_b200.so (csrc/, C ABI in include/amwg.h).  There is no CPU fallback.
"""
from . import _ffi, mcmc, parallel, summary, tracer   # noqa: F401
from . import distributions as ld           # noqa: F401
from .tracer import JsThrow                 # noqa: F401

__all__ = ["mcmc", "ld", "JsThrow"]
