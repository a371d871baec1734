"""Nested R-hat and superchain starting points on the GPU: amwg_summary_nested against the fsum restatement within its derived
bound (tests/nested_ref.py), the same bits on a repeated call, NaN propagation and every refused argument; superchains that start
at one point under options.init_radius, whichever handles hold them, in the Python and the JavaScript host; twin handles whose
every other summary key keeps its bits; and the statistic on a converged ensemble of short chains and on two modes."""
import ctypes as C

import numpy as np
import pytest

import models
import nested_ref
from conftest import config2_data

pytestmark = pytest.mark.gpu


def _block(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


@pytest.mark.parametrize("M, rows, chains, first", [(1, 3, 1000, 0), (3, 5, 1001, 2), (16, 2, 1000, 7), (16, 1, 999, 0),
                                                     (256, 2, 1300, 100), (256, 4, 768, 0)])
def test_reducer_matches_the_definition(gpu_pkg, M, rows, chains, first):
    from bayes_js_b200.summary import CudaBlockReducer, finalize_nested, merge_nested_records
    rng = np.random.default_rng(M + rows + chains)
    x = 1e6 * (M == 16) + rng.normal(size=(rows, 3, chains)) * [[[1.0], [3.0], [0.1]]] + rng.normal(size=(1, 1, chains)) * 0.2
    red = CudaBlockReducer(0)
    blk = _block(x)
    got = red.nested(blk, first, M)
    exact, bound = nested_ref.check_record(got, x, first, M, (M, rows, chains, first))
    assert red.nested(blk, first, M).tobytes() == got.tobytes()                     # same bits on a repeated call
    if first % M == 0 and chains % M == 0:
        rh = finalize_nested(merge_nested_records([got], M, rows))
        lo, hi = nested_ref.rhat_interval(exact[:, :4], bound[:, :4])
        assert np.all((lo <= rh) & (rh <= hi)), (rh, lo, hi)


def test_reducer_propagates_nan_and_inf(gpu_pkg):
    from bayes_js_b200.summary import CudaBlockReducer, finalize_nested, merge_nested_records
    x = np.random.default_rng(5).normal(size=(4, 3, 96))
    x[2, 1, 40] = np.nan
    x[0, 2, 7] = np.inf
    got = CudaBlockReducer(0).nested(_block(x), 0, 8)
    assert np.isnan(got[1, 1:4]).any() and not np.isfinite(got[2, 1:4]).all() and np.isfinite(got[0, :4]).all()
    rh = finalize_nested(merge_nested_records([got], 8, 4))
    assert np.isfinite(rh[0]) and np.isnan(rh[1]) and np.isnan(rh[2])


def test_refused_abi_arguments(gpu_pkg):
    L = gpu_pkg._ffi.lib()
    blk = _block(np.zeros((3, 5, 7)))
    p = blk.data_ptr()
    o = np.empty(5 * 14).ctypes.data
    for args, msg in (((0, p, 0, 5, 7, 0, 1, o), b"empty sample block"), ((0, p, 3, 0, 7, 0, 1, o), b"empty sample block"),
                      ((0, p, 3, 5, 0, 0, 1, o), b"empty sample block"), ((0, None, 3, 5, 7, 0, 1, o), b"null pointer"),
                      ((0, p, 3, 5, 7, 0, 1, None), b"null pointer"), ((0, p, 3, 5, 7, 0, 0, o), b"superchain_size must be >= 1"),
                      ((0, p, 3, 5, 7, -1, 2, o), b"first_chain must be >= 0"),
                      ((0, p, 3, 5, 7, 2**53 - 6, 2, o), b"first_chain + chains must be at most 2^53"),
                      ((64, p, 3, 5, 7, 0, 1, o), b"device index out of range")):
        assert L.amwg_summary_nested(*args) != 0 and msg in L.amwg_last_error(), args
    assert L.amwg_summary_nested(0, p, 3, 5, 7, 2**53 - 7, 2, o) == 0
    # the dispersal refuses a superchain size below 1 before anything changes
    s = gpu_pkg.mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(gpu_pkg.ld), config2_data().tolist(), {"chains": 32, "seed": 3})
    before = s.state
    failed = C.c_int64(0)
    assert L.amwg_disperse_state_superchains(s._handle, 2.0, 0, C.byref(failed)) != 0
    assert b"amwg_disperse_state: superchain_size must be >= 1" in L.amwg_last_error()
    for k in before:
        assert np.asarray(before[k]).tobytes() == np.asarray(s.state[k]).tobytes()
    s.close()


def _sampler(gpu_pkg, chains, **opts):
    return gpu_pkg.mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(gpu_pkg.ld), config2_data().tolist(),
                                    dict({"chains": chains, "seed": 12}, **opts))


def _state(s):
    st = s.state
    return np.stack([np.asarray(st["mu"], np.float64), np.asarray(st["sigma"], np.float64)])


def test_superchains_start_together_and_apart(gpu_pkg):
    M, Cn = 16, 1024
    s = _sampler(gpu_pkg, Cn, init_radius=2, superchain_size=M)
    x = _state(s).reshape(2, Cn // M, M)
    assert np.array_equal(x.view(np.uint64), np.repeat(x[:, :, :1], M, axis=2).view(np.uint64))      # bit-identical in a superchain
    lead = x[0, :, 0]
    assert len(np.unique(lead)) == Cn // M                                                           # distinct superchains
    s.close()
    # M = 1 is the dispersal without superchains, byte for byte
    a, b = _sampler(gpu_pkg, Cn, init_radius=2, superchain_size=1), _sampler(gpu_pkg, Cn, init_radius=2)
    assert _state(a).tobytes() == _state(b).tobytes()
    a.close(); b.close()


def test_handles_that_cut_a_superchain_disperse_like_one(gpu_pkg):
    L = gpu_pkg._ffi.lib()
    M = 16
    one = _state(_sampler(gpu_pkg, 64, init_radius=2, superchain_size=M))
    parts = []
    for first, n in ((0, 40), (40, 24)):                       # 40 cuts superchain 2
        s = _sampler(gpu_pkg, n, first_chain=first)
        failed = C.c_int64(0)
        assert L.amwg_disperse_state_superchains(s._handle, 2.0, M, C.byref(failed)) == 0
        parts.append(_state(s))
        s.close()
    assert np.concatenate(parts, axis=1).tobytes() == one.tobytes()


def test_javascript_host_gives_the_python_hosts_bits(gpu_pkg):
    from js_host import JsHost, to_py
    from js_native_inits import InitsDeviceNative
    from oracle.minijs.minijs import to_js

    class SuperchainNative(InitsDeviceNative):
        """disperse_state(handle, radius[, superchain_size]) as js/amwg_napi.cc binds it"""

        def __call__(self, host):
            o = super().__call__(host)
            L = self.pkg._ffi.lib()

            def disperse_state(this, a):
                failed = C.c_int64(0)
                if len(a) > 2:
                    rc = L.amwg_disperse_state_superchains(self.handles[a[0]], float(a[1]), int(a[2]), C.byref(failed))
                else:
                    rc = L.amwg_disperse_state(self.handles[a[0]], float(a[1]), C.byref(failed))
                if rc != 0 and failed.value == 0:
                    self._fail()
                return float(failed.value)
            o.put("disperse_state", host.it.make_native("disperse_state", disperse_state))
            return o

    h = JsHost(native=SuperchainNative(gpu_pkg))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.it.set_global("ld", h.load("distributions"))
    h.run("""
var readme_norm_post = function(state, data) {
  var log_post = 0;
  log_post += ld.norm(state.mu, 0, 100);
  log_post += ld.unif(state.sigma, 0, 100);
  for(var i = 0; i < data.length; i++) {
    log_post += ld.norm(data[i], state.mu, state.sigma);
  }
  return log_post;
};""")
    h.it.set_global("the_data", to_js(h.it, [float(v) for v in config2_data()]))
    h.run("""
      var T = new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, readme_norm_post, the_data,
                                   {chains: 256, seed: 12, init_radius: 2, superchain_size: 8});
      var t0 = T.state();
      T.close();
    """)
    js = to_py(h.get("t0"))
    py = _sampler(gpu_pkg, 256, init_radius=2, superchain_size=8).state
    for k in ("mu", "sigma"):
        assert np.asarray(js[k], np.float64).tobytes() == np.asarray(py[k], np.float64).tobytes(), k


def test_twins_keep_every_other_key_and_the_chains(gpu_pkg):
    hist = {"bins": 20, "pairs": [("mu", "sigma")]}
    a, b = (_sampler(gpu_pkg, 4096, init_radius=2, superchain_size=16) for _ in range(2))
    for s in (a, b):
        s.burn(300)
    got = a.sample_summary(100, diagnostics="rank", histogram=hist, covariance=True, nested=16)
    base = b.sample_summary(100, diagnostics="rank", histogram=hist, covariance=True)
    assert set(got) == set(base)
    for name in base:
        extra = {"rhat_nested"} if name in ("mu", "sigma") else set()
        assert set(got[name]) == set(base[name]) | extra, name
        for key, val in base[name].items():
            if isinstance(val, (list, tuple)):
                val, gv = repr(val), repr(got[name][key])
                assert gv == val, (name, key)
            else:
                assert np.asarray(got[name][key]).tobytes() == np.asarray(val).tobytes(), (name, key)
    assert np.isfinite(got["mu"]["rhat_nested"]) and np.isfinite(got["sigma"]["rhat_nested"])
    assert _state(a).tobytes() == _state(b).tobytes()
    a.close(); b.close()


def test_converged_short_chains(gpu_pkg):
    """2^16 chains in 1024 superchains of 64, one kept row after burn(1000): rhat is not defined (NaN) and rhat_nested is the
    value for independent stationary draws, sqrt(1 + 1/M) = 1.00778; its sampling sd is about 0.0004 here (B^ has K - 1 = 1023
    degrees of freedom), so the test allows 0.003. One H100 run gave 1.00765 (mu) and 1.00796 (sigma)."""
    s = _sampler(gpu_pkg, 1 << 16, init_radius=2, superchain_size=64)
    s.burn(1000)
    out = s.sample_summary(1, nested=True)
    print("converged rhat_nested", out["mu"]["rhat_nested"], out["sigma"]["rhat_nested"])
    for k in ("mu", "sigma"):
        assert np.isnan(out[k]["rhat"])
        assert abs(out[k]["rhat_nested"] - np.sqrt(1 + 1 / 64)) < 0.003, (k, out[k]["rhat_nested"])
    s.close()


def test_two_modes_are_flagged(gpu_pkg):
    """The two modes of test_dispersal_exposes_a_mode_identical_starts_hide: superchains that start in the other mode stay there, so
    the superchain means disagree by about 20 against a variance of about 1 inside the superchains. One H100 run gave 3.49; the
    test asks for more than 2."""
    ld, mcmc = gpu_pkg.ld, gpu_pkg.mcmc

    def f(state, data):
        return mcmc.Math.log(0.5 * mcmc.Math.exp(ld.norm(state.x, -10, 1)) + 0.5 * mcmc.Math.exp(ld.norm(state.x, 10, 1)))
    s = mcmc.AmwgSampler({"x": {"type": "real", "init": 10}}, f, None, {"chains": 1 << 14, "seed": 2, "init_radius": 20, "superchain_size": 64})
    s.burn(500)
    out = s.sample_summary(10, nested=64)
    print("two modes rhat_nested", out["x"]["rhat_nested"])
    assert out["x"]["rhat_nested"] > 2.0, out["x"]["rhat_nested"]
    s.close()
