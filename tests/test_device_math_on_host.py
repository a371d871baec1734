"""The product's device arithmetic, compiled for the HOST, against the oracle -- without a GPU.

csrc/amwg_math.cuh (Math.log / Math.exp as fdlibm, Math.round, the Philox "Math.random()" stream, rnorm of mcmc.js:43-54) and
csrc/amwg_ld.cuh (every scalar ld.* of distributions.js:63-284) are the files nvcc and NVRTC compile for sm_90a. Here g++ compiles the
same text (tests/host_shim supplies the five CUDA intrinsics they use; -ffp-contract=off matches --fmad=false) and the results are
held against the C oracle bit for bit on the inputs tests/test_gpu_parity.py uses on the GPU. What this adds to the GPU tests: an edit
to either header is caught by the CPU suite; what it cannot show: that the GPU's own sqrt / division / pow round like the host's
(they are IEEE-correct for sqrt and division; pow is compared to a few ulp on the GPU side)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("devmath") / "libdevmath_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", "device_math_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    d = C.c_double
    for name, n in (("js_log", 1), ("js_exp", 1), ("js_round", 1), ("js_max", 2), ("js_min", 2), ("lgamma", 1), ("lfactorial", 1), ("lchoose", 2),
                    ("lbeta", 2), ("beta", 3), ("cauchy", 3), ("norm", 3), ("laplace", 3), ("gamma", 3), ("invgamma", 3), ("lnorm", 3), ("pareto", 3),
                    ("t", 4), ("weibull", 3), ("logis", 3), ("exp", 2), ("unif", 3), ("bern", 2), ("binom", 3), ("nbinom", 3), ("hyper", 4), ("pois", 2)):
        f = getattr(lib, "hs_" + name)
        f.restype, f.argtypes = d, [d] * n
    lib.hs_uniform.restype, lib.hs_uniform.argtypes = d, [C.c_uint64] * 3
    lib.hs_rnorm.restype, lib.hs_rnorm.argtypes = d, [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), d, d]
    return lib


def _same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def test_log_exp_round_random_stream_and_rnorm(H, orc):
    O = orc.lib()
    rng = np.random.default_rng(0)
    x = np.concatenate([np.exp(rng.uniform(-700, 700, 60000)), rng.uniform(1e-3, 10, 60000),
                        [0.0, -0.0, -1.0, np.inf, -np.inf, 1.0, 5e-324, 2.2250738585072014e-308, np.nan]])
    assert _same_bits([H.hs_js_log(v) for v in x], [O.orc_log(v) for v in x])
    x = np.concatenate([rng.uniform(-745, 710, 60000), rng.uniform(-5, 5, 60000), [0.0, -np.inf, np.inf, 709.9, -745.2, 1e-10, np.nan]])
    assert _same_bits([H.hs_js_exp(v) for v in x], [O.orc_exp(v) for v in x])
    x = np.concatenate([rng.uniform(-10, 10, 10000), [-2.5, 2.5, 0.5, -0.5, 0.49999999999999994, -0.0, 1e300, np.nan, np.inf]])
    assert _same_bits([H.hs_js_round(v) for v in x], [O.orc_js_round(v) for v in x])
    # Math.max / Math.min propagate NaN (ADVICE r1): the device helpers against numpy's NaN-propagating pair
    for a, b in ((1.0, 2.0), (2.0, 1.0), (np.nan, 1.0), (1.0, np.nan), (-0.0, 0.0), (np.inf, -np.inf)):
        assert _same_bits([H.hs_js_max(a, b)], [np.maximum(a, b)]) or (a == b)
        assert _same_bits([H.hs_js_min(a, b)], [np.minimum(a, b)]) or (a == b)
    # the Math.random() stream: uniform #n of (seed, chain), chain ids and positions beyond 32 bits
    for seed, chain in ((12345, 77), (0, 0), (2**40 + 3, 2**35 + 1), (2**64 - 1, 2**22 - 1)):
        ns = list(range(0, 300)) + [2**32 - 1, 2**32, 2**32 + 1, 2**45 + 7]
        assert _same_bits([H.hs_uniform(seed, chain, n) for n in ns], [O.orc_stream_uniform(seed, chain, n) for n in ns])
    # rnorm (Leva): values AND the number of uniforms each call consumes, from an even and an odd stream position
    for start in (0, 7):
        ph, po = C.c_uint64(start), C.c_uint64(start)
        for _ in range(5000):
            a, b = H.hs_rnorm(9, 3, C.byref(ph), 10.0, 5.0), O.orc_rnorm(9, 3, C.byref(po), 10.0, 5.0)
            assert a == b and ph.value == po.value


def test_every_scalar_ld_function(H, orc):
    O = orc.lib()
    rng = np.random.default_rng(1)
    n = 5000
    ints = lambda lo, hi: rng.integers(lo, hi, n).astype(float)
    cases = {
        "norm": (rng.normal(0, 50, n), rng.normal(0, 50, n), rng.uniform(0.01, 100, n)),
        "unif": (rng.uniform(-1, 2, n), np.zeros(n), np.ones(n)),
        "beta": (rng.uniform(-0.1, 1.1, n), rng.uniform(0.5, 5, n), rng.uniform(0.5, 5, n)),
        "bern": (ints(0, 3), rng.uniform(0, 1, n)),
        "pois": (ints(-1, 50), rng.uniform(0.01, 40, n)),
        "lgamma": (rng.uniform(0.01, 200, n),),
        "lfactorial": (ints(-1, 100),),
        "lchoose": (ints(1, 60), ints(0, 30)),
        "lbeta": (rng.uniform(0.1, 30, n), rng.uniform(0.1, 30, n)),
        "cauchy": (rng.normal(0, 5, n), rng.normal(0, 5, n), rng.uniform(0.1, 5, n)),
        "laplace": (rng.normal(0, 5, n), rng.normal(0, 5, n), rng.uniform(0.1, 5, n)),
        "gamma": (rng.uniform(-0.5, 20, n), rng.uniform(0.2, 9, n), rng.uniform(0.2, 9, n)),
        "invgamma": (rng.uniform(-0.5, 20, n), rng.uniform(0.2, 9, n), rng.uniform(0.2, 9, n)),
        "lnorm": (rng.uniform(-0.5, 20, n), rng.normal(0, 2, n), rng.uniform(0.2, 3, n)),
        "pareto": (rng.uniform(0.1, 20, n), rng.uniform(0.2, 9, n), rng.uniform(0.2, 9, n)),
        "logis": (rng.normal(0, 5, n), rng.normal(0, 5, n), rng.uniform(0.1, 5, n)),
        "exp": (rng.uniform(-0.5, 20, n), rng.uniform(0.1, 5, n)),
        "binom": (ints(-1, 30), ints(1, 30), rng.uniform(0, 1, n)),
        "nbinom": (ints(-1, 30), ints(1, 30), rng.uniform(0.01, 0.99, n)),
        "hyper": (ints(0, 10), ints(10, 30), ints(10, 30), ints(5, 10)),
        # Math.pow with a non-integer exponent: the same libm pow on both sides here (on the GPU: CUDA's pow, compared to a few ulp)
        "t": (rng.normal(0, 5, n), rng.normal(0, 5, n), rng.uniform(0.1, 5, n), rng.uniform(0.5, 30, n)),
        "weibull": (rng.uniform(-0.5, 20, n), rng.uniform(0.2, 9, n), rng.uniform(0.2, 9, n)),
    }
    for name, args in cases.items():
        f, g = getattr(H, "hs_" + name), getattr(O, "orc_ld_" + name)
        g.restype, g.argtypes = C.c_double, [C.c_double] * len(args)
        got = [f(*[float(a[i]) for a in args]) for i in range(n)]
        ref = [g(*[float(a[i]) for a in args]) for i in range(n)]
        assert _same_bits(got, ref), name
