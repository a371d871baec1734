import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import __graft_entry__ as graft  # noqa: E402

graft.load_package()          # registers `bayes_js_b200` (the directory name bayes.js_b200 is not an identifier)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def pkg():
    return graft.load_package()


@pytest.fixture(scope="session")
def orc():
    return graft.load_oracle()


@pytest.fixture(scope="session")
def gpu_pkg(pkg):
    """The package with the CUDA library loaded; GPU tests fail loudly if the extension is missing."""
    lib = pkg._ffi.lib()
    assert lib.amwg_abi_version() == 8
    return pkg


# ---- the reference's fixtures, tests/test_data.js -------------------------------------------------------------
PRESIDENTS = [183, 192, 182, 183, 177, 185, 188, 188, 182, 185]            # README.md:20
NORM_DATA = [100, 62, 96, 122, 141, 144, 74, 73, 78, 128]                  # tests/test_data.js:77


def config2_data():
    """BASELINE config 2: N=1024 synthetic Normal data."""
    return np.random.default_rng(1024).normal(184.5, 4.5, 1024)


def config3_data():
    """BASELINE config 3: N=256 Bernoulli(0.7) data."""
    return (np.random.default_rng(256).random(256) < 0.7).astype(np.float64)
