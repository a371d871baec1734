"""The predictive-check samplers on the GPU across each family's domain: every point of the GRID of
tests/test_ppc_sampler_domain_host.py (algorithm switches on both sides, counts up to 1e18, binomial q down to 1e-15, shapes down to
1e-3, scales into the subnormals and past DBL_MAX) drawn by the device kernel for 1000 points x 1000 chains. At each point, 2000
of the 10^6 draws equal the restatement of tests/ppc_ref.py bit for bit, none is NaN, and the 10^6 draws pass the same checks as
the host's 10^5 (atoms by binomial tests, a chi-square against the law of the fp64-rounded variate, standardised mean and
variance), each at p > 1e-6."""
import numpy as np
import pytest

import ppc_ref
from test_gpu_summary_ppc import _replicated
from test_ppc_sampler_domain_host import GRID, _id, check_draws

pytestmark = pytest.mark.gpu

N = 1000
CHAINS = 1000
SEED = 2


@pytest.fixture(scope="module")
def sampler(gpu_pkg):
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    s = mcmc.AmwgSampler({"mu": {"type": "real"}}, lambda t, d: ld.norm(t.mu, 0, 1), {"y": [0.0] * N}, {"chains": CHAINS, "seed": SEED})
    s.burn(10)
    return s


@pytest.mark.parametrize("point", GRID, ids=_id)
def test_device_draws_across_the_domain(gpu_pkg, orc, sampler, point):
    fam, p = point
    O = orc.lib()
    call = getattr(gpu_pkg.ld, fam)
    _, yrep, _ = _replicated(sampler, lambda t, d, i: call(d.y[i], *p), N, 1)
    rng = np.random.default_rng(GRID.index(point))
    for _ in range(2000):
        c, i = int(rng.integers(CHAINS)), int(rng.integers(N))
        want, _ = ppc_ref.draw_at(O, fam, p, SEED, c, 0, N, i)
        assert np.float64(yrep[0, i, c]).tobytes() == np.float64(want).tobytes(), (fam, p, c, i, yrep[0, i, c], want)
    x = yrep.ravel()
    assert x.size == N * CHAINS
    check_draws(x, fam, p)
