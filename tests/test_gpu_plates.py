"""The factorised likelihood plates on the GPU, for their value: the carried log_post of every chain of an interpreter handle (what
the init kernel and the sweep kernels computed at each chain's accepted proposal) against the extended-precision reference of
tests/plate_ref.py at the chain's state, within the worst-case bound of the kernel's fp64 operations. Straight after construction,
after one sweep and after twenty more. Every Poisson instance K runs on each data path (resident in shared memory, the TMA tile
ring, global/L2), and every case asserts the path it took (AmwgSampler.plate_sources, which reports the kernels' own choice)."""
import os
from contextlib import contextmanager

import numpy as np
import pytest

import plate_ref as pr
from plate_ref import edge_data, pois_data, ragged_groups

pytestmark = pytest.mark.gpu

BUDGET = 200 * 1024                     # csrc kSmemBudget: data bytes a CTA stages in shared memory
RING_STAGE = 16 * 1024                  # csrc kRingStageBytes: one tile of the ring
POIS_K = (1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 16)


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def at_checkpoints(s, check):
    """after construction (the init kernel), after one sweep and after twenty more"""
    check(s, "init")
    s.burn(1)
    check(s, "burn 1")
    s.burn(20)
    check(s, "burn 21")


# ---- Poisson regression (BASELINE config 5) --------------------------------------------------------------------------------
def pois_post(ld, mcmc, K, tau=False):
    def f(state, d):
        lp = 0
        beta = [state.beta] if K == 1 else [state.beta[k] for k in range(K)]
        for k in range(K):
            lp += ld.norm(beta[k], 0, 10)
        if tau:
            lp += ld.norm(state.tau, 0, 1)
        for i in mcmc.points(len(d.y)):
            eta = 0
            for k in range(K):
                eta += d.X[i][k] * beta[k]
            lp += ld.pois(d.y[i], mcmc.Math.exp(eta))
        return lp
    return f


def pois_sampler(pkg, y, X, chains, seed, init=None, tau=False, faithful=False):
    K = X.shape[1]
    params = {"beta": {"type": "real", "dim": [K]}}
    if init is not None:
        params["beta"]["init"] = init[0] if K == 1 else list(init)
    if tau:
        params["tau"] = {"type": "real"}
    s = pkg.mcmc.AmwgSampler(params, pois_post(pkg.ld, pkg.mcmc, K, tau), {"y": y.tolist(), "X": X.tolist()},
                             {"chains": chains, "seed": seed, "faithful": faithful})
    if not faithful:
        assert f"plate POIS_LOGLIN n={y.size} K={K}" in s.program_summary()
    return s


def pois_check(orc, y, X, partials, tau=False):
    K = X.shape[1]

    def check(s, what):
        st = s.state
        C = s.n_chains
        cols = [np.asarray(st["beta"], np.float64).reshape(C, K)]
        if tau:
            cols.append(np.asarray(st["tau"], np.float64).reshape(C, 1))
        S = np.concatenate(cols, axis=1)

        def ref(u):
            terms = [pr.norm_term(u[:, k], 0.0, 10.0) for k in range(K)]
            if tau:
                terms.append(pr.norm_term(u[:, K], 0.0, 1.0))
            return pr.combine(terms + [pr.pois_loglin(orc, y, X, u[:, :K], partials)])
        pr.per_state(ref, S).check(s.log_post(), f"K={K} {what}")
    return check


def ring_rows(K):
    """X above the staging budget (so the ring, or L2 without it), >= 3 tiles, n mod (rows per tile) != 0 and n mod 8 != 0"""
    R = (RING_STAGE // (8 * K)) & ~1
    n = BUDGET // (8 * K) + 37
    while n % 8 == 0 or n % R == 0:
        n += 1
    assert 8 * n * K > BUDGET and n >= 3 * R
    return n


@pytest.mark.parametrize("K", POIS_K)
def test_poisson_plate_every_k_on_every_path(gpu_pkg, orc, K):
    pr.require_extended()
    chains = 33 if POIS_K.index(K) % 2 == 0 else 200
    # resident: the 4-row blocks (K <= 8) or 2-row blocks, and sizes below them
    for n in (1, 3, 1003):
        y, X = pois_data(K, n, 100 + K)
        if n < 4:
            y = np.maximum(y, 1.0)          # y >= 1 keeps exp(eta), what a lone row adds, near y at the chains' states
        assert 8 * n * (K + 1) < BUDGET
        s = pois_sampler(gpu_pkg, y, X, chains, seed=K)
        assert s.plate_sources() == ["shared"]
        at_checkpoints(s, pois_check(orc, y, X, partials=2))
    n = ring_rows(K)
    y, X = pois_data(K, n, 200 + K)
    s = pois_sampler(gpu_pkg, y, X, chains, seed=K)
    assert s.plate_sources() == ["ring"]
    at_checkpoints(s, pois_check(orc, y, X, partials=8 if K == 8 else 2))          # K = 8: DMMA.8x8x4 on the ring
    with env(AMWG_PHASE_SYNC="0"):                                                   # no CTA-uniform steps: no ring
        s = pois_sampler(gpu_pkg, y, X, chains, seed=K)
    assert s.plate_sources() == ["L2"]
    at_checkpoints(s, pois_check(orc, y, X, partials=2))


def test_poisson_plate_with_a_second_parameter(gpu_pkg, orc):
    """beta[K] + a scalar tau. K = 3: the vector parameter makes the steps non-uniform across chains, so X comes from L2 without any
    switch. K = 1: two scalar components, log_post is evaluated per component from the term cache, and a step on tau adds the
    plate's cached value instead of recomputing it."""
    y, X = pois_data(3, ring_rows(3), 7)
    s = pois_sampler(gpu_pkg, y, X, 200, seed=1, tau=True)
    assert s.plate_sources() == ["L2"]
    at_checkpoints(s, pois_check(orc, y, X, partials=2, tau=True))
    y, X = pois_data(1, 2001, 8)
    s = pois_sampler(gpu_pkg, y, X, 33, seed=2, tau=True)
    assert s.plate_sources() == ["shared"]
    assert any(x.startswith("dependency-aware evaluation") for x in s.program_summary())
    at_checkpoints(s, pois_check(orc, y, X, partials=2, tau=True))


def test_poisson_dmma_with_partial_warps_and_shadow_lanes(gpu_pkg, orc):
    """K = 8 on the ring with 4096 + 37 chains: the last CTA has a partial warp and shadow threads that take part in the ring"""
    K = 8
    n = ring_rows(K)
    y, X = pois_data(K, n, 9)
    with env(AMWG_JIT="0"):
        s = pois_sampler(gpu_pkg, y, X, 4096 + 37, seed=3)
    assert s.plate_sources() == ["ring"]
    at_checkpoints(s, pois_check(orc, y, X, partials=8))


@pytest.mark.parametrize("kind", ["mixed", "high"])
def test_poisson_plate_edges_of_exp(gpu_pkg, orc, kind):
    """On the register path (resident, L2) and the DMMA path (ring). The plate agrees with the exact value where exp underflows with
    y > 0 (the reference's loop gives -Infinity there: DESIGN.md section 2)."""
    init = [1.0] + [0.0] * 7
    for path, n, envs in (("shared", 1003, {}), ("ring", ring_rows(8), {}), ("L2", ring_rows(8), {"AMWG_PHASE_SYNC": "0"})):
        y, X = edge_data(n, 11, kind)
        with env(**envs):
            s = pois_sampler(gpu_pkg, y, X, 200, seed=4, init=init)
        assert s.plate_sources() == [path]
        eta0 = X @ np.array(init)
        if kind == "high":
            assert np.all((eta0 > 690) & (eta0 < 709))
        else:
            assert np.sum((eta0 < -745) & (y > 0)) == 5 and np.sum(y == 0) >= 35 and np.sum(y > 9000) >= 30
        at_checkpoints(s, pois_check(orc, y, X, partials=8 if path == "ring" else 2))


def test_poisson_plate_exp_overflow_and_negative_counts(gpu_pkg, orc):
    """One row with eta > 709.8: exp overflows, the plate gives -Infinity (the reference's loop: NaN, log(Infinity) * y - Infinity;
    DESIGN.md section 2). A negative count: ld.pois is -Infinity (distributions.js:282-284); the model keeps the term-by-term loop and
    agrees with a faithful handle."""
    init = [1.0] + [0.0] * 7
    for path, n, envs in (("shared", 1003, {}), ("ring", ring_rows(8), {})):
        y, X = edge_data(n, 12, "mixed")
        X[n // 2, 0] = 712.0
        with env(**envs):
            s = pois_sampler(gpu_pkg, y, X, 33, seed=5, init=init)
        assert s.plate_sources() == [path]
        assert np.all(s.log_post() == -np.inf), path
        f = pois_sampler(gpu_pkg, y, X, 33, seed=5, init=init, faithful=True)
        assert np.all(np.isnan(f.log_post())), path
    y, X = pois_data(2, 300, 13)
    y[17] = -1.0
    params = {"beta": {"type": "real", "dim": [2]}}
    data = {"y": y.tolist(), "X": X.tolist()}
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    s = mcmc.AmwgSampler(params, pois_post(ld, mcmc, 2), data, {"chains": 33, "seed": 6})
    f = mcmc.AmwgSampler(params, pois_post(ld, mcmc, 2), data, {"chains": 33, "seed": 6, "faithful": True})
    assert s.program_summary()[-1] == "plate GENERIC n=300 body=LD_POIS" and s.plate_sources() == ["loop"]
    for what in ("init", "burn"):
        assert np.all(s.log_post() == -np.inf) and np.array_equal(s.log_post(), f.log_post()), what
        s.burn(5)
        f.burn(5)


# ---- Normal plates ------------------------------------------------------------------------------------------------------------
PARAMS_NORM = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}


def norm_points(ld, mcmc, m0=0.0, s0=100.0):
    def f(state, d):
        lp = 0
        lp += ld.norm(state.mu, m0, s0)
        lp += ld.unif(state.sigma, 0, 100)
        for i in mcmc.points(len(d)):
            lp += ld.norm(d[i], state.mu, state.sigma)
        return lp
    return f


def norm_split(ld, k):
    """one column, two plates: [0, k) and [k, n), the priors between them (so the loops are not merged into one plate)"""
    def f(state, d):
        lp = 0
        for i in range(k):
            lp += ld.norm(d[i], state.mu, state.sigma)
        lp += ld.norm(state.mu, 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in range(k, len(d)):
            lp += ld.norm(d[i], state.mu, state.sigma)
        return lp
    return f


def norm_check(x, m0=0.0, s0=100.0, split=None):
    def check(s, what):
        st = s.state
        S = np.column_stack([np.asarray(st["mu"], np.float64), np.asarray(st["sigma"], np.float64)])

        def ref(u):
            mu, sg = u[:, 0], u[:, 1]
            pri = [pr.norm_term(mu, m0, s0), pr.unif_term(sg, 0, 100)]
            if split is None:
                return pr.combine(pri + [pr.norm_plate(x, mu, sg)])
            return pr.combine([pr.norm_plate(x[:split], mu, sg)] + pri + [pr.norm_plate(x[split:], mu, sg)])
        pr.per_state(ref, S).check(s.log_post(), f"n={x.size} {what}")
    return check


NORM_MODES = (("stat", {}), ("cache", {"AMWG_STAT_LOWERING": "0"}))


@pytest.mark.parametrize("n", [1, 7, 9, 1021])
def test_normal_iid_plate_sizes(gpu_pkg, n):
    """n = 1 (the smallest plate), 7 and 9 (around one block of eight), 1021 (blocks and a tail; the statistics sweep). The column
    sits at offset 0 of its own column: a 16-byte aligned start."""
    pr.require_extended()
    x = np.random.default_rng(n).normal(184.5, 4.5, n)
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    for mode, envs in NORM_MODES:
        with env(**envs):
            s = mcmc.AmwgSampler(PARAMS_NORM, norm_points(ld, mcmc), x.tolist(), {"chains": 33 if n < 100 else 200, "seed": n})
        assert f"plate NORM_IID n={n}" in s.program_summary()
        assert any(t.startswith("pre-evaluated statistics") for t in s.program_summary()) == (mode == "stat" and n >= 64)
        assert s.plate_sources() == ["shared"]
        at_checkpoints(s, norm_check(x))


def test_normal_plate_starting_at_an_odd_index(gpu_pkg):
    """The second plate starts at point 9: sum_sq_dev peels one point to align its 16-byte loads."""
    x = np.random.default_rng(5).normal(184.5, 4.5, 1021)
    ld = gpu_pkg.ld
    for mode, envs in NORM_MODES:
        with env(**envs):
            s = gpu_pkg.mcmc.AmwgSampler(PARAMS_NORM, norm_split(ld, 9), x.tolist(), {"chains": 200, "seed": 6})
        assert [t for t in s.program_summary() if t.startswith("plate")] == ["plate NORM_IID n=9", "plate NORM_IID n=1012"]
        assert s.plate_sources() == ["shared", "shared"]
        at_checkpoints(s, norm_check(x, split=9))


def test_normal_plates_on_the_ring_and_l2(gpu_pkg):
    """30001 points (> the staging budget): the first plate (6149 points, three full tiles of 2048 and a partial one, aligned start)
    streams through the ring; the second starts at an odd index, which the ring cannot serve, and reads L2 inside the same ring
    model. Without CTA-uniform steps (and with the full program) both read L2."""
    n, k = 30001, 6149
    assert 8 * n > BUDGET and k > 3 * (RING_STAGE // 8) and k % (RING_STAGE // 8) != 0
    x = np.random.default_rng(7).normal(184.5, 4.5, n)
    ld = gpu_pkg.ld
    for mode, envs, where in (("stat", {}, ["ring", "L2"]), ("cache", {"AMWG_STAT_LOWERING": "0"}, ["ring", "L2"]),
                              ("l2", {"AMWG_STAT_LOWERING": "0", "AMWG_PHASE_SYNC": "0"}, ["L2", "L2"])):
        with env(**envs):
            s = gpu_pkg.mcmc.AmwgSampler(PARAMS_NORM, norm_split(ld, k), x.tolist(), {"chains": 200, "seed": 8})
        assert s.plate_sources() == where, mode
        at_checkpoints(s, norm_check(x, split=k))


def test_normal_plate_cancellation_near_1e6(gpu_pkg):
    """data near 1e6 with sd ~ 1: the plate must sum (x_i - mean)^2, not expand it (x^2 - 2 x mean + mean^2 loses ~1e-4 per point)"""
    x = 1e6 + np.random.default_rng(9).normal(0.0, 1.0, 1021)
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real", "init": 1e6 + 0.3}, "sigma": {"type": "real", "lower": 0, "init": 1.2}}
    for mode, envs in NORM_MODES:
        with env(**envs):
            s = mcmc.AmwgSampler(params, norm_points(ld, mcmc, 1e6, 100.0), x.tolist(), {"chains": 200, "seed": 10})
        assert "plate NORM_IID n=1021" in s.program_summary() and s.plate_sources() == ["shared"]
        assert any(t.startswith("pre-evaluated statistics") for t in s.program_summary()) == (mode == "stat")
        at_checkpoints(s, norm_check(x, 1e6, 100.0))


def hier_points(ld, mcmc, J):
    def f(state, d):
        lp = 0
        for j in range(J):
            lp += ld.norm(state.mu[j], 0, 100)
        lp += ld.unif(state.sigma, 0, 100)
        for i in mcmc.points(len(d.y)):
            lp += ld.norm(d.y[i], state.mu[d.g[i]], state.sigma)
        return lp
    return f


@pytest.mark.parametrize("total,where", [(501, "shared"), (30011, "L2")])
def test_normal_grouped_plate_with_ragged_groups(gpu_pkg, total, where):
    y, g, J = ragged_groups(total, total)
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    for mode, envs in NORM_MODES:
        with env(**envs):
            s = mcmc.AmwgSampler(params, hier_points(ld, mcmc, J), {"y": y.tolist(), "g": g.tolist()}, {"chains": 33, "seed": 11})
        assert f"plate NORM_GROUPED n={total} groups={J}" in s.program_summary()
        assert s.plate_sources() == [where]

        def check(s, what):
            st = s.state
            mu = np.asarray(st["mu"], np.float64).reshape(33, J)
            S = np.column_stack([mu, np.asarray(st["sigma"], np.float64)])

            def ref(u):
                terms = [pr.norm_term(u[:, j], 0.0, 100.0) for j in range(J)] + [pr.unif_term(u[:, J], 0, 100)]
                return pr.combine(terms + [pr.norm_plate(y, pr.group_means(u[:, :J], g), u[:, J], n_groups=J)])
            pr.per_state(ref, S).check(s.log_post(), f"{mode} {what}")
        at_checkpoints(s, check)


def test_normal_plates_on_jit_handles_with_shadow_threads(gpu_pkg):
    """AMWG_JIT=1 at 4096 + 37 chains: the run-time specialised statistics sweep; log_post() re-evaluates every chain's state with
    amwg_relp_kernel, whose last CTA has shadow threads that walk the ring with the others."""
    n, k = 30001, 6149
    x = np.random.default_rng(12).normal(184.5, 4.5, n)
    ld = gpu_pkg.ld
    with env(AMWG_JIT="1"):
        s = gpu_pkg.mcmc.AmwgSampler(PARAMS_NORM, norm_split(ld, k), x.tolist(), {"chains": 4096 + 37, "seed": 13})
    on, note = s.jit_status()
    assert on and "one streamed column" in note, note              # the specialised sweep streams the column too
    assert s.plate_sources() == ["ring", "L2"]                       # log_post(): the interpreter's re-evaluation, first plate on the ring
    at_checkpoints(s, norm_check(x, split=k))
