"""The extended-precision plate reference (tests/plate_ref.py) against the oracle's term-by-term C models (orc_model_*): where the
reference's own loop is finite, the two agree within the oracle's fp64 error. So when a GPU value test fails, the kernel is wrong."""
import numpy as np
import pytest

import plate_ref as pr
from plate_ref import U, gamma
from plate_ref import edge_data, pois_data, ragged_groups


def _oracle_pois_error(orc, y, X, beta):
    """the oracle's own fp64 error: per row the K-term dot product (gamma_K sum_k |X_ik beta_k|), exp and log within 1 ulp each, three
    roundings of log(lam) * y - lam - lfactorial(y); the K priors; then the running sum over K + n terms"""
    K = X.shape[1]
    eta = X @ beta
    a = gamma(K) * (np.abs(X) @ np.abs(beta))
    e = np.exp(eta)
    lf = pr.lfactorial_ref(orc, y)
    row = np.abs(y) * (a + 3 * U + 2 * U * np.abs(eta)) + e * (np.expm1(a) + 2 * U) + 3 * U * (np.abs(y * eta) + e + np.abs(lf))
    prior = pr.norm_term(beta, 0.0, 10.0)
    mag = np.sum(np.abs(y * eta - e - lf)) + np.sum(np.abs(prior[0].astype(float)))
    return float(np.sum(row) + np.sum(prior[1]) + gamma(n_terms := K + y.size) * mag * (1 + gamma(n_terms)))


def _oracle_norm_error(x, mean, sd, priors):
    """per point -0.5 log(2 pi) - log(sd) - (x - mean)^2 / (2 sd sd): two logs within 1 ulp and six roundings; the priors' own
    error (plate_ref's bound for the same operations); the running sum over every term"""
    c = abs(-0.5 * np.log(2 * np.pi))
    q = (x - mean) ** 2 / (2 * sd * sd)
    row = 6 * U * (c + abs(np.log(sd)) + q)
    prior_mag = sum(float(np.sum(np.abs(v.astype(float)) + b)) for v, b in priors)
    return float(np.sum(row) + sum(float(np.sum(b)) for _, b in priors) +
                 gamma(x.size + len(priors)) * (np.sum(c + abs(np.log(sd)) + q) + prior_mag))


def test_reference_has_an_extended_significand():
    pr.require_extended()
    assert np.finfo(pr.LD).eps < 2.0 ** -62


@pytest.mark.parametrize("K", [1, 3, 8, 16])
def test_poisson_reference_matches_the_oracle(orc, K):
    pr.require_extended()
    rng = np.random.default_rng(K)
    for n in (1, 3, 517):
        y, X = pois_data(K, n, K * 10 + n)
        params = {"beta": {"type": "real", "dim": [K]}}
        states = [rng.normal(0, 0.3, K) for _ in range(6)]
        got = pr.oracle_logpost(orc, "pois_reg", {"y": y, "X": X}, params, states)
        for st, o in zip(states, got):
            ref = pr.combine([pr.norm_term(st[k:k + 1], 0.0, 10.0) for k in range(K)] + [pr.pois_loglin(orc, y, X, st[None, :])])
            tol = _oracle_pois_error(orc, y, X, st)
            assert tol < 1e-3 * ref.row_median[0] and ref.bound[0] < 1e-3 * ref.row_median[0]
            assert abs(pr.LD(o) - ref.value[0]) <= tol, (K, n, float(o), float(ref.value[0]), tol)


def test_poisson_reference_at_the_edges(orc):
    """K = 8 edge data: zero counts, counts near 1e4, an all-zero column, eta in (690, 694) -- the reference and the oracle agree.
    Where exp(eta) underflows with y > 0 the oracle (the reference's loop) gives -Infinity and the exact value is finite; where it
    overflows the oracle gives NaN. The plate follows the exact value in the first case and gives -Infinity in the second
    (tests/test_gpu_plates.py, DESIGN.md section 2)."""
    init = np.array([1.0] + [0.0] * 7)
    params = {"beta": {"type": "real", "dim": [8]}}
    y, X = edge_data(400, 3, "high")
    o = pr.oracle_logpost(orc, "pois_reg", {"y": y, "X": X}, params, [init])[0]
    ref = pr.combine([pr.norm_term(init[k:k + 1], 0.0, 10.0) for k in range(8)] + [pr.pois_loglin(orc, y, X, init[None, :])])
    assert np.isfinite(o) and abs(pr.LD(o) - ref.value[0]) <= _oracle_pois_error(orc, y, X, init)
    y, X = edge_data(400, 3, "mixed")
    keep = X[:, 0] > -745
    o = pr.oracle_logpost(orc, "pois_reg", {"y": y[keep], "X": X[keep]}, params, [init])[0]
    ref = pr.combine([pr.norm_term(init[k:k + 1], 0.0, 10.0) for k in range(8)] + [pr.pois_loglin(orc, y[keep], X[keep], init[None, :])])
    assert abs(pr.LD(o) - ref.value[0]) <= _oracle_pois_error(orc, y[keep], X[keep], init)
    assert pr.oracle_logpost(orc, "pois_reg", {"y": y, "X": X}, params, [init])[0] == -np.inf
    assert np.isfinite(pr.pois_loglin(orc, y, X, init[None, :])[0][0])
    X[7, 0] = 712.0
    assert np.isnan(pr.oracle_logpost(orc, "pois_reg", {"y": y, "X": X}, params, [init])[0])


def test_normal_reference_matches_the_oracle(orc):
    pr.require_extended()
    rng = np.random.default_rng(4)
    P = {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    for n, loc, scale in ((1, 184.5, 4.5), (9, 184.5, 4.5), (1021, 184.5, 4.5), (1021, 1e6, 1.0)):
        x = rng.normal(loc, scale, n)
        states = [(loc + rng.normal(0, scale / 3), scale * rng.uniform(0.7, 1.4)) for _ in range(6)]
        got = pr.oracle_logpost(orc, "norm_readme", x, P, states)
        for (mu, sg), o in zip(states, got):
            priors = [pr.norm_term([mu], 0.0, 100.0), pr.unif_term([sg], 0, 100)]
            ref = pr.combine(priors + [pr.norm_plate(x, [mu], [sg])])
            tol = _oracle_norm_error(x, mu, sg, priors)
            assert tol < 1e-3 * ref.row_median[0]
            assert abs(pr.LD(o) - ref.value[0]) <= tol, (n, float(o), float(ref.value[0]), tol)
    y, g, J = ragged_groups(301, 5)
    params = {"mu": {"type": "real", "dim": [J]}, "sigma": {"type": "real", "lower": 0}}
    for _ in range(4):
        mu, sg = rng.normal(100, 20, J), rng.uniform(3, 8)
        o = pr.oracle_logpost(orc, "hier_norm", {"y": y, "g": g}, params, [list(mu) + [sg]])[0]
        priors = [pr.norm_term(mu[j:j + 1], 0.0, 100.0) for j in range(J)] + [pr.unif_term([sg], 0, 100)]
        ref = pr.combine(priors + [pr.norm_plate(y, pr.group_means(mu[None, :], g), [sg], n_groups=J)])
        tol = _oracle_norm_error(y, mu[g], sg, priors)
        assert tol < 1e-3 * ref.row_median[0]
        assert abs(pr.LD(o) - ref.value[0]) <= tol, (float(o), float(ref.value[0]), tol)
