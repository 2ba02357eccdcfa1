"""Validate the simulation-smoother spec (tests/simsmooth_oracle.py) exactly, not statistically: a draw is affine in the
vector u of all normals it consumes, (f~, x~_missing) = m + G u.  m (u = 0) must be the smoother's posterior mean
(forecast_oracle.smooth_forecast), and G G' the joint posterior covariance from brute-force Gaussian conditioning on tiny
problems (the stacked system of test_oracle_forecast._brute_force).  CPU only."""
import numpy as np
import pytest

from oracle import kalman_em as K
from oracle import dgp
from forecast_oracle import smooth_forecast
import simsmooth_oracle as SO
from simsmooth_oracle import draw_prepared, normals, prepare, psd_cholesky, simulation_smoother
from test_oracle_forecast import _problem


def _joint_posterior(X, Lam, Rv, A, Q, P0, p, H):
    """Mean and covariance of (f_1..f_Tp, x_it missing with i in the model, row-major over (t, i)) given the observed cells."""
    T, N = X.shape; r = Lam.shape[1]; k = r * p; Tp = T + H
    use = ~np.isnan(Lam).any(1) & ~np.isnan(Rv)
    Lu, Ru = Lam[use], Rv[use]; n = int(use.sum())
    Xp = np.vstack([X[:, use], np.full((H, n), np.nan)])
    M = K.companion(A, r, p); Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    covs = [P0]
    for _ in range(1, Tp):
        covs.append(M @ covs[-1] @ M.T + Qt)
    Sz = np.zeros((Tp * k, Tp * k))
    for s in range(Tp):
        blk = covs[s]
        for t in range(s, Tp):
            Sz[t * k:(t + 1) * k, s * k:(s + 1) * k] = blk
            Sz[s * k:(s + 1) * k, t * k:(t + 1) * k] = blk.T
            blk = M @ blk
    Hm = np.zeros((Tp * n, Tp * k))
    for t in range(Tp):
        Hm[t * n:(t + 1) * n, t * k:t * k + r] = Lu
    S = np.block([[Sz, Sz @ Hm.T], [Hm @ Sz, Hm @ Sz @ Hm.T + np.diag(np.tile(Ru, Tp))]])
    xo_mask = ~np.isnan(Xp).ravel()
    o = np.concatenate([np.zeros(Tp * k, bool), xo_mask])
    fidx = np.array([t * k + a for t in range(Tp) for a in range(r)])
    want = np.concatenate([fidx, Tp * k + np.flatnonzero(~xo_mask)])
    Kg = S[np.ix_(want, o)] @ np.linalg.inv(S[np.ix_(o, o)])
    mean = Kg @ Xp.ravel()[xo_mask]
    cov = S[np.ix_(want, want)] - Kg @ S[np.ix_(o, want)]
    return mean, cov, use


def _case(p, miss, exclude):
    X, Lam, Rv, A, Q, P0 = _problem(p, miss, exclude)
    if miss:
        X[3, 1:] = np.nan                      # a period observing one series (< r = 2)
    return X, Lam, Rv, A, Q, P0


def _stack(F, Xd, X, use):
    """(f~ row-major over (t, a); x~ at the missing cells of the series in the model, row-major over (t, i))."""
    Tp = F.shape[0]
    Xp = np.vstack([X, np.full((Tp - X.shape[0], X.shape[1]), np.nan)])[:, use]
    return np.concatenate([F.ravel(), Xd[:, use][np.isnan(Xp)]])


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("miss", [0.0, 0.2])
@pytest.mark.parametrize("H", [0, 3])
@pytest.mark.parametrize("exclude", [False, True])
def test_draw_is_exact_posterior(p, miss, H, exclude):
    X, Lam, Rv, A, Q, P0 = _case(p, miss, exclude)
    T, N = X.shape; r = Lam.shape[1]; k = r * p; Tp = T + H
    g = prepare(X, Lam, Rv, A, Q, P0, p, H)
    shapes = [(k,), (Tp, r), (Tp, r), (N, Tp)]
    sizes = [int(np.prod(s)) for s in shapes]

    def draw(u):
        parts, o = [], 0
        for s, n in zip(shapes, sizes):
            parts.append(u[o:o + n].reshape(s)); o += n
        return draw_prepared(g, *parts)

    F0, X0 = draw(np.zeros(sum(sizes)))
    ref = smooth_forecast(X, Lam, Rv, A, Q, P0, p, H)
    np.testing.assert_allclose(F0, ref["F"], atol=1e-12)
    np.testing.assert_allclose(X0, ref["xhat"], atol=1e-12)                 # observed cells: the data; excluded: NaN
    assert (np.isnan(X0) == np.isnan(ref["xhat"])).all()
    mean, cov, use = _joint_posterior(X, Lam, Rv, A, Q, P0, p, H)
    m = _stack(F0, X0, X, use)
    np.testing.assert_allclose(m, mean, atol=1e-10)
    G = np.empty((len(m), sum(sizes)))
    for j in range(sum(sizes)):
        e = np.zeros(sum(sizes)); e[j] = 1.0
        G[:, j] = _stack(*draw(e), X, use) - m
    np.testing.assert_allclose(G @ G.T, cov, atol=1e-10)
    F1, X1 = draw(np.ones(sum(sizes)))
    Xp = np.vstack([X, np.full((H, N), np.nan)])
    obs = ~np.isnan(Xp)
    assert np.array_equal(X1[obs & use[None, :]], Xp[obs & use[None, :]])     # observed cells stay the data whatever the normals


def test_psd_cholesky_zero_pivots():
    rng = np.random.default_rng(0)
    V = rng.standard_normal((5, 2))
    S = V @ V.T                                                              # rank 2
    L = psd_cholesky(S)
    np.testing.assert_allclose(L @ L.T, S, atol=1e-12)
    assert np.count_nonzero(np.abs(np.diag(L)) > 0) == 2
    assert not psd_cholesky(np.zeros((3, 3))).any()
    P = np.diag([2.0, 0.0, 1.0])
    np.testing.assert_allclose(psd_cholesky(P), np.sqrt(P))


def test_stream_tags():
    assert (SO.RNG_SS_Z0, SO.RNG_SS_ETA, SO.RNG_SS_OBS, SO.RNG_SS_MISS) == (7, 8, 9, 10)
    assert dgp.RNG_BETA == 6                                                   # the new tags follow the generators' streams
    seed, d, k, r, Tp, N = 123, 5, 4, 2, 6, 3
    nu, eta, xi, eps = normals(seed, d, k, r, Tp, N)
    np.testing.assert_array_equal(nu, dgp.rng_normal(seed, d, 7, np.arange(k)))
    np.testing.assert_array_equal(eta[2, 1], dgp.rng_normal(seed, d, 8, 2 * r + 1))
    np.testing.assert_array_equal(xi[4, 0], dgp.rng_normal(seed, d, 9, 4 * r))
    np.testing.assert_array_equal(eps[2, 5], dgp.rng_normal(seed, d, 10, 2 * Tp + 5))
    assert not np.array_equal(nu, normals(seed, d + 1, k, r, Tp, N)[0])


def test_draws_are_a_function_of_the_draw_id():
    X, Lam, Rv, A, Q, P0 = _case(2, 0.2, False)
    Fa, Xa = simulation_smoother(X, Lam, Rv, A, Q, P0, 2, 3, 7, [0, 1, 2, 3])
    Fb, Xb = simulation_smoother(X, Lam, Rv, A, Q, P0, 2, 3, 7, [2, 3])
    np.testing.assert_array_equal(Fa[2:], Fb)
    np.testing.assert_array_equal(Xa[2:], Xb)
