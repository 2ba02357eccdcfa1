"""Validate the forecasting / imputation spec (tests/forecast_oracle.py) by brute-force joint-Gaussian conditioning on tiny
problems, the standard tests/test_oracle_kalman.py sets for the E-step.  CPU only."""
import numpy as np
import pytest

from oracle import kalman_em as K
from oracle.dgp import simulate_panel
from forecast_oracle import smooth_forecast
from forecast_checks import check_closed_forms


def _brute_force(X, Lam, Rv, A, Q, P0, p, H):
    """Stack (z_1..z_{T+H}, x_1..x_{T+H}) of the series in the model, condition on the observed cells."""
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
    # joint covariance of [z; x]
    Sx = Hm @ Sz @ Hm.T + np.diag(np.tile(Ru, Tp))
    S = np.block([[Sz, Sz @ Hm.T], [Hm @ Sz, Sx]])
    o = np.concatenate([np.zeros(Tp * k, bool), ~np.isnan(Xp).ravel()])
    u = ~o
    xo = Xp.ravel()[o[Tp * k:]]
    Kg = S[np.ix_(u, o)] @ np.linalg.inv(S[np.ix_(o, o)])
    mean = Kg @ xo
    cov = S[np.ix_(u, u)] - Kg @ S[np.ix_(o, u)]
    full_m = np.zeros(len(o)); full_m[u] = mean; full_m[o] = xo               # observed cells: the data, variance 0
    full_v = np.zeros(len(o)); full_v[u] = np.diag(cov)
    zs = full_m[:Tp * k].reshape(Tp, k)
    Pz = np.zeros((len(o), len(o))); Pz[np.ix_(u, u)] = cov
    PF = np.stack([Pz[t * k:t * k + r, t * k:t * k + r] for t in range(Tp)])
    xm = full_m[Tp * k:].reshape(Tp, n); xv = full_v[Tp * k:].reshape(Tp, n)
    _, ld = np.linalg.slogdet(S[np.ix_(o, o)])
    ll = -0.5 * (len(xo) * np.log(2 * np.pi) + ld + xo @ np.linalg.solve(S[np.ix_(o, o)], xo))
    return dict(F=zs[:, :r], PF=PF, xmean=xm, xvar=xv, loglik=ll, use=use)


def _problem(p, miss, exclude, T=8, N=5, r=2, seed=0):
    rng = np.random.default_rng(seed + 10 * p)
    k = r * p
    X, _ = simulate_panel(N, r, T, rep=3 + p, missing_frac=miss)
    if miss:
        X[-1, :2] = np.nan; X[-2, 0] = np.nan                         # ragged edge
    Lam = rng.standard_normal((N, r)); Rv = rng.uniform(0.5, 1.5, N)
    if exclude:
        Lam[3] = np.nan
    A = 0.3 * rng.standard_normal((r, k)); Q = np.eye(r) + 0.1 * np.ones((r, r))
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    return X, Lam, Rv, A, Q, P0


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("miss", [0.0, 0.2])
@pytest.mark.parametrize("H", [0, 3])
@pytest.mark.parametrize("exclude", [False, True])
def test_smooth_forecast_matches_brute_force(p, miss, H, exclude):
    X, Lam, Rv, A, Q, P0 = _problem(p, miss, exclude)
    ref = smooth_forecast(X, Lam, Rv, A, Q, P0, p, H)
    bf = _brute_force(X, Lam, Rv, A, Q, P0, p, H)
    use = bf["use"]
    np.testing.assert_allclose(ref["F"], bf["F"], atol=1e-10)
    np.testing.assert_allclose(ref["PF"], bf["PF"], atol=1e-10)
    np.testing.assert_allclose(ref["loglik"], bf["loglik"], rtol=1e-10)
    np.testing.assert_allclose(ref["xhat"][:, use], bf["xmean"], atol=1e-10)           # observed cells: the data, exactly
    np.testing.assert_allclose(ref["xvar"][:, use], bf["xvar"], atol=1e-10)            # observed cells: 0
    assert np.isnan(ref["xhat"][:, ~use]).all() and np.isnan(ref["xvar"][:, ~use]).all()


@pytest.mark.parametrize("p", [1, 2])
def test_forecast_closed_forms_and_padding(p):
    T, H = 40, 6
    X, Lam, Rv, A, Q, P0 = _problem(p, 0.1, False, T=T, N=7)
    ref = smooth_forecast(X, Lam, Rv, A, Q, P0, p, H)
    check_closed_forms(ref, A, Q, p, T, H)
    base = K.e_step(X, Lam, Rv, A, Q, P0, p)
    assert ref["loglik"] == base["loglik"]                                                # padding adds no information
    np.testing.assert_array_equal(ref["zs"][:T], base["zs"])
