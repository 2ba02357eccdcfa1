"""Validate the news-decomposition spec (tests/news_oracle.py) against brute-force joint-Gaussian conditioning on tiny
panels: the weights are Cov(y, I | old) Var(I | old)^-1 formed densely over the stacked states and cells, and the
contributions add up to the revision of smooth_forecast's xhat between the two vintages.  CPU only."""
import numpy as np
import pytest

from oracle import kalman_em as K
from oracle.dgp import simulate_panel
from forecast_oracle import smooth_forecast
from news_oracle import news


def _joint(Lam, Rv, A, Q, P0, p, Tp, use):
    """Covariance of the stacked (z_1..z_Tp, x_1..x_Tp) over the series in the model (x row-major: t * n + i)."""
    r = Lam.shape[1]; k = r * p
    Lu, Ru = Lam[use], Rv[use]; n = int(use.sum())
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
    Sx = Hm @ Sz @ Hm.T + np.diag(np.tile(Ru, Tp))
    return Sx


def _brute_weights(X_old, X_new, Lam, Rv, A, Q, P0, p, H, targets):
    """w = Cov(y, I | old) Var(I | old)^-1 densely, for each target; zeros for a target observed in the old vintage."""
    T, N = X_old.shape; Tp = T + H
    use = ~np.isnan(Lam).any(1) & ~np.isnan(Rv)
    cols = np.nonzero(use)[0]; n = len(cols)
    Sx = _joint(Lam, Rv, A, Q, P0, p, Tp, use)
    Xo = np.vstack([X_old[:, use], np.full((H, n), np.nan)]).ravel()
    Xn = np.vstack([X_new[:, use], np.full((H, n), np.nan)]).ravel()
    o = ~np.isnan(Xo)
    J = np.isnan(Xo) & ~np.isnan(Xn)
    cond = Sx - Sx[:, o] @ np.linalg.solve(Sx[np.ix_(o, o)], Sx[o, :])            # Var(x | old)
    cond[o, :] = 0.0; cond[:, o] = 0.0
    VI = cond[np.ix_(J, J)]
    out = []
    for i, t in targets:
        c = int(np.nonzero(cols == i)[0][0])
        out.append(np.linalg.solve(VI, cond[J, t * n + c]))
    cells = [(int(e // n), int(cols[e % n])) for e in np.nonzero(J)[0]]
    return cells, out


def _problem(p, miss, exclude, H, T=8, N=5, r=2, seed=0):
    rng = np.random.default_rng(seed + 10 * p + H)
    k = r * p
    X, _ = simulate_panel(N, r, T, rep=3 + p, missing_frac=miss)
    X[-1, :3] = np.nan; X[-2, 1] = np.nan                                        # ragged edge
    Lam = rng.standard_normal((N, r)); Rv = rng.uniform(0.5, 1.5, N)
    if exclude:
        Lam[3] = np.nan
    A = 0.3 * rng.standard_normal((r, k)); Q = np.eye(r) + 0.1 * np.ones((r, r))
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    X_new = X.copy()
    X_old = X.copy()
    X_old[-1, 3:] = np.nan; X_old[-2, 2:4] = np.nan; X_old[-3, 0] = np.nan        # released in the last three rows
    X_new[-1, 1] = 0.7                                                           # a new cell where the full panel had a hole
    return X_old, X_new, Lam, Rv, A, Q, P0


def _identity(X_old, X_new, Lam, Rv, A, Q, P0, p, H, targets, got, atol=1e-10):
    so = smooth_forecast(X_old, Lam, Rv, A, Q, P0, p, H)["xhat"]
    sn = smooth_forecast(X_new, Lam, Rv, A, Q, P0, p, H)["xhat"]
    for q, (i, t) in enumerate(targets):
        if np.isnan(so[t, i]):
            assert np.isnan(got["new"][q]) and np.isnan(got["old"][q])
            continue
        np.testing.assert_allclose(got["old"][q], so[t, i], rtol=0, atol=atol)
        np.testing.assert_allclose(got["contrib"][:, :, q].sum(), sn[t, i] - so[t, i], rtol=0, atol=atol)
        np.testing.assert_allclose(got["new"][q], sn[t, i], rtol=0, atol=atol)


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("miss", [0.0, 0.2])
@pytest.mark.parametrize("H", [0, 3])
@pytest.mark.parametrize("exclude", [False, True])
def test_news_matches_brute_force(p, miss, H, exclude):
    X_old, X_new, Lam, Rv, A, Q, P0 = _problem(p, miss, exclude, H)
    T, N = X_old.shape
    targets = [(0, T - 1), (4, T - 2), (2, T - 1)] + [(1, T + h) for h in range(H)]
    if exclude:
        targets.append((3, T - 1))                                               # out of the model
    nr = 3
    got = news(X_old, X_new, Lam, Rv, A, Q, P0, p, H, targets, nr)
    assert got["status"] == 0
    _identity(X_old, X_new, Lam, Rv, A, Q, P0, p, H, targets, got)
    tq = [q for q, (i, _) in enumerate(targets) if not (exclude and i == 3)]
    cells, bw = _brute_weights(X_old, X_new, Lam, Rv, A, Q, P0, p, H, [targets[q] for q in tq])
    for q, w in zip(tq, bw):
        for (t, i), wj in zip(cells, w):
            assert abs(got["weight"][t - (T - nr), i, q] - wj) <= 1e-10, (q, t, i, got["weight"][t - (T - nr), i, q], wj)
    use = ~np.isnan(Lam).any(1)
    released = np.isnan(X_old[T - nr:]) & ~np.isnan(X_new[T - nr:])
    assert (np.isnan(got["news"]) == ~(released & use[None, :])).all()
    for q in tq:                                                                 # weights vanish off the news cells
        assert (got["weight"][:, :, q][~(released & use[None, :])] == 0.0).all()
    if exclude:
        q = len(targets) - 1
        assert np.isnan(got["old"][q]) and np.isnan(got["new"][q])


def test_special_targets():
    X_old, X_new, Lam, Rv, A, Q, P0 = _problem(1, 0.0, False, 2)
    T = X_old.shape[0]
    targets = [(4, T - 1), (0, T - 4), (1, T)]                                   # released, observed in the old vintage, forecast
    got = news(X_old, X_new, Lam, Rv, A, Q, P0, 1, 2, targets, 3)
    w = got["weight"]
    assert w[2, 4, 0] == 1.0 and np.count_nonzero(w[:, :, 0]) == 1               # released target: weight e_j
    np.testing.assert_allclose(got["new"][0], X_new[T - 1, 4], rtol=0, atol=1e-12)
    assert (w[:, :, 1] == 0.0).all() and got["new"][1] == got["old"][1] == X_old[T - 4, 0]
    assert np.count_nonzero(w[:, :, 2]) > 1
    _identity(X_old, X_new, Lam, Rv, A, Q, P0, 1, 2, targets, got)


def test_no_news():
    X_old, _, Lam, Rv, A, Q, P0 = _problem(2, 0.1, False, 3)
    T = X_old.shape[0]
    targets = [(0, T - 1), (2, T + 1)]
    got = news(X_old, X_old.copy(), Lam, Rv, A, Q, P0, 2, 3, targets, 2)
    assert got["status"] == 0
    assert np.isnan(got["news"]).all() and (got["weight"] == 0.0).all() and (got["contrib"] == 0.0).all()
    np.testing.assert_array_equal(got["new"], got["old"])


def test_new_cell_out_of_model_is_not_news():
    X_old, X_new, Lam, Rv, A, Q, P0 = _problem(1, 0.0, True, 0)
    T = X_old.shape[0]
    got = news(X_old, X_new, Lam, Rv, A, Q, P0, 1, 0, [(0, T - 1)], 3)
    assert np.isnan(got["news"][2, 3]) and got["weight"][2, 3, 0] == 0.0
    _identity(X_old, X_new, Lam, Rv, A, Q, P0, 1, 0, [(0, T - 1)], got)


def test_inconsistent_vintages():
    X_old, X_new, Lam, Rv, A, Q, P0 = _problem(1, 0.0, False, 0)
    T = X_old.shape[0]
    bad = X_new.copy(); bad[0, 0] += 1.0                                         # an old cell changed
    assert news(X_old, bad, Lam, Rv, A, Q, P0, 1, 0, [(0, T - 1)], 3)["status"] == 1
    bad = X_new.copy(); bad[T - 2, 0] = np.nan                                   # an old cell gone
    assert news(X_old, bad, Lam, Rv, A, Q, P0, 1, 0, [(0, T - 1)], 3)["status"] == 1
    got = news(X_old, X_new, Lam, Rv, A, Q, P0, 1, 0, [(0, T - 1)], 2)         # a new cell above the window
    assert got["status"] == 1 and np.isnan(got["weight"]).all()
