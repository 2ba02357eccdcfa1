"""CPU-only: the spec of the restricted state-space EM (tests/em_constr_oracle.py) on its own -- feasibility, the KKT
conditions and optimality of the restricted M-step, the EM's monotone log-likelihood, and the identification property of
api.series_irf under a named-factor restriction."""
import numpy as np
import pytest

import em_constr_oracle as O
import ss_bootstrap_oracle as SO
from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel


def _panel(p, N=14, r=3, T=60, miss=0.08, rep=5):
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    F0 = R.pca_score(np.nan_to_num(X), r)
    return X, K.init_from_factors(X, F0, p)


def _constr(r, rng):
    """Series 0: loadings e_1 (named factor); series 3: two general rows; series 7: one general row."""
    idx = [0] * r + [3, 3, 7]
    H = np.vstack([np.eye(r), rng.standard_normal((3, r))])
    h = np.r_[1.0, np.zeros(r - 1), rng.standard_normal(3)]
    return np.array(idx), H, h


def _estep(X, th, p):
    Lam, Rv, A, Q = th
    r = Lam.shape[1]; k = r * p
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    return K.e_step(X, Lam, Rv, A, Q, K.lyapunov_doubling(K.companion(A, r, p), Qt), p)


@pytest.mark.parametrize("p", [1, 2])
def test_mstep_feasible_kkt_optimal(p):
    X, th = _panel(p)
    r = th[0].shape[1]
    rng = np.random.default_rng(11)
    cons = _constr(r, rng)
    es = _estep(X, th, p)
    Lam, Rv, A, Q = O.m_step(X, es, r, p, cons)
    L0, R0, A0, Q0 = K.m_step(X, es, r, p)
    np.testing.assert_array_equal(A, A0); np.testing.assert_array_equal(Q, Q0)
    S, s, sxx, Ti = O.moments(X, es, r)
    rows = O.by_series(cons, X.shape[1])
    for i in range(X.shape[1]):
        if i not in rows:
            np.testing.assert_array_equal(Lam[i], L0[i]); np.testing.assert_array_equal(Rv[i], R0[i])
            continue
        Hi, hi = rows[i]
        np.testing.assert_allclose(Hi @ Lam[i], hi, rtol=0, atol=1e-12 * max(1.0, np.abs(hi).max()))
        g = S[i] @ Lam[i] - s[i]                                     # KKT: gradient in the row space of H_i
        mu = np.linalg.lstsq(Hi.T, g, rcond=None)[0]
        np.testing.assert_allclose(Hi.T @ mu, g, rtol=0, atol=1e-10 * np.abs(s[i]).max())
        best = O.expected_cdll_series(Lam[i], Rv[i], S[i], s[i], sxx[i], Ti[i])
        ns = np.linalg.svd(Hi)[2][Hi.shape[0]:].T                   # null space of H_i
        for _ in range(50):
            lam = Lam[i] + ns @ (rng.standard_normal(ns.shape[1]) * 10.0 ** rng.uniform(-4, 0)) if ns.size else Lam[i]
            Rb = (sxx[i] - 2.0 * lam @ s[i] + lam @ S[i] @ lam) / Ti[i]          # the best R_i for this lam
            assert O.expected_cdll_series(lam, Rb, S[i], s[i], sxx[i], Ti[i]) <= best + 1e-12 * abs(best)
        assert Rv[i] >= R0[i] * (1 - 1e-12)                          # a restriction cannot lower the residual variance


def test_identity_rows_pin_the_loadings():
    X, th = _panel(2)
    r = th[0].shape[1]
    h = np.array([0.3, -1.2, 0.7])
    es = _estep(X, th, 2)
    Lam, _, _, _ = O.m_step(X, es, r, 2, (np.array([5, 5, 5]), np.eye(r), h))
    np.testing.assert_allclose(Lam[5], h, rtol=0, atol=1e-13)


@pytest.mark.parametrize("p", [1, 2])
def test_empty_restriction_is_m_step_bit_for_bit(p):
    X, th = _panel(p)
    r = th[0].shape[1]
    es = _estep(X, th, p)
    ref = K.m_step(X, es, r, p)
    for cons in (None, (np.zeros(0, int), np.zeros((0, r)), np.zeros(0))):
        got = O.m_step(X, es, r, p, cons)
        for a, b in zip(got, ref):
            np.testing.assert_array_equal(a, b)
    e1 = K.em_kalman(X, *th, p=p, max_iter=3)
    e2 = O.em_kalman(X, *th, p=p, max_iter=3, constr=None)
    np.testing.assert_array_equal(e1["loglik"], e2["loglik"]); np.testing.assert_array_equal(e1["Lam"], e2["Lam"])


@pytest.mark.parametrize("p", [1, 2])
def test_em_loglik_monotone_from_iteration_1(p):
    X, th = _panel(p)
    r = th[0].shape[1]
    cons = _constr(r, np.random.default_rng(12))
    out = O.em_kalman(X, *th, p=p, max_iter=12, constr=cons)
    ll = out["loglik"][1:]
    assert (np.diff(ll) >= -1e-9 * np.abs(ll[:-1])).all(), np.diff(ll)
    for i, (Hi, hi) in O.by_series(cons, X.shape[1]).items():
        np.testing.assert_allclose(Hi @ out["Lam"][i], hi, rtol=0, atol=1e-12 * max(1.0, np.abs(hi).max()))


def test_dependent_rows_are_singular():
    X, th = _panel(1)
    r = th[0].shape[1]
    es = _estep(X, th, 1)
    H = np.array([[1.0, 0.5, 0.0], [2.0, 1.0, 0.0]])
    with pytest.raises(O.ConstraintSingular):
        O.m_step(X, es, r, 1, (np.array([2, 2]), H, np.array([1.0, 2.0])))


def test_series_irf_shock1_invariant_under_named_factor_rotations():
    """A restricted fit (series 0 and 1 load e_1' only) rotated by K with first row e_1' satisfies the same restriction; the
    series responses to shock 1 do not move (1e-12), those to the other shocks do."""
    p, H = 2, 8
    X, th = _panel(p, N=16, r=3, T=80, rep=7)
    r = 3
    cons = (np.array([0, 0, 0, 1, 1, 1]), np.vstack([np.eye(r)] * 2), np.r_[1.0, 0, 0, 1.0, 0, 0])
    fit = O.em_kalman(X, *th, p=p, max_iter=6, constr=cons)
    theta = dict(Lam=fit["Lam"], R=fit["R"], A=fit["A"], Q=fit["Q"], P0=fit["P0"])
    xstd = np.linspace(0.5, 2.0, X.shape[1])
    Km = np.array([[1.0, 0.0, 0.0], [0.4, 1.3, -0.2], [-0.7, 0.5, 0.9]])
    rot = SO.rotate(theta, Km, p)
    np.testing.assert_allclose(rot["Lam"][[0, 1]], np.tile(np.r_[1.0, 0, 0], (2, 1)), atol=1e-12)
    irf0 = SO.irf(theta["A"], theta["Q"], p, H).transpose(2, 1, 0)
    irf1 = SO.irf(rot["A"], rot["Q"], p, H).transpose(2, 1, 0)
    s0 = O.series_irf(theta["Lam"], xstd, irf0); s1 = O.series_irf(rot["Lam"], xstd, irf1)
    scale = np.abs(s0[:, :, 0]).max()
    np.testing.assert_allclose(s1[:, :, 0], s0[:, :, 0], rtol=0, atol=1e-12 * scale)
    assert np.abs(s1[:, :, 1:] - s0[:, :, 1:]).max() > 1e-3 * scale
