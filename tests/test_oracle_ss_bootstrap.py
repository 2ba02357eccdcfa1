"""CPU-only checks of the NumPy spec of the parametric bootstrap (tests/ss_bootstrap_oracle.py): the alignment undoes any
invertible rotation of the factors, rotations leave the likelihood and the impulse responses unchanged, and the simulator's
panels have the covariance of the state-space model."""
import numpy as np

from oracle import kalman_em as K
import ss_bootstrap_checks as BC
import ss_bootstrap_oracle as O


def _rotated(seed=3):
    X, th = BC.fitted(N=14, r=3, T=40, p=2, miss=0.1, exclude=(4,), ragged=3)
    rng = np.random.default_rng(seed)
    Km = rng.standard_normal((3, 3)) + 2.0 * np.eye(3)
    return X, th, O.rotate(th, Km, 2), Km


def test_alignment_undoes_a_rotation():
    X, th, rot, Km = _rotated()
    al = O.align(th["Lam"], th["R"], rot["Lam"], rot["R"], rot["A"], rot["Q"], 2)
    assert al is not None
    np.testing.assert_allclose(al["X"], Km, atol=1e-12)
    for n in ("Lam", "R", "A", "Q"):
        ok = ~np.isnan(th[n])
        assert (np.isnan(al[n]) == ~ok).all()
        assert np.max(np.abs(al[n][ok] - th[n][ok])) <= 1e-12, n


def test_rotation_keeps_the_likelihood():
    X, th, rot, _ = _rotated(5)
    a = K.e_step(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], 2)["loglik"]
    b = K.e_step(X, rot["Lam"], rot["R"], rot["A"], rot["Q"], rot["P0"], 2)["loglik"]
    assert abs(a - b) <= 1e-12 * abs(a)


def test_aligned_irf_equals_original():
    X, th, rot, _ = _rotated(7)
    al = O.align(th["Lam"], th["R"], rot["Lam"], rot["R"], rot["A"], rot["Q"], 2)
    np.testing.assert_allclose(O.irf(al["A"], al["Q"], 2, 12), O.irf(th["A"], th["Q"], 2, 12), atol=1e-12)


def test_alignment_fails_on_singular_loadings():
    X, th, rot, _ = _rotated()
    Ls = rot["Lam"].copy(); Ls[:, 2] = Ls[:, 1]                     # Lam*' W Lam* singular
    assert O.align(th["Lam"], th["R"], Ls, rot["R"], rot["A"], rot["Q"], 2) is None
    Q = -np.eye(3)                                                  # Q~ not positive definite
    assert O.align(th["Lam"], th["R"], rot["Lam"], rot["R"], rot["A"], Q, 2) is None


def test_simulator_moments():
    """Tiny model (N = 3, r = 2, p = 2, T = 5): over 3000 spec panels the sample covariance of (x_2, x_3) matches the brute-force
    state-space covariance within 5 sampling standard errors sqrt((S_ii S_jj + S_ij^2) / n) per element."""
    rng = np.random.default_rng(11)
    N, r, p, T, n = 3, 2, 2, 5, 3000
    Lam = rng.standard_normal((N, r)); R = rng.uniform(0.3, 1.0, N)
    A = np.hstack([np.diag([0.5, -0.3]), np.array([[0.1, 0.0], [0.05, 0.2]])])
    Q = np.array([[1.0, 0.3], [0.3, 0.5]])
    k = r * p
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    Xt = np.zeros((T, N))
    draws = np.stack([O.simulate_panel(Xt, Lam, R, A, Q, P0, p, 99, rep)[0][2:4].ravel() for rep in range(n)])
    S = O.state_space_cov(Lam, R, A, Q, P0, p, T)[2 * N:4 * N, 2 * N:4 * N]
    C = np.cov(draws, rowvar=False, bias=True) + np.outer(draws.mean(0), draws.mean(0))      # E[x x'] (mean zero)
    se = np.sqrt((np.outer(np.diag(S), np.diag(S)) + S ** 2) / n)
    assert (np.abs(C - S) <= 5 * se).all(), np.max(np.abs(C - S) / se)


def test_simulator_template_and_excluded_series():
    X, th = BC.fitted(N=10, r=2, T=30, p=1, miss=0.2, exclude=(3,))
    Xd, F = O.simulate_panel(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], 1, 4, 0)
    use = O.in_model(th["Lam"], th["R"])
    assert np.isnan(Xd[:, ~use]).all()
    assert (np.isnan(Xd[:, use]) == np.isnan(X[:, use])).all()
    assert F.shape == (30, 2)
