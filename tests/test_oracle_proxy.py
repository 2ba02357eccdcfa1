"""CPU-only properties of the NumPy spec of the proxy (external instrument) identification, tests/proxy_oracle.py: invariance under
the normalisation of the factors, recovery of a known impact column, and the q = 0 first stage against White's formula."""
import numpy as np

import identified_oracle as IO
import proxy_oracle as PO
import sign_checks as SC
from oracle import kalman_em as K
from proxy_checks import instruments, paths


def test_normalisation_invariance():
    """f -> K f with a random K applied to theta and the path: resp, fevd, eps, reliability and F agree to 1e-10 (DESIGN.md 4.16)."""
    r, p, N, Tp, H = 3, 2, 12, 80, 6
    Lam, R, A, Q, sc = SC.models(r, p, N, 1, seed=3)
    F, e = paths(A, Q, p, Tp, 4)
    Z = instruments(e[0], 2, 5)
    rng = np.random.default_rng(6)
    for _ in range(3):
        Km = rng.standard_normal((r, r)) + 2 * np.eye(r)
        Lk, Ak, Qk = IO.rotate(Lam[0], A[0], Q[0], Km, p)
        a = PO.identify(Lam[0], R[0], A[0], Q[0], F[0], Z, p, H, 1, q=3, block=4, n_boot=3, seed=1, scale=sc)
        b = PO.identify(Lk, R[0], Ak, Qk, F[0] @ Km.T, Z, p, H, 1, q=3, block=4, n_boot=3, seed=1, scale=sc)
        for n in ("resp", "fevd", "eps", "reliability", "fs_pi", "fs_F"):
            scale = max(1.0, np.nanmax(np.abs(a[n])))
            assert np.nanmax(np.abs(a[n] - b[n])) <= 1e-10 * scale, n
        # omega itself rotates: omega~ = U' omega, U = L^-1 K^-1 L~ orthogonal
        U = np.linalg.solve(np.linalg.cholesky(Q[0]), np.linalg.solve(Km, np.linalg.cholesky(Qk)))
        assert np.allclose(U.T @ U, np.eye(r), atol=1e-12)
        assert np.allclose(b["omega"], a["omega"] @ U, atol=1e-10)


def test_recovers_the_instrumented_shock():
    """A DFM (r = 4, N = 100, T = 2000, L = I) whose instrument is shock 1 plus noise of standard deviation sigma: at the true
    parameters along the smoothed path, omega recovers e_1.  Each other component of Gamma is a mean of T products of independent
    unit-variance shocks with (eps_1 + noise), standard error sqrt((1 + sigma^2) / T), against Gamma_1 ~ 1; the tolerance is five
    such standard errors on the norm of the r - 1 components, plus the smoothing error of the path (about 1 / N per component)."""
    r, p, N, T, sig = 4, 1, 100, 2000, 1.0
    rng = np.random.default_rng(11)
    Lam = rng.standard_normal((N, r)); R = np.ones(N)
    A = 0.5 * np.eye(r); Q = np.eye(r)
    e = rng.standard_normal((T, r))
    F = np.zeros((T, r))
    for t in range(T):
        F[t] = e[t] + (A @ F[t - 1] if t else 0.0)
    X = F @ Lam.T + rng.standard_normal((T, N))
    P0 = np.linalg.inv(np.eye(r) - 0.25 * np.eye(r))
    Fs = K.e_step(X, Lam, R, A, Q, P0, p)["zs"][:, :r]
    z = e[:, 0] + sig * rng.standard_normal(T)
    i0 = int(np.argmax(np.abs(Lam[:, 0]) / np.linalg.norm(Lam, axis=1)))     # the series that loads most on factor 1
    o = PO.identify(Lam, R, A, Q, Fs, z, p, 4, i0)
    assert o["status"][0] == 0
    tol = 5 * np.sqrt((r - 1) * (1 + sig ** 2) / T) + r / N
    err = np.linalg.norm(o["omega"][0, 0] - np.eye(r)[0])
    assert err < tol, (err, tol)
    assert abs(o["reliability"][0] - 1 / (1 + sig ** 2)) < 0.1
    assert o["fs_F"][0] > 100


def test_first_stage_q0_is_white():
    rng = np.random.default_rng(2)
    n = 60
    z = rng.standard_normal(n); y = 0.7 * z + rng.standard_normal(n) * (1 + 0.5 * np.abs(z))
    pi, F = PO.first_stage(y, z, 0)
    X = np.column_stack([np.ones(n), z])
    beta = np.linalg.solve(X.T @ X, X.T @ y)
    v = y - X @ beta
    XXi = np.linalg.inv(X.T @ X)
    V = XXi @ (X.T * v ** 2) @ X @ XXi
    assert abs(pi - beta[1]) < 1e-12
    assert abs(F - beta[1] ** 2 / V[1, 1]) < 1e-10 * F


def test_block_indices():
    """Blocks of length l cover n positions, start inside 0 .. n - l, and block = n gives the sample itself."""
    for n, l in ((10, 1), (10, 3), (11, 4), (7, 7)):
        ix = PO.block_indices(n, l, 5, 9, 1, 3, 2, 40)
        assert len(ix) == n and ix.min() >= 0 and ix.max() < n
        assert (np.diff(ix.reshape(-1)[: (n // l) * l].reshape(-1, l), axis=1) == 1).all()
    np.testing.assert_array_equal(PO.block_indices(9, 100, 5, 9, 0, 1, 1, 40), np.arange(9))
