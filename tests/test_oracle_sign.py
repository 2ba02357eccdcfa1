"""CPU-only checks of the NumPy spec tests/sign_oracle.py: the candidate rotations are orthogonal and Haar distributed, the
acceptance probabilities match their closed forms, the accepted responses do not depend on the normalisation of the factors,
negated signs mirror the accepted set, and the rotated responses and decompositions add up to the unrotated ones."""
import numpy as np

import identified_oracle as IO
import sign_oracle as SO
from sign_checks import models

SEED = 20261018


def test_omega_orthogonal():
    for r in (1, 3, 8, 12):
        Om = SO.omegas(SEED, 7, np.arange(400), r)
        err = np.abs(np.einsum("cab,cad->cbd", Om, Om) - np.eye(r)).max()
        assert err < 1e-13, (r, err)


def test_haar_second_moment():
    """E[omega_1 omega_1'] = I / r over 20 000 draws at r = 3, within 4.5 standard errors (sphere moments: Var x_a^2 =
    3 / (r (r + 2)) - 1 / r^2, Var x_a x_b = 1 / (r (r + 2)))."""
    r, n = 3, 20000
    w = SO.omegas(SEED, 3, np.arange(n), r)[:, :, 0]
    m = np.einsum("ca,cb->ab", w, w) / n
    sd = np.where(np.eye(r, dtype=bool), np.sqrt(3 / (r * (r + 2)) - 1 / r ** 2), np.sqrt(1 / (r * (r + 2)))) / np.sqrt(n)
    assert (np.abs(m - np.eye(r) / r) < 4.5 * sd).all(), (m, sd)


def test_acceptance_closed_forms():
    """One row on a shock: acceptance 1.  Two rows c_1, c_2 on one shock: (pi - theta) / pi, theta the angle between them."""
    rng = np.random.default_rng(1)
    n = 20000
    for r in (2, 5):
        C = rng.standard_normal((1, r))
        assert SO.acceptance(C, [1], SEED, r, 500) == 1.0
        for th in (0.3, 1.5, 2.6):
            u = rng.standard_normal(r); u /= np.linalg.norm(u)
            v = rng.standard_normal(r); v -= (v @ u) * u; v /= np.linalg.norm(v)
            C2 = np.stack([2.0 * u, 0.5 * (np.cos(th) * u + np.sin(th) * v)])
            a, p0 = SO.acceptance(C2, [1, 1], SEED, 100 + r, n), (np.pi - th) / np.pi
            assert abs(a - p0) < 4 * np.sqrt(p0 * (1 - p0) / n), (r, th, a, p0)


def _rows():
    return [(0, 0, 1, 1), (0, 1, 1, 1), (2, 0, 1, -1), (1, 2, 2, 1), (3, 0, 3, -1), (4, 1, 3, -1)]


def test_normalisation_invariance():
    """Under f -> K f (general invertible K): candidate Omega at theta and U' Omega at the rotated model, U = L^-1 K^-1 chol(K Q K'),
    give the same accept decisions, resp and fevd to 1e-10."""
    r, p, H, ns = 4, 2, 5, 3
    Lam, R, A, Q, sc = models(r, p, 7, 1, seed=3)
    Lam, R, A, Q = Lam[0], R[0], A[0], Q[0]
    Km = np.eye(r) + 0.4 * np.random.default_rng(2).standard_normal((r, r))
    L2, A2, Q2 = IO.rotate(Lam, A, Q, Km, p)
    U = np.linalg.solve(np.linalg.cholesky(Q), np.linalg.solve(Km, np.linalg.cholesky(Q2)))
    np.testing.assert_allclose(U.T @ U, np.eye(r), atol=1e-12)
    rows = _rows(); sh = [j for _, _, j, _ in rows]
    Om = SO.omegas(SEED, 0, np.arange(2000), r)
    ok1, f1, mg = SO.decide(SO.row_vectors(Lam, A, Q, p, rows, H), sh, Om)
    Om2 = np.einsum("ba,cbj->caj", U, Om)                                       # U' Omega
    ok2, f2, _ = SO.decide(SO.row_vectors(L2, A2, Q2, p, rows, H), sh, Om2)
    assert mg.min() > 1e-9 and ok1.any() and not ok1.all()
    np.testing.assert_array_equal(ok1, ok2)
    np.testing.assert_array_equal(f1[ok1], f2[ok1])
    k = np.flatnonzero(ok1)
    r1 = SO.rotated_responses(Lam, R, IO.psi(A, Q, p, H), Om[k] * f1[k][:, None, :], ns, sc)
    r2 = SO.rotated_responses(L2, R, IO.psi(A2, Q2, p, H), Om2[k] * f2[k][:, None, :], ns, sc)
    for a, b in zip(r1, r2):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-10 * np.abs(a).max())


def _feasible(Lam, A, Q, p, rows, H, mid):
    """rows with the signs of candidate 0 of model id `mid` (which is then accepted)."""
    om = SO.omegas(SEED, mid, [0], Lam.shape[1])[0]
    C = SO.row_vectors(Lam, A, Q, p, rows, H)
    return [(i, h, j, int(np.sign(C[q] @ om[:, j - 1]))) for q, (i, h, j, s) in enumerate(rows)]


def test_negated_signs():
    """Negating every sign keeps the same candidates, negates resp on the restricted shocks (1 and 3; shock 2 is unrestricted)
    and leaves fevd unchanged."""
    r, p, H, ns = 3, 1, 4, 3
    Lam, R, A, Q, sc = models(r, p, 6, 1, seed=5)
    rows = _feasible(Lam[0], A[0], Q[0], p, [(0, 0, 1, 1), (0, 1, 1, 1), (2, 0, 1, 1), (3, 0, 3, 1), (4, 1, 3, 1)], H, 9)
    a = SO.identify(Lam[0], R[0], A[0], Q[0], p, rows, H, ns, 3000, 50, seed=SEED, mid=9, scale=sc)
    b = SO.identify(Lam[0], R[0], A[0], Q[0], p, [(i, h, j, -s) for i, h, j, s in rows], H, ns, 3000, 50, seed=SEED, mid=9, scale=sc)
    assert a["n_accept"] > 50 and a["margin"] > 1e-9 and a["cand"][0] == 0
    assert a["n_accept"] == b["n_accept"]
    np.testing.assert_array_equal(a["cand"], b["cand"])
    np.testing.assert_allclose(b["resp"][..., [0, 2]], -a["resp"][..., [0, 2]], rtol=0, atol=1e-14)   # (shock 2 is unrestricted)
    np.testing.assert_array_equal(b["resp"][..., 1], a["resp"][..., 1])
    np.testing.assert_allclose(b["fevd"], a["fevd"], rtol=1e-14)


def test_no_rows_adds_up():
    """n_shock = r and no rows: every candidate is kept, fevd sums to variance_decomposition's total, and resp is the unrotated
    responses times Omega."""
    r, p, H = 4, 2, 6
    Lam, R, A, Q, sc = models(r, p, 8, 1, seed=6)
    Lam[0, 5] = np.nan
    o = SO.identify(Lam[0], R[0], A[0], Q[0], p, [], H, r, 20, 20, seed=SEED, mid=1, scale=sc)
    assert o["n_accept"] == 20 and (o["cand"] == np.arange(20)).all()
    resp, fevd, st = IO.responses(Lam[0], R[0], A[0], Q[0], p, H, scale=sc)
    assert st == 0
    for k in range(20):
        np.testing.assert_allclose(o["fevd"][k].sum(-1), fevd.sum(-1), rtol=1e-12, equal_nan=True)
        np.testing.assert_allclose(o["resp"][k], np.einsum("ihb,bj->ihj", resp, o["rot"][k]), rtol=1e-12, atol=1e-14, equal_nan=True)


def test_resp_is_rotated_series_irf():
    """With rows: the kept resp equals the unrotated responses times Omega[:, :n_shock]."""
    r, p, H, ns = 5, 1, 4, 2
    Lam, R, A, Q, sc = models(r, p, 6, 1, seed=8)
    rows = _feasible(Lam[0], A[0], Q[0], p, _rows()[:4], H, 4)
    o = SO.identify(Lam[0], R[0], A[0], Q[0], p, rows, H, ns, 2000, 30, seed=SEED, mid=4, scale=sc)
    resp = IO.responses(Lam[0], R[0], A[0], Q[0], p, H, scale=sc)[0]
    nk = min(o["n_accept"], 30)
    assert nk > 0
    for k in range(nk):
        np.testing.assert_allclose(o["resp"][k], np.einsum("ihb,bj->ihj", resp, o["rot"][k][:, :ns]), rtol=1e-12, atol=1e-14)
