"""CPU-only: the NumPy spec of the historical decompositions (tests/history_oracle.py) on paths simulated from known models:
it recovers the shocks and every piece, the pieces add up to the common component, and the named shock's column does not depend
on the rotations a restriction naming factor 1 leaves free."""
import numpy as np
import pytest

import history_oracle as HO
import identified_oracle as IO


def stable_model(r, p, N, rng):
    """A stationary VAR(p) (companion spectral radius 0.9), a well-conditioned Q, loadings and variances."""
    A = HO.stable_lags(rng.standard_normal((r, r * p)) / np.sqrt(r * p), p, 0.9)
    B = rng.standard_normal((r, r))
    Q = B @ B.T / r + 0.5 * np.eye(r)
    return rng.standard_normal((N, r)), 0.5 + rng.random(N), A, Q


@pytest.mark.parametrize("r,p,t0", [(1, 1, 0), (3, 2, 1), (3, 2, 17), (4, 4, 10), (8, 1, 39)])
def test_recovers_shocks_and_pieces(r, p, t0):
    rng = np.random.default_rng(100 * r + p)
    N, Tp = 7, 40
    Lam, R, A, Q = stable_model(r, p, N, rng)
    F, E, pc = HO.simulate(Lam, A, Q, p, Tp, t0, rng)
    sc = 0.5 + rng.random(N)
    got_E, contrib, rest, base, st = HO.decompose(Lam, R, A, Q, F, p, t0, n_shock=r, scale=sc)
    assert st == 0
    np.testing.assert_allclose(got_E[p:], E[p:], rtol=0, atol=1e-12 * np.abs(E[p:]).max())
    assert np.isnan(got_E[:p]).all()
    scale = np.abs(sc[:, None] * (Lam @ F.T)).max()
    np.testing.assert_allclose(base, sc[:, None] * (Lam @ pc["base"].T), rtol=0, atol=1e-12 * scale)
    for j in range(r):
        np.testing.assert_allclose(contrib[:, :, j], sc[:, None] * (Lam @ pc["shock"][j].T), rtol=0, atol=1e-12 * scale)
    np.testing.assert_array_equal(rest, 0.0)
    assert (contrib[:, :t0 + 1] == 0).all()


@pytest.mark.parametrize("ns", [1, 2, 4])
def test_identity_and_rest(ns):
    rng = np.random.default_rng(7 + ns)
    r, p, N, Tp, t0 = 4, 3, 9, 50, 12
    Lam, R, A, Q = stable_model(r, p, N, rng)
    F = rng.standard_normal((Tp, r))                                          # any path: the identity does not need the model's
    R[3] = np.nan; Lam[5, 2] = np.nan
    sc = 0.5 + rng.random(N)
    E, contrib, rest, base, st = HO.decompose(Lam, R, A, Q, F, p, t0, n_shock=ns, scale=sc)
    full = HO.decompose(Lam, R, A, Q, F, p, t0, n_shock=r, scale=sc)[1]
    common = sc[:, None] * (np.where(np.isnan(Lam), 0, Lam) @ F.T)
    inm = np.isfinite(Lam).all(1) & np.isfinite(R)
    tot = base + contrib.sum(-1) + rest
    np.testing.assert_allclose(tot[inm], common[inm], rtol=0, atol=1e-12 * np.abs(common).max())
    np.testing.assert_allclose(rest[inm], full[inm][:, :, ns:].sum(-1), rtol=0, atol=1e-12 * np.abs(common).max())
    np.testing.assert_array_equal(contrib[inm], full[inm][:, :, :ns])
    assert np.isnan(tot[~inm]).all()


def test_failed_models_are_nan():
    rng = np.random.default_rng(3)
    r, p, N, Tp = 3, 2, 5, 20
    Lam, R, A, Q = stable_model(r, p, N, rng)
    F = rng.standard_normal((Tp, r))
    for a, q, f in ((np.full_like(A, np.nan), Q, F), (A, np.diag([1.0, -1.0, 1.0]), F), (A, Q, np.where(np.arange(Tp)[:, None] == 6, np.nan, F))):
        out = HO.decompose(Lam, R, a, q, f, p, p - 1)
        assert out[-1] == 3 and all(np.isnan(o).all() for o in out[:-1])


def test_rotation_invariance_of_the_named_shock():
    rng = np.random.default_rng(11)
    r, p, N, Tp, t0 = 4, 2, 8, 45, 9
    Lam, R, A, Q = stable_model(r, p, N, rng)
    F, _, _ = HO.simulate(Lam, A, Q, p, Tp, t0, rng)
    sc = 0.5 + rng.random(N)
    E, c, rest, base, _ = HO.decompose(Lam, R, A, Q, F, p, t0, n_shock=1, scale=sc)
    Kf = np.eye(r) + 0.4 * rng.standard_normal((r, r)); Kf[0] = np.r_[1.0, np.zeros(r - 1)]    # first row e_1'
    Lr, Ar, Qr = IO.rotate(Lam, A, Q, Kf, p)
    E2, c2, rest2, base2, _ = HO.decompose(Lr, R, Ar, Qr, HO.rotate_path(F, Kf), p, t0, n_shock=1, scale=sc)
    s = np.abs(base).max()
    np.testing.assert_allclose(c2[..., 0], c[..., 0], rtol=0, atol=1e-10 * s)
    np.testing.assert_allclose(rest2, rest, rtol=0, atol=1e-10 * s)
    np.testing.assert_allclose(base2, base, rtol=0, atol=1e-10 * s)
    np.testing.assert_allclose(E2[p:, 0], E[p:, 0], rtol=0, atol=1e-10 * np.abs(E[p:, 0]).max())
    Kg = np.eye(r) + 0.4 * rng.standard_normal((r, r))                                          # a general rotation
    Lg, Ag, Qg = IO.rotate(Lam, A, Q, Kg, p)
    c3 = HO.decompose(Lg, R, Ag, Qg, HO.rotate_path(F, Kg), p, t0, n_shock=1, scale=sc)[1]
    assert np.abs(c3[..., 0] - c[..., 0]).max() > 1e-3 * s
    full = HO.decompose(Lam, R, A, Q, F, p, t0, scale=sc)[1]
    full2 = HO.decompose(Lr, R, Ar, Qr, HO.rotate_path(F, Kf), p, t0, scale=sc)[1]
    np.testing.assert_allclose(full2[..., 1:].sum(-1), full[..., 1:].sum(-1), rtol=0, atol=1e-10 * s)
    assert np.abs(full2[..., 1] - full[..., 1]).max() > 1e-3 * s                              # a single other column moves
