"""CPU-only checks of the NumPy spec tests/identified_oracle.py: the restricted conditional draws against their analytic moments,
a Geweke (2004) joint-distribution test of the restricted sweep, n_constr = 0 as gibbs_oracle, and the series responses /
variance decompositions against brute-force recursions, their adding-up and their behaviour under rotations of the factors."""
import numpy as np
import pytest

from oracle import kalman_em as K
import gibbs_oracle as G
import identified_oracle as IO
from test_oracle_gibbs import _conj_problem, _zstat, _prior_draw, _simulate, _simulate_given, _g

SEED = 20261017


def _constr():
    """r = 2: series 0 fully pinned (m = r), series 1 one row, series 3 one row (excluded in the tests that exclude it)."""
    idx = np.array([0, 0, 1, 3], np.int32)
    H = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, -1.0], [0.0, 1.0]])
    h = np.array([0.8, 0.0, 0.3, 0.5])
    return idx, H, h


def test_restricted_conditional_moments():
    """20 000 parameter draws at a fixed path (p = 2, missing cells, series 3 excluded) against E[R] = beta / (alpha - 1),
    E[lam] = lam*, Var lam = E[R] diag(S~^-1 - Y G^-1 Y'); every draw on its rows to 1e-12 |h|."""
    p = 2
    X, Z, use = _conj_problem(p, 0.1, (3,))
    T, N = X.shape; r = 2
    pr = dict(kap_lam=0.5, a_R=3.0, b_R=1.0, kap_A=0.5, nu_Q=r + 4.0, s_Q=1.0)
    c = _constr()
    n = 20000
    dr = [IO.draw_params(X, Z, use, p, pr, SEED, G.gibbs_id(2, s), c) for s in range(n)]
    Lam = np.stack([d["Lam"] for d in dr]); R = np.stack([d["R"] for d in dr])
    assert np.isnan(Lam[:, 3]).all() and np.isnan(R[:, 3]).all()
    F = Z[:T, :r]
    for i in (0, 1):
        Hi, hi = IO.rows_of(c, i)
        a, b, ls, C = IO.restricted_moments(X, F, i, Hi, hi, pr)
        assert b >= pr["b_R"]
        ER, VR = b / (a - 1), b * b / ((a - 1) ** 2 * (a - 2))
        assert _zstat(R[:, i].mean(), ER, np.sqrt(VR), n) < 5
        res = Lam[:, i] @ Hi.T - hi
        assert np.max(np.abs(res)) <= 1e-12 * np.abs(hi).max()
        if len(hi) == r:
            np.testing.assert_allclose(Lam[:, i], np.broadcast_to(ls, Lam[:, i].shape), rtol=0, atol=1e-12)
            continue
        assert _zstat(Lam[:, i].mean(0), ls, Lam[:, i].std(0), n) < 5
        d2 = (Lam[:, i] - ls) ** 2
        assert _zstat(d2.mean(0), ER * np.diag(C), d2.std(0), n) < 5
    # the unrestricted series and the transition step are gibbs_oracle's
    ref = G.draw_params(X, Z, use, p, pr, SEED, G.gibbs_id(2, 0))
    for nm in ("A", "Q"):
        np.testing.assert_array_equal(dr[0][nm], ref[nm])
    np.testing.assert_array_equal(dr[0]["Lam"][2:], ref["Lam"][2:])


def test_beta_forms_agree():
    X, Z, use = _conj_problem(1, 0.15, ())
    T = X.shape[0]; r = 2
    pr = dict(kap_lam=0.5, a_R=3.0, b_R=1.0)
    F = Z[:T, :r]
    for i in (0, 1):
        Hi, hi = IO.rows_of(_constr(), i)
        _, b, ls, _ = IO.restricted_moments(X, F, i, Hi, hi, pr)
        o = ~np.isnan(X[:, i])
        h0 = Hi.T @ np.linalg.solve(Hi @ Hi.T, hi)
        b2 = pr["b_R"] + 0.5 * (np.sum((X[o, i] - F[o] @ ls) ** 2) + pr["kap_lam"] * np.sum((ls - h0) ** 2))
        assert abs(b - b2) < 1e-10 * b2


def test_no_rows_is_gibbs_oracle():
    X, Z, use = _conj_problem(2, 0.1, (0,))
    pr = G.default_prior(2)
    empty = (np.zeros(0, np.int32), np.zeros((0, 2)), np.zeros(0))
    for c in (None, empty):
        a = IO.draw_params(X, Z, use, 2, pr, SEED, G.gibbs_id(1, 3), c)
        b = G.draw_params(X, Z, use, 2, pr, SEED, G.gibbs_id(1, 3))
        for nm in a:
            np.testing.assert_array_equal(a[nm], b[nm])


def _prior_draw_restricted(rng, N, r, p, pr, c):
    th = _prior_draw(rng, N, r, p, pr)
    for i in sorted(set(int(v) for v in c[0])):
        Hi, hi = IO.rows_of(c, i)
        th["Lam"][i] = IO.correct(th["Lam"][i], np.eye(r), Hi, hi)      # N(0, R / kap I) conditioned on the rows
    return th


def test_geweke_joint_distribution_restricted():
    """Geweke (2004) with the prior drawn on the restricted set: marginal-conditional and successive-conditional simulators agree
    on the means of lam, R, A, Q and f~_1."""
    T, N, r, p = 8, 3, 2, 1
    pr = dict(kap_lam=1.0, a_R=5.0, b_R=2.0, kap_A=2.0, nu_Q=8.0, s_Q=2.0)
    c = (np.array([0, 0, 1], np.int32), np.array([[1.0, 0.0], [0.0, 1.0], [1.0, -1.0]]), np.array([0.8, 0.0, 0.3]))
    P0 = np.eye(r)
    miss = np.zeros((T, N), bool); miss[2, 0] = miss[5, 1] = miss[7, 2] = True
    rng = np.random.default_rng(11)
    n_mc = 40000
    mc = []
    for _ in range(n_mc):
        th = _prior_draw_restricted(rng, N, r, p, pr, c)
        _, z = _simulate(rng, th, P0, T, p, miss)
        mc.append(_g(th, z[:, :r]))
    mc = np.array(mc)
    th = _prior_draw_restricted(rng, N, r, p, pr, c); th["P0"] = P0
    X, _ = _simulate(rng, th, P0, T, p, miss)
    n_sc = 8000
    sc = []
    for s in range(n_sc):
        new, F, _, _, _ = IO.sweep(X, th, p, 0, pr, SEED, G.gibbs_id(0, s), c)
        sc.append(_g(new, F))
        X, _ = _simulate_given(rng, new, F, miss)
        th = new
    sc = np.array(sc)
    keep = mc.std(0) > 1e-9                                             # the pinned loadings are constants
    nb = 60
    bm = sc[: n_sc // nb * nb].reshape(nb, -1, sc.shape[1]).mean(1)
    se = np.sqrt(mc.var(0) / n_mc + bm.var(0, ddof=1) / nb)
    z = (mc.mean(0) - sc.mean(0))[keep] / se[keep]
    assert np.all(np.abs(z) < 4), z
    np.testing.assert_allclose(sc[:, :1], 0.8, atol=1e-12)             # lam_0 = (0.8, 0) in every sweep


def _model(N=9, r=3, p=2, seed=4):
    rng = np.random.default_rng(seed)
    Lam = rng.standard_normal((N, r)); R = 0.3 + rng.random(N)
    A = 0.3 * rng.standard_normal((r, r * p)) / p
    B = rng.standard_normal((r, r)); Q = B @ B.T + 0.5 * np.eye(r)
    Lam[4] = np.nan
    return Lam, R, A, Q


def test_responses_against_recursion():
    """resp and fevd against the state recursion z_h = M z_{h-1}, z_0 = [chol(Q) e_j; 0], and the FEV sums written out."""
    Lam, R, A, Q = _model()
    N, r = Lam.shape; p = 2; H = 9
    sc = 0.5 + np.arange(N) / N
    resp, fevd, st = IO.responses(Lam, R, A, Q, p, H, scale=sc)
    assert st == 0
    M = K.companion(A, r, p); L = np.linalg.cholesky(Q)
    c = np.zeros((N, H, r))
    for j in range(r):
        z = np.zeros(r * p); z[:r] = L[:, j]
        for h in range(H):
            c[:, h, j] = Lam @ z[:r]
            z = M @ z
    ok = ~np.isnan(Lam[:, 0])
    np.testing.assert_allclose(resp[ok], (sc[:, None, None] * c)[ok], rtol=1e-12, atol=1e-13)
    for i in np.flatnonzero(ok):
        for h in range(H):
            tot = sum(c[i, l, j] ** 2 for l in range(h + 1) for j in range(r)) + R[i]
            for j in range(r):
                assert abs(fevd[i, h, j] - sum(c[i, l, j] ** 2 for l in range(h + 1)) / tot) < 1e-13
    assert np.isnan(resp[4]).all() and np.isnan(fevd[4]).all()
    r1, f1, _ = IO.responses(Lam, R, A, Q, p, H, n_shock=1, scale=sc)
    np.testing.assert_array_equal(r1, resp[:, :, :1]); np.testing.assert_array_equal(f1, fevd[:, :, :1])


def test_fevd_adds_up():
    Lam, R, A, Q = _model()
    _, fevd, _ = IO.responses(Lam, R, A, Q, 2, 11)
    ok = ~np.isnan(Lam[:, 0])
    tot = fevd.sum(2) + IO.idiosyncratic_share(Lam, R, A, Q, 2, 11)
    np.testing.assert_allclose(tot[ok], 1.0, rtol=0, atol=1e-13)


def test_failed_models():
    Lam, R, A, Q = _model()
    for A_, Q_ in ((np.full_like(A, np.nan), Q), (A, np.diag([1.0, -1.0, 1.0]))):
        resp, fevd, st = IO.responses(Lam, R, A_, Q_, 2, 5)
        assert st == 3 and np.isnan(resp).all() and np.isnan(fevd).all()


@pytest.mark.parametrize("s", [1, 2])
def test_rotation_invariance_of_named_shocks(s):
    """Under K whose first s rows are unit rows (the rotations a restriction naming factors 1..s leaves free), resp and fevd of
    shocks < s do not change (1e-10); under a general K they do."""
    Lam, R, A, Q = _model()
    p, H = 2, 8
    rng = np.random.default_rng(s)
    Km = rng.standard_normal((3, 3)) + 3 * np.eye(3)
    Km[:s] = np.eye(3)[:s]
    r0, f0, _ = IO.responses(Lam, R, A, Q, p, H)
    r1, f1, _ = IO.responses(*IO.rotate(Lam, A, Q, Km, p)[:1], R, *IO.rotate(Lam, A, Q, Km, p)[1:], p, H)
    ok = ~np.isnan(Lam[:, 0])
    np.testing.assert_allclose(r1[ok, :, :s], r0[ok, :, :s], rtol=0, atol=1e-10)
    np.testing.assert_allclose(f1[ok, :, :s], f0[ok, :, :s], rtol=0, atol=1e-10)
    np.testing.assert_allclose(f1[ok].sum(2), f0[ok].sum(2), rtol=0, atol=1e-10)
    G_ = rng.standard_normal((3, 3)) + 3 * np.eye(3)
    r2, f2, _ = IO.responses(*IO.rotate(Lam, A, Q, G_, p)[:1], R, *IO.rotate(Lam, A, Q, G_, p)[1:], p, H)
    assert np.max(np.abs(r2[ok, :, 0] - r0[ok, :, 0])) > 1e-3 and np.max(np.abs(f2[ok, :, 0] - f0[ok, :, 0])) > 1e-3
