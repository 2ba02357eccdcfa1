"""CPU-only checks of the NumPy spec of the Gibbs sampler (tests/gibbs_oracle.py): the Gamma sampler against scipy, the conjugate
parameter steps against their analytic posteriors, and a Geweke (2004) joint-distribution test of the whole sweep."""
import numpy as np
import pytest
from scipy import stats

from oracle import kalman_em as K
import gibbs_oracle as G
import simsmooth_oracle as SO
from simsmooth_checks import problem

SEED = 20261016


@pytest.mark.parametrize("alpha", [1.0, 1.5, 7.3, 120.0])
def test_gamma_sampler_matches_scipy(alpha):
    n = 20000
    vals, fb = [], 0
    for rid in range(4):
        v, f = G.gamma_mt(alpha, SEED, G.gibbs_id(3, rid), np.arange(n // 4))
        vals.append(v); fb += int(f.sum())
    v = np.concatenate(vals)
    assert fb == 0
    assert stats.kstest(v, stats.gamma(alpha).cdf).pvalue > 1e-3


def test_factor_step_is_the_simulation_smoother():
    """The path of a sweep is dfm_simulation_smoother's draw gibbs_id(c, s) at theta (simsmooth_oracle), and z~_0's lag block
    continues the path (z~_1 = [f~_1; z~_0 without its last block])."""
    X, Lam, Rv, A, Q = problem(N=12, r=2, T=30, p=2, miss=0.1, exclude=(3,))
    k = 4
    Qt = np.zeros((k, k)); Qt[:2, :2] = Q
    P0 = K.lyapunov_doubling(K.companion(A, 2, 2), Qt)
    th = dict(Lam=Lam, R=Rv, A=A, Q=Q, P0=P0)
    rid = G.gibbs_id(5, 7)
    _, F, Xd, ll, z0 = G.sweep(X, th, 2, 3, G.default_prior(2), SEED, rid)
    Fr, Xr = SO.simulation_smoother(X, Lam, Rv, A, Q, P0, 2, 3, SEED, [rid])
    assert np.max(np.abs(F - Fr[0])) < 1e-10
    ok = ~np.isnan(Xr[0])
    assert (np.isnan(Xd) == ~ok).all() and np.max(np.abs(Xd[ok] - Xr[0][ok])) < 1e-10
    assert abs(ll - K.e_step(np.vstack([X, np.full((3, 12), np.nan)]), Lam, Rv, A, Q, P0, 2)["loglik"]) < 1e-9 * abs(ll)
    g = G.prepare(np.vstack([X, np.full((3, 12), np.nan)]), Lam, Rv, A, Q, P0, 2)
    Z, _ = G.draw_states(g, *SO.normals(SEED, rid, k, 2, 33, 12))
    assert np.allclose(Z[1, 2:], Z[0, :2], atol=1e-10) and np.allclose(Z[0, :2], F[0])


def _conj_problem(p, miss, exclude):
    rng = np.random.default_rng(p * 10 + int(miss * 100))
    T, N, r = 60, 5, 2
    k = r * p
    Z = rng.standard_normal((T, k))
    for t in range(1, T):
        Z[t, r:] = Z[t - 1, :k - r]
    X = Z[:, :r] @ rng.standard_normal((r, N)) + 0.7 * rng.standard_normal((T, N))
    X[rng.random((T, N)) < miss] = np.nan
    use = np.ones(N, bool); use[list(exclude)] = False
    return X, Z, use


def _zstat(mean, ref, sd, n):
    return np.max(np.abs(mean - ref) / (sd / np.sqrt(n)))


@pytest.mark.parametrize("p,miss,exclude", [(1, 0.0, ()), (1, 0.15, (3,)), (2, 0.1, (0,))])
def test_conjugate_steps_match_analytic_posterior(p, miss, exclude):
    """>= 20 000 parameter draws at a fixed path and panel against the NIG / NIW posterior means and variances."""
    X, Z, use = _conj_problem(p, miss, exclude)
    T, N = X.shape; r = 2; k = r * p
    pr = dict(kap_lam=0.5, a_R=3.0, b_R=1.0, kap_A=0.5, nu_Q=r + 4.0, s_Q=1.0)
    n = 20000
    dr = [G.draw_params(X, Z, use, p, pr, SEED, G.gibbs_id(1, s)) for s in range(n)]
    Lam = np.stack([d["Lam"] for d in dr]); R = np.stack([d["R"] for d in dr])
    A = np.stack([d["A"] for d in dr]); Q = np.stack([d["Q"] for d in dr])
    assert np.isnan(Lam[:, ~use]).all() and np.isnan(R[:, ~use]).all()
    obs = ~np.isnan(X); F = Z[:, :r]
    for i in np.flatnonzero(use):
        o = obs[:, i]; Fi = F[o]; xi = X[o, i]
        P = pr["kap_lam"] * np.eye(r) + Fi.T @ Fi
        m = np.linalg.solve(P, Fi.T @ xi)
        a = pr["a_R"] + o.sum() / 2; b = pr["b_R"] + (xi @ xi - (Fi.T @ xi) @ m) / 2
        ER, VR = b / (a - 1), b * b / ((a - 1) ** 2 * (a - 2))
        assert _zstat(R[:, i].mean(), ER, np.sqrt(VR), n) < 5
        assert _zstat(Lam[:, i].mean(0), m, Lam[:, i].std(0), n) < 5
        cov = ER * np.linalg.inv(P)                                     # Student-t covariance of lam_i
        d2 = (Lam[:, i] - m) ** 2
        assert _zstat(d2.mean(0), np.diag(cov), d2.std(0), n) < 5
    Y, Zl = G.regression(Z, T, r, p)
    Gm = pr["kap_A"] * np.eye(k) + Zl.T @ Zl
    Bh = np.linalg.solve(Gm, Zl.T @ Y)
    S = pr["s_Q"] * np.eye(r) + Y.T @ Y - Bh.T @ Zl.T @ Y
    nu = pr["nu_Q"] + T - 1
    EQ = S / (nu - r - 1)
    assert _zstat(Q.mean(0), EQ, Q.std(0), n) < 5
    # Var(Q_ij) of the inverse Wishart
    den = (nu - r) * (nu - r - 1) ** 2 * (nu - r - 3)
    VQ = ((nu - r + 1) * S * S + (nu - r - 1) * np.outer(np.diag(S), np.diag(S))) / den
    dq = (Q - EQ) ** 2
    assert _zstat(dq.mean(0), VQ, dq.std(0), n) < 5
    At = A.transpose(0, 2, 1)                                           # A' (k x r)
    assert _zstat(At.mean(0), Bh, At.std(0), n) < 5
    VA = np.outer(np.diag(np.linalg.inv(Gm)), np.diag(EQ))              # Var(A'_ab) = [Gm^-1]_aa E[Q_bb]
    da = (At - Bh) ** 2
    assert _zstat(da.mean(0), VA, da.std(0), n) < 5


def _prior_draw(rng, N, r, p, pr):
    k = r * p
    R = pr["b_R"] / rng.gamma(pr["a_R"], size=N)
    Lam = rng.standard_normal((N, r)) * np.sqrt(R / pr["kap_lam"])[:, None]
    W = stats.invwishart(df=pr["nu_Q"], scale=pr["s_Q"] * np.eye(r)).rvs(random_state=rng)
    Q = np.atleast_2d(W)
    At = rng.standard_normal((k, r)) / np.sqrt(pr["kap_A"]) @ np.linalg.cholesky(Q).T
    return dict(Lam=Lam, R=R, A=At.T, Q=Q)


def _simulate(rng, th, P0, T, p, miss):
    r = th["Q"].shape[0]; k = r * p; N = th["Lam"].shape[0]
    M = K.companion(th["A"], r, p); LQ = np.linalg.cholesky(th["Q"])
    z = np.zeros((T, k)); z[0] = np.linalg.cholesky(P0) @ rng.standard_normal(k)
    for t in range(1, T):
        z[t] = M @ z[t - 1]; z[t, :r] += LQ @ rng.standard_normal(r)
    X = z[:, :r] @ th["Lam"].T + np.sqrt(th["R"])[None, :] * rng.standard_normal((T, N))
    X[miss] = np.nan
    return X, z


def _g(th, F):
    return np.concatenate([th["Lam"].ravel(), th["R"], th["A"].ravel(), th["Q"].ravel(), F[1]])


def test_geweke_joint_distribution():
    """Geweke (2004): the marginal-conditional simulator (theta from the prior, then z, then x) and the successive-conditional
    one (Gibbs sweep given x, then x given (theta, z)) agree on the means of lam, R, A, Q and f~_1."""
    T, N, r, p = 8, 3, 1, 1
    pr = dict(kap_lam=1.0, a_R=5.0, b_R=2.0, kap_A=2.0, nu_Q=8.0, s_Q=2.0)
    P0 = np.eye(1)
    miss = np.zeros((T, N), bool); miss[2, 0] = miss[5, 1] = miss[7, 2] = True
    rng = np.random.default_rng(7)
    n_mc = 40000
    mc = []
    for _ in range(n_mc):
        th = _prior_draw(rng, N, r, p, pr)
        _, z = _simulate(rng, th, P0, T, p, miss)
        mc.append(_g(th, z[:, :r]))
    mc = np.array(mc)
    th = _prior_draw(rng, N, r, p, pr); th["P0"] = P0
    X, _ = _simulate(rng, th, P0, T, p, miss)
    n_sc = 12000
    sc = []
    for s in range(n_sc):
        new, F, _, _, _ = G.sweep(X, th, p, 0, pr, SEED, G.gibbs_id(0, s))
        sc.append(_g(new, F))
        X, _ = _simulate_given(rng, new, F, miss)
        th = new
    sc = np.array(sc)
    nb = 60                                                             # batch means for the autocorrelated chain
    bm = sc[: n_sc // nb * nb].reshape(nb, -1, sc.shape[1]).mean(1)
    se = np.sqrt(mc.var(0) / n_mc + bm.var(0, ddof=1) / nb)
    z = (mc.mean(0) - sc.mean(0)) / se
    assert np.all(np.abs(z) < 4), z


def _simulate_given(rng, th, F, miss):
    T, N = miss.shape
    X = F @ th["Lam"].T + np.sqrt(th["R"])[None, :] * rng.standard_normal((T, N))
    X[miss] = np.nan
    return X, None


def test_split_rhat():
    rng = np.random.default_rng(1)
    d = rng.standard_normal((4, 400))
    assert abs(G.split_rhat(d) - 1.0) < 0.02
    d[0] += 3.0
    assert G.split_rhat(d) > 1.3
