"""CPU-only: properties of the narrative-restriction spec tests/narrative_oracle.py (no library)."""
import numpy as np

import history_oracle as HOR
import identified_oracle as IO
import narrative_oracle as NO
import sign_checks as SC
import sign_oracle as SO


def model(r=3, p=2, N=6, Tp=14, seed=1):
    Lam, R, A, Q, sc = SC.models(r, p, N, 1, seed=seed)
    F = np.random.default_rng(seed + 1).standard_normal((Tp, r))
    return Lam[0], R[0], A[0], Q[0], F


def test_contribution_is_the_historical_decomposition_on_the_rotated_model():
    """H_{i,k}(t, h) = history_oracle's contrib[i, t+h, k] from base row t - 1 on the model rotated by K = Omega' L^-1: loadings
    Lam K^-1, lags K A_l K^-1, Q = I, path K f."""
    r, p = 3, 2
    Lam, R, A, Q, F = model(r, p)
    H = 5
    Om = SO.omegas(3, 0, [4], r)[0]
    L = np.linalg.cholesky(Q)
    K = Om.T @ np.linalg.inv(L); Ki = np.linalg.inv(K)
    Ar = np.hstack([K @ A[:, l * r:(l + 1) * r] @ Ki for l in range(p)])
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, H)
    for t, h in ((p, 0), (p + 1, 3), (9, H - 1)):
        ref = HOR.decompose(Lam @ Ki, R, Ar, np.eye(r), F @ K.T, p, t - 1)
        for i in range(Lam.shape[0]):
            Hk = NO.contributions(Lam[i] @ P, Om, U, t, h)
            np.testing.assert_allclose(Hk, ref[1][i, t + h], rtol=0, atol=1e-10 * max(1, np.abs(Hk).max()))


def test_contributions_add_up_to_the_forecast_error():
    """sum_k H_{i,k}(t, h) = lam_i' (f_{t+h} - [M^{h+1} z_{t-1}]_{1:r})."""
    r, p = 3, 2
    Lam, R, A, Q, F = model(r, p)
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, 6)
    Om = SO.omegas(5, 1, [0], r)[0]
    k = r * p
    M = np.zeros((k, k)); M[:r] = A; M[r:, :-r] = np.eye(k - r)
    for t, h in ((p, 0), (4, 3), (8, 5)):
        z = np.concatenate([F[t - 1 - l] for l in range(p)])
        fc = (np.linalg.matrix_power(M, h + 1) @ z)[:r]
        for i in range(Lam.shape[0]):
            tot = NO.contributions(Lam[i] @ P, Om, U, t, h).sum()
            np.testing.assert_allclose(tot, Lam[i] @ (F[t + h] - fc), rtol=1e-10, atol=1e-12)


def test_kind0_probability_and_kind2_within_kind1():
    r = 3
    Om = SO.omegas(2, 0, [1], r)[0]
    narr = [(0, 1, 0, 3, 0, 1), (0, 2, 0, 3, 0, -1), (0, 1, 0, 6, 0, -1), (0, 3, 0, 7, 0, 1)]
    n_sim = 1 << 15
    n_ok, _ = NO.omega_sim(lambda i: np.zeros((1, r)), narr, r, n_sim, 9, 4)
    sd = np.sqrt(2 ** -4 * (1 - 2 ** -4) / n_sim)
    assert abs(n_ok / n_sim - 2 ** -4) < 5 * sd
    Lam, R, A, Q, F = model(r, 1, Tp=12)
    P = IO.psi(A, Q, 1, 4)
    cOm = lambda i: (Lam[i] @ P) @ Om
    for j in (1, 2, 3):
        n1, _ = NO.omega_sim(cOm, [(1, j, 2, 5, 3, 1)], r, 4096, 1, 0)
        n2, _ = NO.omega_sim(cOm, [(2, j, 2, 5, 3, 1)], r, 4096, 1, 0)
        n12, _ = NO.omega_sim(cOm, [(1, j, 2, 5, 3, 1), (2, j, 2, 5, 3, 1)], r, 4096, 1, 0)
        assert n12 == n2 <= n1                                 # overwhelming implies most important


def test_normalisation_invariance():
    """Under f -> K f (Lam -> Lam K^-1, A_l -> K A_l K^-1, Q -> K Q K'), chol changes to K L = L~ U' with U orthogonal; the
    candidate Omega~ = U Omega gives the same eps~, decisions and omega."""
    r, p = 3, 1
    Lam, R, A, Q, F = model(r, p, Tp=12)
    rng = np.random.default_rng(3)
    K = rng.standard_normal((r, r)) + 2 * np.eye(r); Ki = np.linalg.inv(K)
    Lk, Ak, Qk, Fk = Lam @ Ki, K @ A @ Ki, K @ Q @ K.T, F @ K.T
    L, Lt = np.linalg.cholesky(Q), np.linalg.cholesky(Qk)
    Uo = np.linalg.solve(Lt, K @ L)                          # K L = Lt Uo
    np.testing.assert_allclose(Uo @ Uo.T, np.eye(r), atol=1e-12)
    Om = SO.omegas(1, 0, np.arange(50), r)
    U1, U2 = NO.shocks_u(A, Q, F, p), NO.shocks_u(Ak, Qk, Fk, p)
    P1, P2 = IO.psi(A, Q, p, 4), IO.psi(Ak, Qk, p, 4)
    narr = [(0, 1, 0, 3, 0, 1), (1, 2, 1, 4, 2, 1), (3, 1, 2, 5, 1, -1)]
    c1, c2 = (lambda i: Lam[i] @ P1), (lambda i: Lk[i] @ P2)
    for om in Om:
        om2 = Uo @ om
        np.testing.assert_allclose(U2[p:] @ om2, U1[p:] @ om, atol=1e-10)
        d1 = NO.decide(om, np.zeros((0, r)), [], narr, c1, U1, r)
        d2 = NO.decide(om2, np.zeros((0, r)), [], narr, c2, U2, r)
        assert d1[0] == d2[0] and (d1[1] == d2[1]).all()
        np.testing.assert_allclose(c2(1) @ om2, c1(1) @ om, atol=1e-10)
        assert NO.omega_sim(lambda i: c1(i) @ om, narr, r, 256, 2, 0) == NO.omega_sim(lambda i: c2(i) @ om2, narr, r, 256, 2, 0)


def test_no_rows_is_sign_oracle_and_flip_group():
    r, p, H = 3, 2, 4
    Lam, R, A, Q, F = model(r, p)
    rows = SC.expand([(0, 1, 1, (0, 1)), (2, 2, -1, 1)])
    a = NO.identify(Lam, R, A, Q, F, p, rows, [], H, 2, 200, 20, 64, seed=4)
    b = SO.identify(Lam, R, A, Q, p, rows, H, 2, 200, 20, seed=4)
    assert a["n_accept"] == b["n_accept"]
    np.testing.assert_array_equal(a["cand"], b["cand"])
    for n in ("rot", "resp", "fevd"):
        np.testing.assert_array_equal(a[n], b[n])
    kept = a["cand"] >= 0
    assert (a["weight"][kept] == 1).all()
    # a shock with kind-0 rows only: negating every sign of its flip group flips the kept column
    narr = [(0, 3, 0, 4, 0, 1), (0, 3, 0, 9, 0, 1)]
    neg = [(k, j, i, t, h, -s) for k, j, i, t, h, s in narr]
    x = NO.identify(Lam, R, A, Q, F, p, [], narr, H, 3, 300, 300, 16)
    y = NO.identify(Lam, R, A, Q, F, p, [], neg, H, 3, 300, 300, 16)
    np.testing.assert_array_equal(x["cand"], y["cand"])
    k = x["cand"] >= 0
    np.testing.assert_array_equal(x["rot"][k][:, :, 2], -y["rot"][k][:, :, 2])
    np.testing.assert_array_equal(x["rot"][k][:, :, :2], y["rot"][k][:, :, :2])


def test_decide_batch_is_decide():
    """decide_batch (quadratic forms, all candidates at once) against the scalar decide (explicit convolution) on 3 000
    candidates, rows of every kind on two shocks: the same accept bits, flips, and margins to 1e-9."""
    import narrative_checks as NC
    r, p, H = 3, 2, 4
    Lam, R, A, Q, sc = SC.models(r, p, 8, 1, seed=1)
    Lam, R, A, Q = Lam[0], R[0], A[0], Q[0]
    F = np.random.default_rng(2).standard_normal((16, r))
    rows, narr = NC.case(Lam, A, Q, F, p, H, 5, 2)
    narr += [(3, 3, 4, 7, 2, -1), (0, 3, 0, 9, 0, 1)]
    C = SO.row_vectors(Lam, A, Q, p, rows, H)
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, H)
    c_of = lambda i: np.einsum("a,hab->hb", Lam[i], P)
    Om = SO.omegas(5, 2, np.arange(3000), r)
    shocks = [j for _, _, j, _ in rows]
    ok, flip, m = NO.decide_batch(Om, C, shocks, narr, c_of, U, r)
    for c in range(len(Om)):
        o1, f1, m1 = NO.decide(Om[c], C, shocks, narr, c_of, U, r)
        assert o1 == ok[c], c
        if o1:
            np.testing.assert_array_equal(f1, flip[c])
        assert abs(m1 - m[c]) <= 1e-9 * max(1.0, m1), (c, m1, m[c])
    assert 0 < ok.sum() < len(Om) and (flip[ok] < 0).any()


def test_weighted_percentiles_exact_rule():
    """The exact rule (100 sum_{j <= i} w_j >= q sum_j w_j) is numpy's weighted inverted_cdf wherever numpy's rounded cdf is more
    than 2^-40 from q / 100, and with equal weights numpy's unweighted inverted_cdf at every size; the near-tie bounds hold the
    exact record."""
    rng = np.random.default_rng(3)
    q = (0, 5, 10, 16, 25, 50, 75, 84, 90, 95, 100)
    seen = 0
    for n in (1, 2, 5, 130, 300, 1000, 4097):
        x = rng.standard_normal(n)
        for w in (rng.random(n) + 0.01, rng.integers(1, 5, n) * (2.0 ** 20 / 37), np.exp(rng.uniform(-20, 20, n))):
            got = NO.weighted_percentiles(x[:, None], w, q)[:, 0]
            o = np.argsort(x, kind="stable")
            cdf = np.cumsum(w[o]) / w.sum()
            for k, qq in enumerate(q):
                if np.abs(cdf - qq / 100).min() > 2.0 ** -40:
                    assert got[k] == np.percentile(x, qq, weights=w, method="inverted_cdf"), (n, qq)
                    seen += 1
            lo, hi = NO.weighted_percentiles(x[:, None], w, q, near=True)
            assert (lo[:, 0] <= got).all() and (got <= hi[:, 0]).all()
        for c in (1.0, 2.0 ** 20 / 3, 2.0 ** 20 / 37, 2.0 ** 20 / 12345):
            got = NO.weighted_percentiles(x[:, None], np.full(n, c), q)[:, 0]
            np.testing.assert_array_equal(got, np.percentile(x, q, method="inverted_cdf"), err_msg=str((n, c)))
        # unit weights: numpy's weighted rule too (its cdf i / n and fl(q / 100) round alike where i / n = q / 100)
        np.testing.assert_array_equal(NO.weighted_percentiles(x[:, None], np.ones(n), q)[:, 0],
                                      np.percentile(x, q, weights=np.ones(n), method="inverted_cdf"))
    assert seen > 100
    # numpy's weighted rule rounds: 130 equal weights 2^20 / 37 give record 65 at q = 50, the exact rule (and numpy without
    # weights) record 64; 300 records at q = 5: 100 * 15 = 5 * 300, so record 14 (the rule with fl(0.05) > 0.05 would give 15)
    x = np.arange(130.0)
    assert NO.weighted_percentiles(x[:, None], np.full(130, 2.0 ** 20 / 37), [50])[0, 0] == 64.0
    assert NO.weighted_percentiles(np.arange(300.0)[:, None], np.ones(300), [5])[0, 0] == 14.0
