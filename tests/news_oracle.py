"""FP64 spec of the news decomposition of a nowcast revision (dfm_news).  ORACLE / TEST INFRASTRUCTURE ONLY (NumPy;
validated by brute-force joint-Gaussian conditioning in tests/test_oracle_news.py).

At fixed state-space parameters (the model of oracle/kalman_em.py, panels padded with H all-NaN rows), the revision of a
target y = x_{i*, t*} between two data vintages Omega_old (X_old) and Omega_new (X_new, which only adds cells) is written
as a sum over the newly released cells j (Banbura & Modugno 2014):
    E[y | new] - E[y | old] = sum_j w_j I_j,    I_j = x_j - E[x_j | old],    w = Cov(y, I | old) Var(I | old)^-1.
  1. E-step on the old vintage (kalman_em.e_step over the padded panel): E[f_t | old], the filter covariances.
  2. P = the distinct periods holding a news cell or a target (W of them); only the factors f_s, s in P, enter.
  3. Sigma (W r x W r) = Cov((f_s)_{s in P} | old): diagonal blocks Ps_s[:r, :r], off-diagonal blocks the top-left r x r
     block of J_s J_{s+1} .. J_{t-1} Ps_t (s < t), J_t = Pf_t M' Pp_{t+1}^-1 the RTS smoother gain.
  4. C^J = blockdiag_s (sum_{j news at s} lam_j lam_j' / R_j).
  5. L = psd_cholesky(Sigma), S = I + L' C^J L, G = L S^-1 L' = (Sigma^-1 + C^J)^-1, and w_j = lam_{i*}' G_{t*, s} lam_i / R_i
     for a news cell j = (i, s): Cov(y, I) Var(I)^-1 by the Woodbury identity, without an n_news x n_news matrix.
  6. A target observed in the old vintage: revision 0, weights 0.  A released target: weight 1 on its own cell.  A target
     out of the model (NaN loading or R): NaN.  A new cell of a series out of the model is not news (news NaN, weight 0).
  7. sum_j w_j I_j = xhat(X_new) - xhat(X_old) of smooth_forecast at the target (the invariant the tests check).
The new vintage may only add cells in rows T - news_rows .. T - 1 (the release window); otherwise status 1 (bad argument).
"""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

from oracle import kalman_em as K
from simsmooth_oracle import psd_cholesky


def _nan_out(T, N, nq, news_rows, status):
    nan = np.full((news_rows, N), np.nan)
    return dict(old=np.full(nq, np.nan), new=np.full(nq, np.nan), news=nan, weight=np.full((news_rows, N, nq), np.nan),
                contrib=np.full((news_rows, N, nq), np.nan), status=status, periods=np.zeros(0, int))


def consistent(X_old, X_new, news_rows):
    """Every cell observed in X_old is observed with the same value in X_new, and new cells lie in the release window."""
    X_old = np.asarray(X_old, float); X_new = np.asarray(X_new, float)
    oo = ~np.isnan(X_old)
    if (np.isnan(X_new[oo])).any() or (X_new[oo] != X_old[oo]).any():
        return False
    added = np.isnan(X_old) & ~np.isnan(X_new)
    return not added[:X_old.shape[0] - news_rows].any()


def news(X_old, X_new, Lam, R, A, Q, P0, p, H, targets, news_rows):
    """X_old, X_new (T, N) standardized with NaN; targets: list of (series, period) 0-based, period < T + H.  Returns dict
    old, new (n_target), news (news_rows, N), weight / contrib (news_rows, N, n_target), status, periods (P)."""
    X_old = np.asarray(X_old, float); X_new = np.asarray(X_new, float)
    T, N = X_old.shape; r = Lam.shape[1]; k = r * p; Tp = T + H; nq = len(targets); w0 = T - news_rows
    if not consistent(X_old, X_new, news_rows):
        return _nan_out(T, N, nq, news_rows, 1)
    if P0 is None:
        Qt = np.zeros((k, k)); Qt[:r, :r] = Q
        P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    Xp = np.vstack([X_old, np.full((H, N), np.nan)])
    if (np.asarray(R)[~np.isnan(R)] <= 0).any():
        return _nan_out(T, N, nq, news_rows, 3)
    es = K.e_step(Xp, Lam, R, A, Q, P0, p)
    use = es["use"]; M = K.companion(A, r, p)
    F = es["zs"][:, :r]
    Lam0 = np.where(use[:, None], Lam, 0.0); Rinv = np.where(use, 1.0 / np.where(use, R, 1.0), 0.0)
    mask = np.isnan(X_old[w0:]) & ~np.isnan(X_new[w0:]) & use[None, :]          # news cells (news_rows, N)
    P = sorted(set((w0 + np.nonzero(mask.any(1))[0]).tolist()) | {int(t) for _, t in targets})
    W = len(P); n = W * r; pos = {s: a for a, s in enumerate(P)}
    # Sigma from the RTS smoother: Ps_t and the gains J_t
    Ps, Pf, Pp = es["Ps"], es["Pf"], es["Pp"]
    J = {t: cho_solve(cho_factor(Pp[t + 1], lower=True), M @ Pf[t]).T for t in range(P[0], Tp - 1)}
    Sig = np.zeros((n, n))
    for a, s in enumerate(P):
        Sig[a * r:(a + 1) * r, a * r:(a + 1) * r] = Ps[s][:r, :r]
        for b in range(a + 1, W):
            t = P[b]; X = Ps[t]
            for u in range(t - 1, s - 1, -1):
                X = J[u] @ X
            Sig[a * r:(a + 1) * r, b * r:(b + 1) * r] = X[:r, :r]
            Sig[b * r:(b + 1) * r, a * r:(a + 1) * r] = X[:r, :r].T
    CJ = np.zeros((n, n))
    for a, s in enumerate(P):
        if s >= w0 and s < T:
            m = mask[s - w0]
            CJ[a * r:(a + 1) * r, a * r:(a + 1) * r] = (Lam0[m] * Rinv[m][:, None]).T @ Lam0[m]
    L = psd_cholesky(Sig)
    S = np.eye(n) + L.T @ CJ @ L
    G = L @ np.linalg.solve(S, L.T)
    common = F[w0:T] @ Lam0.T                                                     # E[x | old] over the window
    I = np.where(mask, X_new[w0:] - common, np.nan)
    weight = np.zeros((news_rows, N, nq)); old = np.zeros(nq)
    for q, (i, t) in enumerate(targets):
        if not use[i]:
            old[q] = np.nan; weight[:, :, q] = np.where(mask, np.nan, 0.0)
            continue
        obs_old = t < T and not np.isnan(X_old[t, i])
        old[q] = X_old[t, i] if obs_old else Lam[i] @ F[t]
        if obs_old:
            continue
        if w0 <= t < T and mask[t - w0, i]:
            weight[t - w0, i, q] = 1.0
            continue
        b = pos[t]
        for s in range(w0, T):
            if mask[s - w0].any():
                g = G[pos[s] * r:(pos[s] + 1) * r, b * r:(b + 1) * r] @ Lam[i]
                weight[s - w0, :, q] = np.where(mask[s - w0], (Lam0 @ g) * Rinv, 0.0)
    contrib = np.where(mask[:, :, None], weight * np.nan_to_num(I)[:, :, None], 0.0)
    new = old + contrib.sum((0, 1))
    return dict(old=old, new=new, news=I, weight=weight, contrib=contrib, status=0, periods=np.array(P))
