"""FP64 spec of the historical decompositions of the state-space DFM (dfm_historical_decomposition).  ORACLE / TEST
INFRASTRUCTURE ONLY (NumPy; checked in tests/test_oracle_history.py).

One model (Lam N x r, R N, A = [A_1 .. A_p] r x k, Q r x r, k = r p) and one factor path f_0 .. f_{Tp-1} (Tp x r):
  L = chol(Q), M the companion matrix of A, Psi_h = [M^h]_{1:r,1:r} L (identified_oracle.psi);
  eps_t = L^-1 (f_t - sum_{l=1..p} A_l f_{t-l}) for t >= p, NaN for t < p;
  base row t0 (p - 1 <= t0 < Tp), z_t0 = [f_t0; ..; f_{t0-p+1}];
  t > t0:  contrib[i,t,j] = scale_i lam_i' sum_{s=t0+1..t} Psi_{t-s} e_j eps_{j,s}   (j < n_shock)
           rest[i,t]      = the same sum over j >= n_shock
           base[i,t]      = scale_i lam_i' [M^{t-t0} z_t0]_{1:r}
  t <= t0: contrib = rest = 0, base = scale_i lam_i' f_t.
Series out of the model (NaN Lam row or R_i) are NaN; a model whose A, Q or path holds a NaN, or whose Q is not positive definite,
is NaN throughout (status 3).

This spec writes the Psi convolution out term by term and takes M^h by explicit powers; the kernels run the r-dimensional
recursion y_t = sum_l A_l y_{t-l} + L[:, J] eps_{J,t} instead, so the two agree only if both are right.
"""
import numpy as np
from scipy.linalg import solve_triangular

import gibbs_oracle as O
import identified_oracle as IO
from oracle import kalman_em as K


def shocks(A, Q, F, p):
    """eps (Tp, r), NaN rows t < p."""
    F = np.asarray(F, float); Tp, r = F.shape
    L = np.linalg.cholesky(Q)
    E = np.full((Tp, r), np.nan)
    for t in range(p, Tp):
        u = F[t] - sum(A[:, (l - 1) * r:l * r] @ F[t - l] for l in range(1, p + 1))
        E[t] = solve_triangular(L, u, lower=True)
    return E


def decompose(Lam, R, A, Q, F, p, t0, n_shock=None, scale=None):
    """(shocks (Tp, r), contrib (N, Tp, n_shock), rest (N, Tp), base (N, Tp), status) of one model along the path F."""
    Lam = np.asarray(Lam, float); N, r = Lam.shape
    F = np.asarray(F, float); Tp = F.shape[0]
    ns = r if n_shock is None else n_shock
    nan = (np.full((Tp, r), np.nan), np.full((N, Tp, ns), np.nan), np.full((N, Tp), np.nan), np.full((N, Tp), np.nan))
    if np.isnan(A).any() or np.isnan(Q).any() or np.isnan(F).any():
        return nan + (3,)
    try:
        P = IO.psi(A, Q, p, Tp)                                            # (Tp, r, r)
    except np.linalg.LinAlgError:
        return nan + (3,)
    E = shocks(A, Q, F, p)
    sc = np.ones(N) if scale is None else np.asarray(scale, float)
    c = np.einsum("ia,hab->ihb", Lam, P)                                  # c[i, h, j] = lam_i' Psi_h e_j
    M = K.companion(A, r, p)
    z0 = np.concatenate([F[t0 - l] for l in range(p)])
    contrib = np.zeros((N, Tp, ns)); rest = np.zeros((N, Tp)); base = np.empty((N, Tp))
    base[:, :t0 + 1] = (Lam @ F[:t0 + 1].T)
    Mh = np.eye(r * p)
    for t in range(t0 + 1, Tp):
        Mh = M @ Mh
        base[:, t] = Lam @ (Mh @ z0)[:r]
        s = np.arange(t0 + 1, t + 1)
        term = c[:, t - s, :] * E[s][None, :, :]                           # (N, len(s), r): Psi_{t-s} e_j eps_{j,s}
        contrib[:, t] = term[:, :, :ns].sum(1)
        rest[:, t] = term[:, :, ns:].sum((1, 2))
    contrib *= sc[:, None, None]; rest *= sc[:, None]; base *= sc[:, None]
    out = O.in_model(Lam, R)
    contrib[~out] = np.nan; rest[~out] = np.nan; base[~out] = np.nan
    return E, contrib, rest, base, 0


def stable_lags(A, p, rho_max):
    """A = [A_1 .. A_p] (r x r p) with lag block l multiplied by c^l, c = rho_max / rho (when the companion spectral radius rho
    exceeds rho_max): every companion eigenvalue is multiplied by c, so the result has spectral radius <= rho_max.  (Scaling all
    of A by c does not scale the eigenvalues for p > 1.)"""
    A = np.asarray(A, float); r = A.shape[0]
    rho = np.max(np.abs(np.linalg.eigvals(K.companion(A, r, p))))
    if rho <= rho_max:
        return A.copy()
    c = rho_max / rho
    out = np.hstack([A[:, (l - 1) * r:l * r] * c ** l for l in range(1, p + 1)])
    assert np.max(np.abs(np.linalg.eigvals(K.companion(out, r, p)))) <= rho_max * (1 + 1e-9)
    return out


def rotate_path(F, Km):
    """The path of the model f -> K f (identified_oracle.rotate gives the parameters)."""
    return np.asarray(F, float) @ np.asarray(Km, float).T


def simulate(Lam, A, Q, p, Tp, t0, rng):
    """A path from the model with known pieces: f_0 .. f_{p-1} and eps_p .. eps_{Tp-1} drawn, f_t = sum_l A_l f_{t-l} + L eps_t.
    Returns (F, eps (NaN rows t < p), pieces dict base / shock (r, Tp, r) / the factor-level parts from the base row t0 by
    their own recursions: base from z_t0 with no shocks, shock j from zero with eps_j only)."""
    r = Q.shape[0]
    L = np.linalg.cholesky(Q)
    E = np.full((Tp, r), np.nan); E[p:] = rng.standard_normal((Tp - p, r))
    F = np.zeros((Tp, r)); F[:p] = rng.standard_normal((p, r))
    step = lambda Y, t: sum(A[:, (l - 1) * r:l * r] @ Y[t - l] for l in range(1, p + 1))
    for t in range(p, Tp):
        F[t] = step(F, t) + L @ E[t]
    base = np.zeros((Tp, r)); base[:t0 + 1] = F[:t0 + 1]
    sh = np.zeros((r, Tp, r))
    for t in range(t0 + 1, Tp):
        base[t] = step(base, t)
        for j in range(r):
            sh[j, t] = step(sh[j], t) + L[:, j] * E[t, j]
    return F, E, dict(base=base, shock=sh)
