"""FP64 spec of the state-space EM under linear restrictions on the loadings (LambdaConstraint, dfm_functions.ipynb:1063-1186,
applied to the measurement M-step).  TEST INFRASTRUCTURE ONLY; extends oracle/kalman_em.py, whose E-step it reuses.

A restriction is constr = (index, H, h) in the reference's stacked layout, in standardized units: row q says
H[q] @ lam_{index[q]} = h[q]  (index 0-based, H n_c x r, h n_c).  Take series i with rows H_i (m_i x r, m_i <= r) and its
moments S_i = sum_{t obs} E[f_t f_t' | X], s_i = sum_{t obs} x_it E[f_t | X], sxx_i, T_i.  The restricted M-step is

    lu = S_i^-1 s_i,   Y = S_i^-1 H_i',   G = H_i Y,   lam_i = lu - Y G^-1 (H_i lu - h_i)
    R_i = (sxx_i - 2 lam_i' s_i + lam_i' S_i lam_i) / T_i

the exact maximiser of the expected complete-data likelihood over the feasible set: for any R_i the best lam_i is the restricted
least-squares solution, so the iteration stays an EM and its log-likelihood is monotone.  Unrestricted series, A and Q are
m_step's.  loglik[0] of em_kalman_constr belongs to the initial parameters as given, which may violate the restriction; from
iteration 1 on the parameters satisfy it.  G is singular when the rows of H_i are dependent: the Cholesky pivot test is
relative (pivot <= G_PIVOT_RTOL * G_jj), as in the device kernels, and a singular G raises ConstraintSingular (the device
reports status DFM_ERR_NOT_PD for the panel).  Rows on a series out of the model (NaN loadings or R) are ignored."""
import numpy as np

from oracle import kalman_em as K

G_PIVOT_RTOL = 1e-12


class ConstraintSingular(np.linalg.LinAlgError):
    pass


def by_series(constr, N):
    """{series: (H_i, h_i)} of a stacked restriction (rows in their given order)."""
    if constr is None:
        return {}
    idx, H, h = constr
    idx = np.asarray(idx, int).ravel(); H = np.asarray(H, float); h = np.asarray(h, float).ravel()
    if len(idx) == 0:
        return {}
    out = {}
    for i in sorted(set(idx.tolist())):
        sel = np.flatnonzero(idx == i)
        out[i] = (H[sel], h[sel])
    return out


def moments(X, es, r):
    """Per-series moments of the measurement M-step: S (N, r, r), s (N, r), sxx (N), T_i (N)."""
    zs, Ps, obs = es["zs"], es["Ps"], es["obs"]
    Fs = zs[:, :r]
    E = Fs[:, :, None] * Fs[:, None, :] + Ps[:, :r, :r]
    X0 = np.where(obs, X, 0.0)
    return np.einsum("ti,tab->iab", obs.astype(float), E), X0.T @ Fs, (X0 ** 2).sum(axis=0), obs.sum(axis=0)


def restricted_lam(S, s, Hi, hi):
    """lam minimising lam'S lam - 2 lam's subject to Hi lam = hi (S SPD)."""
    lu = np.linalg.solve(S, s)
    Y = np.linalg.solve(S, Hi.T)
    G = Hi @ Y
    try:
        L = np.linalg.cholesky(0.5 * (G + G.T))
    except np.linalg.LinAlgError as e:
        raise ConstraintSingular("dependent restriction rows") from e
    if (np.diag(L) ** 2 <= G_PIVOT_RTOL * np.diag(G)).any():
        raise ConstraintSingular("dependent restriction rows")
    return lu - Y @ np.linalg.solve(G, Hi @ lu - hi)


def m_step(X, es, r, p, constr=None):
    """oracle.kalman_em.m_step with the restricted update on the series that carry rows of constr."""
    Lam, R, A, Q = K.m_step(X, es, r, p)
    rows = by_series(constr, X.shape[1])
    if not rows:
        return Lam, R, A, Q
    S, s, sxx, Ti = moments(X, es, r)
    for i, (Hi, hi) in rows.items():
        if not es["use"][i] or Ti[i] == 0:
            continue
        lam = restricted_lam(S[i], s[i], Hi, hi)
        Lam[i] = lam
        R[i] = (sxx[i] - 2.0 * lam @ s[i] + lam @ S[i] @ lam) / Ti[i]
    return Lam, R, A, Q


def em_kalman(X, Lam, R, A, Q, p=1, P0=None, max_iter=50, tol=0.0, constr=None):
    """oracle.kalman_em.em_kalman with m_step above (same stopping rule and outputs)."""
    r = Lam.shape[1]; k = r * p
    if P0 is None:
        Qt = np.zeros((k, k)); Qt[:r, :r] = Q
        P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    lls = []
    es = None
    for it in range(1, max_iter + 1):
        es = K.e_step(X, Lam, R, A, Q, P0, p)
        lls.append(es["loglik"])
        Lam, R, A, Q = m_step(X, es, r, p, constr)
        if it >= 2 and abs(lls[-1] - lls[-2]) <= tol * 0.5 * (abs(lls[-1]) + abs(lls[-2])):
            break
    return dict(Lam=Lam, R=R, A=A, Q=Q, P0=P0, F=es["zs"][:, :r], PsF=es["Ps"][:, :r, :r],
                loglik=np.array(lls), iters=len(lls), es=es)


def expected_cdll_series(lam, Ri, S, s, sxx, Ti):
    """Series i's term of the expected complete-data log-likelihood (constants dropped)."""
    return -0.5 * (Ti * np.log(Ri) + (sxx - 2.0 * lam @ s + lam @ S @ lam) / Ri)


def series_irf(Lam, xstd, irf):
    """(ns, H, r) responses of the series, data units: xstd_i lam_i' irf[:, h, j]  (irf: (r, H, r) [variable, horizon, shock])."""
    return xstd[:, None, None] * np.einsum("ia,ahj->ihj", Lam, irf)
