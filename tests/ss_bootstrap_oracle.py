"""FP64 spec of the parametric bootstrap of a fitted state-space DFM (dfm_ss_simulate_panels, dfm_ss_bootstrap).  ORACLE / TEST
INFRASTRUCTURE ONLY (NumPy; checked in tests/test_oracle_ss_bootstrap.py).

Replicate b of a call (replication id rep = rep0 + b) at the fitted parameters theta^ = (Lam, R, A, Q, P0), model of
oracle/kalman_em.py, k = r p:
  1. panel      z_1 = L_P0 nu,  z_t = M z_{t-1} + [L_Q eta_t; 0],  x_it = lam_i' f_t + sqrt(R_i) eps_it where the template panel
                is observed and the series is in the model (Lam row and R_i not NaN), NaN elsewhere.  Standardized model units.
                L_S = simsmooth_oracle.psd_cholesky (a pivot <= 1e-12 max diag is a zero column).
  2. EM         oracle.kalman_em.em_kalman on the panel from theta^, P0 held fixed.
  3. alignment  W = diag(1 / R^_i) over the series in the model;  X = (Lam*' W Lam*)^-1 Lam*' W Lam^,  K = X^-1,
                Lam~ = Lam* X,  A~_l = K A*_l X,  Q~ = K Q* K',  R~ = R*.  Fails (None) when a Cholesky pivot of Lam*' W Lam* is
                <= 1e-12 times its largest diagonal entry, when a partial-pivoting LU pivot of X is <= 1e-12 max |X_ij|, or when
                Q~ is not positive definite.
  4. IRF        irf[j, h, i] = (M~^h G~)[i, j], G~ = [chol(Q~); 0]  (record layout [shock][horizon][variable] of dfm_irf).
  5. forecasts  forecast_oracle.smooth_forecast of the ORIGINAL panel at (Lam~, R~, A~, Q~, P0) with H_fc periods.
Normals: oracle.dgp.rng_normal(seed, rep, stream, element), the NumPy restatement of the device's Philox4x32-10 stream, on three
stream tags after the simulation smoother's 7-10 (the table of include/dfm_b200.h):
  RNG_SSB_Z0   11  nu      z_1 = L_P0 nu                     element a         (a < k)
  RNG_SSB_ETA  12  eta_t   state shocks of periods t >= 1    element t r + a   (a < r)
  RNG_SSB_EPS  13  eps_it  idiosyncratic draw of a cell       element i T + t
"""
import numpy as np
from scipy.linalg import lu_factor

from oracle import kalman_em as K
from oracle.dgp import rng_normal
from simsmooth_oracle import psd_cholesky
from forecast_oracle import smooth_forecast

RNG_SSB_Z0, RNG_SSB_ETA, RNG_SSB_EPS = 11, 12, 13
SING_TOL = 1e-12


def in_model(Lam, R):
    return ~np.isnan(Lam).any(axis=1) & ~np.isnan(R)


def normals(seed, rep, k, r, T, N):
    nu = rng_normal(seed, rep, RNG_SSB_Z0, np.arange(k))
    eta = rng_normal(seed, rep, RNG_SSB_ETA, np.arange(T * r)).reshape(T, r)
    eps = rng_normal(seed, rep, RNG_SSB_EPS, np.arange(N * T)).reshape(N, T).T        # (T, N), element i T + t
    return nu, eta, eps


def simulate_from_normals(Xt, Lam, R, A, Q, P0, p, nu, eta, eps):
    """Panel (T, N) and factors (T, r) of step 1 given the normals."""
    T, N = np.asarray(Xt).shape; r = Lam.shape[1]; k = r * p
    M = K.companion(A, r, p); LP0 = psd_cholesky(P0); LQ = psd_cholesky(Q)
    z = np.zeros((T, k))
    z[0] = LP0 @ nu
    for t in range(1, T):
        z[t] = M @ z[t - 1]
        z[t, :r] += LQ @ eta[t]
    F = z[:, :r]
    use = in_model(Lam, R)
    Lam0 = np.where(use[:, None], Lam, 0.0)
    Xd = F @ Lam0.T + np.sqrt(np.where(use, R, 0.0))[None, :] * eps
    Xd[np.isnan(Xt)] = np.nan
    Xd[:, ~use] = np.nan
    return Xd, F


def simulate_panel(Xt, Lam, R, A, Q, P0, p, seed, rep):
    T, N = np.asarray(Xt).shape; r = Lam.shape[1]
    return simulate_from_normals(Xt, Lam, R, A, Q, P0, p, *normals(seed, rep, r * p, r, T, N))


def align(Lh, Rh, Ls, Rs, As, Qs, p):
    """Step 3: the replicate (Ls, Rs, As, Qs) in the rotation of (Lh, Rh).  Returns dict(Lam, R, A, Q, X, K) or None."""
    r = Lh.shape[1]
    use = in_model(Lh, Rh)
    w = 1.0 / Rh[use]
    L1, L0 = Ls[use], Lh[use]
    G = L1.T @ (w[:, None] * L1)
    Hm = L1.T @ (w[:, None] * L0)
    dmax = float(np.max(np.diag(G)))
    try:
        C = np.linalg.cholesky(G)
    except np.linalg.LinAlgError:
        return None
    if not dmax > 0 or (np.diag(C) ** 2 <= SING_TOL * dmax).any():
        return None
    X = np.linalg.solve(G, Hm)
    lu, _ = lu_factor(X)
    if (np.abs(np.diag(lu)) <= SING_TOL * np.max(np.abs(X))).any():
        return None
    Km = np.linalg.inv(X)
    A2 = np.hstack([Km @ As[:, l * r:(l + 1) * r] @ X for l in range(p)])
    Q2 = Km @ Qs @ Km.T
    Q2 = 0.5 * (Q2 + Q2.T)
    try:
        np.linalg.cholesky(Q2)
    except np.linalg.LinAlgError:
        return None
    Lam = Ls @ X
    Lam[~use] = np.nan
    return dict(Lam=Lam, R=Rs.copy(), A=A2, Q=Q2, X=X, K=Km)


def irf(A, Q, p, H):
    """Step 4: (r_shock, H, r_var) = dfm_irf's record for all r shocks."""
    r = Q.shape[0]; k = r * p
    M = K.companion(A, r, p)
    G = np.zeros((k, r)); G[:r] = np.linalg.cholesky(Q)
    out = np.empty((r, H, r)); x = G.copy()
    for h in range(H):
        out[:, h, :] = x[:r].T
        x = M @ x
    return out


def replicate(Xs, theta, p, seed, rep, max_iter, tol, H_irf, H_fc=0, fc_rows=0):
    """Steps 1-5 for one replicate: dict(panel, em, aligned (or None), irf, xhat, xvar, loglik, iters)."""
    Lam, R, A, Q, P0 = (theta[n] for n in ("Lam", "R", "A", "Q", "P0"))
    Xd, _ = simulate_panel(Xs, Lam, R, A, Q, P0, p, seed, rep)
    em = K.em_kalman(Xd, Lam, R, A, Q, p=p, P0=P0, max_iter=max_iter, tol=tol)
    al = align(Lam, R, em["Lam"], em["R"], em["A"], em["Q"], p)
    out = dict(panel=Xd, em=em, aligned=al, loglik=float(em["loglik"][-1]), iters=int(em["iters"]))
    if al is not None:
        out["irf"] = irf(al["A"], al["Q"], p, H_irf)
        if fc_rows > 0:
            sf = smooth_forecast(Xs, al["Lam"], al["R"], al["A"], al["Q"], P0=P0, p=p, H=H_fc)
            out["xhat"], out["xvar"] = sf["xhat"][-fc_rows:], sf["xvar"][-fc_rows:]
    return out


def rotate(theta, Km, p):
    """theta in the rotation f -> K f: Lam K^-1, K A_l K^-1, K Q K', P0 -> blockdiag(K) P0 blockdiag(K)'."""
    r = Km.shape[0]; Ki = np.linalg.inv(Km)
    Kb = np.kron(np.eye(p), Km)
    return dict(Lam=theta["Lam"] @ Ki, R=theta["R"].copy(),
                A=np.hstack([Km @ theta["A"][:, l * r:(l + 1) * r] @ Ki for l in range(p)]),
                Q=Km @ theta["Q"] @ Km.T, P0=Kb @ theta["P0"] @ Kb.T)


def state_space_cov(Lam, R, A, Q, P0, p, T):
    """Brute-force covariance of vec(x_1 .. x_T) (period-major, all N series) of the model of step 1."""
    r = Lam.shape[1]; k = r * p; N = Lam.shape[0]
    M = K.companion(A, r, p)
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    P = [P0]
    for _ in range(1, T):
        P.append(M @ P[-1] @ M.T + Qt)
    E = np.zeros((r, k)); E[:, :r] = np.eye(r)
    S = np.zeros((T * N, T * N))
    for s in range(T):
        for t in range(s, T):
            Czz = np.linalg.matrix_power(M, t - s) @ P[s]                   # Cov(z_t, z_s)
            blk = Lam @ E @ Czz @ E.T @ Lam.T
            if s == t:
                blk = blk + np.diag(R)
            S[t * N:(t + 1) * N, s * N:(s + 1) * N] = blk
            S[s * N:(s + 1) * N, t * N:(t + 1) * N] = blk.T
    return S
