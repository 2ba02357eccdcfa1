"""FP64 spec of smoothing / nowcasting / forecasting with a fitted state-space DFM (dfm_kalman_smooth).
ORACLE / TEST INFRASTRUCTURE ONLY (NumPy; validated by brute-force joint-Gaussian conditioning in
tests/test_oracle_forecast.py).

A forecast period is a period in which no series is observed: the E-step of oracle/kalman_em.py on the panel padded
with H all-NaN rows gives the smoothed factors of t <= T, the forecasts E[z_{T+h} | x] = M^h z_{T|T} and their
covariances, and the same log-likelihood as the unpadded panel.  The projection onto the series is
    common_it = lam_i' E[f_t | x]        (compute_series, dfm_functions.ipynb:552)
    xhat_it   = x_it where observed, common_it otherwise
    xvar_it   = 0 where observed, lam_i' Var[f_t | x] lam_i + R_i otherwise
Series whose loading row or R_i is NaN are out of the model: NaN in common / xhat / xvar.
"""
import numpy as np

from oracle import kalman_em as K


def smooth_forecast(X, Lam, R, A, Q, P0=None, p=1, H=0):
    """X (T, N) standardized with NaN; returns dict F (T+H, r), PF (T+H, r, r), common, xhat, xvar (T+H, N), loglik."""
    X = np.asarray(X, float); T, N = X.shape; r = Lam.shape[1]; k = r * p
    if P0 is None:
        Qt = np.zeros((k, k)); Qt[:r, :r] = Q
        P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    Xp = np.vstack([X, np.full((H, N), np.nan)])
    es = K.e_step(Xp, Lam, R, A, Q, P0, p)
    F = es["zs"][:, :r]; PF = es["Ps"][:, :r, :r]
    use = es["use"]
    common = F @ np.where(use[:, None], Lam, 0.0).T
    quad = np.einsum("ia,tab,ib->ti", np.where(use[:, None], Lam, 0.0), PF, np.where(use[:, None], Lam, 0.0))
    obs = ~np.isnan(Xp)
    xhat = np.where(obs, Xp, common)
    xvar = np.where(obs, 0.0, quad + np.where(use, R, 0.0)[None, :])
    for a_ in (common, xhat, xvar):
        a_[:, ~use] = np.nan
    return dict(F=F, PF=PF, common=common, xhat=xhat, xvar=xvar, loglik=es["loglik"], zs=es["zs"], Ps=es["Ps"])
