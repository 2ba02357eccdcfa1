"""FP64 spec of the simulation smoother (dfm_simulation_smoother): draws from the JOINT posterior of the factor path and the
missing cells, (f_1 .. f_{T+H}, x_missing) | x_observed, at fixed state-space parameters.  ORACLE / TEST INFRASTRUCTURE ONLY
(NumPy; validated by brute-force joint-Gaussian conditioning in tests/test_oracle_simsmooth.py).

Mean-corrected simulation smoother (Durbin & Koopman 2002) on the model of oracle/kalman_em.py, the panel padded with H
all-missing periods (Tp = T + H).  For one draw:
  1. z+_0 = L_P0 nu,  z+_t = M z+_{t-1} + E' L_Q eta_t                      (the state drawn unconditionally)
  2. c_t  = b_t(x) - C_t E z+_t - L_C,t xi_t                                  (the information of x - x+, never an N-wide x+:
        b_t(x+) = C_t f+_t + sum_{i obs} lam_i e+_it / R_i and the sum is N(0, C_t), independent of everything else)
  3. zhat = RTS smoother means of kalman_em.e_step with b_t replaced by c_t (same covariances)
  4. f~_t = E (z+_t + zhat_t)
  5. x~_it = x_it observed;  lam_i' f~_t + sqrt(R_i) eps_it missing;  NaN for a series out of the model.
L_S = unpivoted lower Cholesky factor of a PSD matrix; a pivot <= 1e-12 max_i S_ii counts as zero (its column is zeroed and
the elimination continues): C_t = 0 in forecast periods, rank-deficient C_t, a singular P0.
Normals: oracle.dgp.rng_normal(seed, draw id, stream, element), the numpy restatement of the device's Philox4x32-10
stream, on four stream tags after the replication generators' RNG_BETA (the table the device kernels use, include/dfm_b200.h):
  RNG_SS_Z0    7   nu      z+_0 = L_P0 nu                        element a          (a < k)
  RNG_SS_ETA   8   eta_t   state shocks of periods t >= 1        element t r + a    (a < r)
  RNG_SS_OBS   9   xi_t    the N(0, C_t) term of c_t             element t r + a    (a < r)
  RNG_SS_MISS 10   eps_it  idiosyncratic draw of a missing cell  element i Tp + t   (drawn for missing cells only)
"""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

from oracle import kalman_em as K
from oracle.dgp import rng_normal

RNG_SS_Z0, RNG_SS_ETA, RNG_SS_OBS, RNG_SS_MISS = 7, 8, 9, 10
PIVOT_TOL = 1e-12


def psd_cholesky(S):
    """Lower factor L with L L' = S of a PSD matrix; pivots <= PIVOT_TOL * max diag are zero columns."""
    A = np.array(S, float, copy=True); n = A.shape[0]
    tol = PIVOT_TOL * max(float(np.max(np.diag(A))) if n else 0.0, 0.0)
    L = np.zeros((n, n))
    for j in range(n):
        d = A[j, j]
        if not d > tol:
            continue
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = A[j + 1:, j] / L[j, j]
        A[j + 1:, j + 1:] -= np.outer(L[j + 1:, j], L[j + 1:, j])
    return L


def prepare(X, Lam, R, A, Q, P0, p, H):
    """Everything the draws share: the E-step's covariances, b_t, C_t and their factors."""
    X = np.asarray(X, float); T, N = X.shape; r = Lam.shape[1]; k = r * p; Tp = T + H
    if P0 is None:
        Qt = np.zeros((k, k)); Qt[:r, :r] = Q
        P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    Xp = np.vstack([X, np.full((H, N), np.nan)])
    es = K.e_step(Xp, Lam, R, A, Q, P0, p)
    use, obs = es["use"], es["obs"]
    Lam0 = np.where(use[:, None], Lam, 0.0)
    W = Lam0 * np.where(use, 1.0 / np.where(use, R, 1.0), 0.0)[:, None]
    B = np.where(obs, Xp, 0.0) @ W
    Ct = np.stack([Lam0[obs[t]].T @ W[obs[t]] for t in range(Tp)])
    return dict(Xp=Xp, Lam=Lam, R=R, use=use, obs=obs, M=K.companion(A, r, p), r=r, k=k, Tp=Tp, B=B, Ct=Ct,
                LC=np.stack([psd_cholesky(c) for c in Ct]), LP0=psd_cholesky(P0), LQ=psd_cholesky(Q), Pf=es["Pf"], Pp=es["Pp"],
                J=[cho_solve(cho_factor(es["Pp"][t + 1], lower=True), K.companion(A, r, p) @ es["Pf"][t]).T for t in range(Tp - 1)])


def draw_prepared(g, nu, eta, xi, eps):
    """One draw from the normals nu (k), eta (Tp, r; row 0 unused), xi (Tp, r), eps (N, Tp; read on missing cells only).
    Returns F (Tp, r) and the panel draw (Tp, N)."""
    r, k, Tp, M = g["r"], g["k"], g["Tp"], g["M"]
    zplus = np.zeros((Tp, k))
    zplus[0] = g["LP0"] @ nu
    for t in range(1, Tp):
        zplus[t] = M @ zplus[t - 1]
        zplus[t, :r] += g["LQ"] @ eta[t]
    zf = np.zeros((Tp, k))
    for t in range(Tp):
        c = g["B"][t] - g["Ct"][t] @ zplus[t, :r] - g["LC"][t] @ xi[t]
        zp = M @ zf[t - 1] if t > 0 else np.zeros(k)
        zf[t] = zp + g["Pf"][t][:, :r] @ (c - g["Ct"][t] @ zp[:r])
    zs = zf.copy()
    for t in range(Tp - 2, -1, -1):
        zs[t] = zf[t] + g["J"][t] @ (zs[t + 1] - M @ zf[t])
    F = zplus[:, :r] + zs[:, :r]
    use, Lam, R = g["use"], g["Lam"], g["R"]
    Lam0 = np.where(use[:, None], Lam, 0.0)
    miss = F @ Lam0.T + np.sqrt(np.where(use, R, 0.0))[None, :] * np.asarray(eps).T
    Xd = np.where(np.isnan(g["Xp"]), miss, g["Xp"])
    Xd[:, ~use] = np.nan
    return F, Xd


def draw_from_normals(X, Lam, R, A, Q, P0, p, H, nu, eta, xi, eps):
    """The algorithm of the module docstring given its normals (shapes as draw_prepared)."""
    return draw_prepared(prepare(X, Lam, R, A, Q, P0, p, H), nu, eta, xi, eps)


def normals(seed, draw_id, k, r, Tp, N):
    """The Philox normals draw `draw_id` consumes (nu, eta, xi, eps), element indices as in the table above."""
    nu = rng_normal(seed, draw_id, RNG_SS_Z0, np.arange(k))
    eta = rng_normal(seed, draw_id, RNG_SS_ETA, np.arange(Tp * r)).reshape(Tp, r)
    xi = rng_normal(seed, draw_id, RNG_SS_OBS, np.arange(Tp * r)).reshape(Tp, r)
    eps = rng_normal(seed, draw_id, RNG_SS_MISS, np.arange(N * Tp)).reshape(N, Tp)
    return nu, eta, xi, eps


def simulation_smoother(X, Lam, R, A, Q, P0, p, H, seed, draw_ids):
    """Draws draw_ids of stream `seed`: F (n, Tp, r) and panel draws (n, Tp, N)."""
    g = prepare(X, Lam, R, A, Q, P0, p, H)
    N = np.asarray(X).shape[1]
    out = [draw_prepared(g, *normals(seed, int(d), g["k"], g["r"], g["Tp"], N)) for d in draw_ids]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])
