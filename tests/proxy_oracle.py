"""FP64 spec of dfm_proxy_identification: shocks of a state-space DFM identified by external instruments (proxy SVAR / SVAR-IV,
Stock & Watson 2018), with a moving-block bootstrap of the instrument moments.  ORACLE / TEST INFRASTRUCTURE ONLY (NumPy;
checked in tests/test_oracle_proxy.py).

One model (Lam N x r, R N, A = [A_1 .. A_p] r x k, Q r x r) and a factor path F (Tp x r): L = chol(Q), Psi_h by explicit matrix
powers (identified_oracle.psi), c_{i,h} = lam_i' Psi_h.
  eta_t = f_t - sum_l A_l f_{t-l} (direct residuals, t >= p), u_t = L^-1 eta_t.
  Instrument k: T_k = {t >= p : z_t finite}; a NaN in f_t .. f_{t-p} at a period of T_k fails the pair (status 3), as do n_k < 3
  and Gamma_k = 0.  zbar, s^2 = mean (z - zbar)^2, Gamma = mean eta_t (z_t - zbar), g = L^-1 Gamma, omega = g / |g|.
  eps_t = omega' u_t; resp[i,h] = scale_i c_{i,h} omega; fevd[i,h] = sum_{l<=h} (c_{i,l} omega)^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i);
  reliability = |g|^2 / s^2; first stage: y = lam_i0' eta on [1, z], F = pi^2 / hac(v, X, q)[1, 1] (oracle.dfm_ref.hac).
  Replicate rho >= 1: l = min(block, n), ceil(n / l) starts floor(u_j (n - l + 1)), u_j = rng_uniform(seed, id, 20,
  (rho n_inst + k) Tp + j); the blocks of T_k's (eta, z) pairs concatenated, cut at n; omega* from Gamma* as above.
Status order: 3 (A / Q NaN, Q not PD), 1 (series i0 out of the model), 3 (path NaN in T_k, n_k < 3, Gamma = 0).
"""
import numpy as np
from scipy.linalg import solve_triangular

import identified_oracle as IO
from oracle.dfm_ref import hac
from oracle.dgp import rng_uniform

RNG_PROXY = 20


def innovations(A, F, p):
    """eta (Tp, r): f_t - sum_l A_l f_{t-l} for t >= p, NaN before (and wherever the path has a NaN)."""
    F = np.asarray(F, float); Tp, r = F.shape
    eta = np.full((Tp, r), np.nan)
    for t in range(p, Tp):
        e = F[t].copy()
        for l in range(1, p + 1):
            e = e - A[:, (l - 1) * r:l * r] @ F[t - l]
        eta[t] = e
    return eta


def periods(z, F, p):
    """(T_k as row indices, whether a NaN in the path touches it)."""
    Tp = len(z)
    Fb = np.isnan(np.asarray(F, float)).any(axis=1)
    T, bad = [], False
    for t in range(p, Tp):
        if np.isfinite(z[t]):
            if Fb[t - p:t + 1].any():
                bad = True
            else:
                T.append(t)
    return np.array(T, int), bad


def omega_of(eta, z, Lc):
    """(omega, |L^-1 Gamma|^2, s^2) of the sample (eta (n, r), z (n,))."""
    zb = z.mean()
    G = (eta * (z - zb)[:, None]).mean(axis=0)
    g = solve_triangular(Lc, G, lower=True)
    n2 = float(g @ g)
    return (g / np.sqrt(n2) if n2 > 0 else np.full(len(g), np.nan)), n2, float(((z - zb) ** 2).mean())


def block_indices(n, block, seed, mid, k, rho, n_inst, Tp):
    """The resampled positions 0 .. n-1 of replicate rho of instrument k."""
    l = min(block, n)
    nb = -(-n // l)
    e = (np.uint64(rho) * np.uint64(n_inst) + np.uint64(k)) * np.uint64(Tp) + np.arange(nb, dtype=np.uint64)
    s = np.floor(rng_uniform(seed, mid, RNG_PROXY, e) * (n - l + 1)).astype(int)
    return (s[:, None] + np.arange(l)[None, :]).ravel()[:n]


def first_stage(y, z, q):
    """(pi, F) of y on [1, z] with hac(v, X, q)."""
    X = np.column_stack([np.ones(len(z)), z])
    beta = np.linalg.lstsq(X, y, rcond=None)[0]
    V, _ = hac(y - X @ beta, X, q)
    return beta[1], beta[1] ** 2 / V[1, 1]


def identify(Lam, R, A, Q, F, Z, p, H, i0, q=0, block=1, n_boot=0, seed=0, mid=0, scale=None):
    """dfm_proxy_identification on one model: dict omega (ni, 1 + n_boot, r), resp / fevd (ni, 1 + n_boot, N, H), eps (ni, Tp),
    n_obs, reliability, fs_pi, fs_F, status (ni,)."""
    Lam = np.asarray(Lam, float); R = np.asarray(R, float); N, r = Lam.shape
    F = np.asarray(F, float); Tp = F.shape[0]
    Z = np.asarray(Z, float).reshape(Tp, -1); ni = Z.shape[1]
    nr = 1 + n_boot
    out = dict(omega=np.full((ni, nr, r), np.nan), resp=np.full((ni, nr, N, H), np.nan), fevd=np.full((ni, nr, N, H), np.nan),
               eps=np.full((ni, Tp), np.nan), n_obs=np.zeros(ni, int), reliability=np.full(ni, np.nan), fs_pi=np.full(ni, np.nan),
               fs_F=np.full(ni, np.nan), status=np.zeros(ni, int))
    model_bad = np.isnan(A).any() or np.isnan(Q).any()
    if not model_bad:
        try:
            Lc = np.linalg.cholesky(Q)
            P = IO.psi(A, Q, p, H)
        except np.linalg.LinAlgError:
            model_bad = True
    i0_out = np.isnan(Lam[i0]).any() or np.isnan(R[i0])
    eta = innovations(A, F, p) if not model_bad else None
    sc = np.ones(N) if scale is None else np.asarray(scale, float)
    inm = ~np.isnan(Lam).any(axis=1) & ~np.isnan(R)
    for k in range(ni):
        z = Z[:, k]
        T, pbad = periods(z, F, p)
        n = len(T)
        out["n_obs"][k] = n
        if model_bad:
            out["status"][k] = 3; continue
        if i0_out:
            out["status"][k] = 1; continue
        if pbad or n < 3:
            out["status"][k] = 3; continue
        om, n2, s2 = omega_of(eta[T], z[T], Lc)
        if not n2 > 0:
            out["status"][k] = 3; continue
        out["reliability"][k] = n2 / s2
        out["fs_pi"][k], out["fs_F"][k] = first_stage(eta[T] @ Lam[i0], z[T], q)
        u = solve_triangular(Lc, eta[p:].T, lower=True, check_finite=False).T
        out["eps"][k, p:] = u @ om
        for rho in range(nr):
            if rho == 0:
                w = om
            else:
                ix = block_indices(n, block, seed, mid, k, rho, ni, Tp)
                w = omega_of(eta[T][ix], z[T][ix], Lc)[0]
            out["omega"][k, rho] = w
            if np.isnan(w).any():
                continue
            c = np.einsum("ia,hab->ihb", Lam, P)                              # c_{i,h} (N, H, r)
            cw = c @ w
            fe = np.cumsum(cw ** 2, axis=1) / (np.cumsum((c ** 2).sum(axis=2), axis=1) + R[:, None])
            out["resp"][k, rho] = np.where(inm[:, None], sc[:, None] * cw, np.nan)
            out["fevd"][k, rho] = np.where(inm[:, None], fe, np.nan)
    return out
