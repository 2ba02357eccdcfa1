"""FP64 spec of the Gibbs sampler under linear restrictions on the loadings (dfm_gibbs_constrained) and of the series responses
and forecast-error variance decompositions (dfm_series_responses).  ORACLE / TEST INFRASTRUCTURE ONLY (NumPy; checked in
tests/test_oracle_identified.py).

Restrictions: constr = (index, H (n_c x r), h) in standardized units, row q saying H[q] @ lam_{index[q]} = h[q] (the CSR of
dfm_em_kalman_constrained).  Model, prior and random numbers are tests/gibbs_oracle.py's; for a restricted series i in the model
(rows H_i, values h_i, m_i <= r) the prior on lam_i is N(0, R_i / kap_lam I) CONDITIONED on H_i lam_i = h_i, so that with
S~ = kap_lam I + S_i, L_i = chol(S~), Y = S~^-1 H_i', G = H_i Y, m_i = S~^-1 s_i and h0 = H_i' (H_i H_i')^-1 h_i:
  lam*_i = m_i - Y G^-1 (H_i m_i - h_i)
  beta_i = b_R + (q_i - 2 s_i' lam*_i + lam*_i' S~ lam*_i - kap_lam |h0|^2) / 2
         = b_R + (sum_obs (x_it - lam*_i' f~_t)^2 + kap_lam |lam*_i - h0|^2) / 2   (>= b_R)
  R_i    = beta_i / Gamma(a_R + n_i / 2)       (the r - m_i free dimensions of lam_i cancel from the shape)
  lam_i  = lam_u - Y G^-1 (H_i lam_u - h_i),   lam_u = m_i + sqrt(R_i) L_i^-T nu_i  (the unrestricted draw, projected)
         ~ N(lam*_i, R_i (S~^-1 - Y G^-1 Y'))
with the unrestricted series' random numbers (tag 14 elements i r + a, Gamma number e = i).  Unrestricted series, the factor
step and the transition step are gibbs_oracle's.

Responses of one model (Lam N x r, R N, A r x k, Q r x r): L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L (M the companion matrix of A),
c_{i,h} = lam_i' Psi_h, and for the leading n_shock shocks
  resp[i,h,j] = scale_i c_{i,h,j},   fevd[i,h,j] = sum_{l<=h} c_{i,l,j}^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i)
(the share of the (h+1)-step forecast-error variance of x_i due to shock j; sum_j fevd + R_i / (...) = 1 at n_shock = r).
Series out of the model (NaN Lam row or R_i) are NaN; a model whose A or Q holds a NaN or whose Q is not positive definite is
NaN throughout (status 3).
"""
import numpy as np
from scipy.linalg import solve_triangular

import gibbs_oracle as O
from oracle import kalman_em as K
from oracle.dgp import rng_normal
from simsmooth_oracle import normals as sim_normals


def rows_of(constr, i):
    """(H_i (m x r), h_i (m,)) of series i, rows in their given order."""
    idx, H, h = constr
    sel = np.flatnonzero(np.asarray(idx) == i)
    return np.asarray(H, float)[sel], np.asarray(h, float)[sel]


def correct(lam, Sinv, Hi, hi):
    """The EM's correction lam - Y G^-1 (H lam - h), Y = Sinv H', G = H Y."""
    Y = Sinv @ Hi.T
    return lam - Y @ np.linalg.solve(Hi @ Y, Hi @ lam - hi)


def restricted_moments(X, F, i, Hi, hi, prior):
    """(alpha, beta, lam*, Cov(lam | R) / R) of a restricted series i at the factor path F (T, r)."""
    r = F.shape[1]
    o = ~np.isnan(X[:, i])
    Fi, xi = F[o], X[o, i]
    St = prior["kap_lam"] * np.eye(r) + Fi.T @ Fi
    si, qi = Fi.T @ xi, xi @ xi
    Sinv = np.linalg.inv(St)
    ls = correct(np.linalg.solve(St, si), Sinv, Hi, hi)
    h0 = Hi.T @ np.linalg.solve(Hi @ Hi.T, hi)
    beta = prior["b_R"] + 0.5 * (qi - 2 * si @ ls + ls @ St @ ls - prior["kap_lam"] * h0 @ h0)
    Y = Sinv @ Hi.T
    return prior["a_R"] + 0.5 * o.sum(), beta, ls, Sinv - Y @ np.linalg.solve(Hi @ Y, Y.T)


def draw_params(X, Z, use, p, prior, seed, rid, constr=None):
    """gibbs_oracle.draw_params with the restricted series of `constr` drawn from their restricted conditional."""
    out = O.draw_params(X, Z, use, p, prior, seed, rid)
    if constr is None or len(constr[0]) == 0:
        return out
    T, N = X.shape; r = Z.shape[1] // p
    F = Z[:T, :r]
    obs = ~np.isnan(X)
    nu = rng_normal(seed, rid, O.RNG_GB_NU, np.arange(N * r)).reshape(N, r)
    for i in sorted(set(int(v) for v in constr[0])):
        if not use[i]:
            continue
        Hi, hi = rows_of(constr, i)
        o = obs[:, i]
        Fi, xi = F[o], X[o, i]
        St = prior["kap_lam"] * np.eye(r) + Fi.T @ Fi
        Li = np.linalg.cholesky(St)
        Sinv = np.linalg.inv(St)
        alpha, beta, ls, _ = restricted_moments(X, F, i, Hi, hi, prior)
        gam, _ = O.gamma_mt(np.array([alpha]), seed, rid, np.array([i]))
        Ri = beta / gam[0]
        mi = solve_triangular(Li, solve_triangular(Li, Fi.T @ xi, lower=True), lower=True, trans="T")
        lam_u = mi + np.sqrt(Ri) * solve_triangular(Li, nu[i], lower=True, trans="T")
        out["R"][i] = Ri
        out["Lam"][i] = correct(lam_u, Sinv, Hi, hi)
    return out


def sweep(X, theta, p, H, prior, seed, rid, constr=None):
    """gibbs_oracle.sweep with the restricted parameter step."""
    X = np.asarray(X, float); T, N = X.shape; r = theta["Lam"].shape[1]; k = r * p; Tp = T + H
    Xp = np.vstack([X, np.full((H, N), np.nan)])
    g = O.prepare(Xp, theta["Lam"], theta["R"], theta["A"], theta["Q"], theta["P0"], p)
    Z, Xd = O.draw_states(g, *sim_normals(seed, rid, k, r, Tp, N))
    new = draw_params(X, Z, O.in_model(theta["Lam"], theta["R"]), p, prior, seed, rid, constr)
    new["P0"] = theta["P0"]
    return new, Z[:, :r].copy(), Xd, g["loglik"], Z[0].copy()


def chain(X, theta, p, prior, seed, c, sweep0, n_burn, n_keep, thin=1, H=0, constr=None):
    """gibbs_oracle.chain under the restrictions."""
    n_sweep = n_burn + n_keep * thin
    th = dict(theta)
    keep = {n: [] for n in ("Lam", "R", "A", "Q", "F", "X")}
    ll = []
    for j in range(n_sweep):
        new, F, Xd, l, _ = sweep(X, th, p, H, prior, seed, O.gibbs_id(c, sweep0 + j), constr)
        ll.append(l)
        if j >= n_burn and (j - n_burn + 1) % thin == 0:
            for n in ("Lam", "R", "A", "Q"):
                keep[n].append(new[n])
            keep["F"].append(F); keep["X"].append(Xd)
        th = new
    out = {n: np.stack(v) if v else None for n, v in keep.items()}
    out["loglik"] = np.array(ll)
    return out


# ------------------------------------------------------------------------------------------------------------ responses
def psi(A, Q, p, H):
    """Psi_h = [M^h]_{1:r,1:r} chol(Q), (H, r, r), by explicit matrix powers."""
    r = Q.shape[0]
    M = K.companion(A, r, p)
    L = np.linalg.cholesky(Q)
    out, Mh = [], np.eye(M.shape[0])
    for _ in range(H):
        out.append(Mh[:r, :r] @ L)
        Mh = M @ Mh
    return np.stack(out)


def responses(Lam, R, A, Q, p, H, n_shock=None, scale=None):
    """(resp, fevd, status) of one model: resp / fevd (N, H, n_shock)."""
    Lam = np.asarray(Lam, float); N, r = Lam.shape
    ns = r if n_shock is None else n_shock
    nan = np.full((N, H, ns), np.nan)
    if np.isnan(A).any() or np.isnan(Q).any():
        return nan, nan.copy(), 3
    try:
        P = psi(A, Q, p, H)
    except np.linalg.LinAlgError:
        return nan, nan.copy(), 3
    c = np.einsum("ia,hab->ihb", Lam, P)                                  # (N, H, r)
    cum = np.cumsum(c ** 2, axis=1)
    den = cum.sum(axis=2) + np.asarray(R, float)[:, None]
    sc = np.ones(N) if scale is None else np.asarray(scale, float)
    resp = sc[:, None, None] * c[:, :, :ns]
    fevd = cum[:, :, :ns] / den[:, :, None]
    out = O.in_model(Lam, R)
    resp[~out] = np.nan; fevd[~out] = np.nan
    return resp, fevd, 0


def idiosyncratic_share(Lam, R, A, Q, p, H):
    """R_i / (sum_{l<=h} |c_{i,l}|^2 + R_i), (N, H)."""
    c = np.einsum("ia,hab->ihb", np.asarray(Lam, float), psi(A, Q, p, H))
    return np.asarray(R, float)[:, None] / (np.cumsum(c ** 2, axis=1).sum(axis=2) + np.asarray(R, float)[:, None])


def rotate(Lam, A, Q, Km, p):
    """The model f -> K f: Lam K^-1, A_l -> K A_l K^-1, Q -> K Q K'."""
    r = Q.shape[0]
    Ki = np.linalg.inv(Km)
    An = np.hstack([Km @ A[:, l * r:(l + 1) * r] @ Ki for l in range(p)])
    return Lam @ Ki, An, Km @ Q @ Km.T
