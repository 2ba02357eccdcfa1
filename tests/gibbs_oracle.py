"""FP64 spec of the Gibbs sampler of the state-space DFM (dfm_gibbs).  ORACLE / TEST INFRASTRUCTURE ONLY (NumPy; checked in
tests/test_oracle_gibbs.py: Gamma sampler against scipy, conjugate steps against the analytic posteriors, and a Geweke (2004)
joint-distribution test of the whole sweep).

Model: the one oracle/kalman_em.py fits (standardized panel, NaN = missing, z_t = [f_t .. f_{t-p+1}], P0 HELD FIXED).
Prior (conjugate, proper, standardized units):
  lam_i | R_i ~ N(0, (R_i / kap_lam) I_r),  R_i ~ IG(a_R, b_R);   A' | Q ~ MN(0, I_k / kap_A, Q),  Q ~ IW(nu_Q, s_Q I_r).
Sweep s of chain c at theta = (Lam, R, A, Q), id = gibbs_id(c, s) = c 2^24 + s, Tp = T + H:
  1. factor step   (z~_0 .. z~_{Tp-1}, x~_missing) exactly as dfm_simulation_smoother's draw `id` at theta
                   (tests/simsmooth_oracle.py); the log-likelihood of theta comes from the same E-step.
  2. measurement   for each series in the model (Lam row and R_i not NaN), over its observed in-sample periods O_i (n_i):
                   S_i = sum f~ f~',  s_i = sum x f~,  q_i = sum x^2,  L_i = chol(kap_lam I + S_i),  m_i = L_i^-T L_i^-1 s_i,
                   alpha_i = a_R + n_i / 2,  beta_i = b_R + (q_i - s_i' m_i) / 2,
                   R_i = beta_i / Gamma(alpha_i, 1),  lam_i = m_i + sqrt(R_i) L_i^-T nu_i.   Series out of the model stay NaN.
  3. transition    Y_t = f~_t on Z_t = z~_{t-1} = [f~_{t-1} .. f~_{t-p}], t = 1 .. T-1 (in sample; the lag block of z~_0
                   supplies the pre-sample lags):  L_Z L_Z' = kap_A I + Z'Z,  B^ = (kap_A I + Z'Z)^-1 Z'Y,
                   S = s_Q I + Y'Y - B^' Z'Y,  nu = nu_Q + T - 1;  Q ~ IW(nu, S) by Bartlett: S = L L', B lower with
                   B_jj^2 = 2 Gamma((nu - j) / 2) (j = 0 .. r-1) and B_ij ~ N(0, 1) (i > j);  U = L B^-T,  Q = U U';
                   A' = B^ + L_Z^-T Xi L_Q',  L_Q = chol(Q),  Xi k x r standard normal.
  4. the forecast periods t >= T are drawn in step 1 only (the predictive output); they do not enter steps 2-3.
The panel draw x~ of a sweep is the simulation smoother's at the theta ENTERING the sweep (with the factor draw of that sweep);
the parameter record of a sweep is the theta LEAVING it.
Random numbers: oracle.dgp's Philox4x32-10 stream with replication id = gibbs_id(c, s); the factor step uses the simulation
smoother's tags 7-10 unchanged, the parameter step four new tags (the table of include/dfm_b200.h):
  RNG_GB_NU   14  nu_i                                    element i r + a          (a < r)
  RNG_GB_W    15  Bartlett B_ij (i > j), then Xi           element i + r j;  r^2 + a + k b   (a < k, b < r)
  RNG_GB_GN   16  normals of the Gamma sampler             element 64 e + j          (attempt j < 64 of Gamma number e)
  RNG_GB_GU   17  uniforms of the Gamma sampler            element 64 e + j
Gamma numbers e: e = i for R_i (i < N, read for series in the model only), e = N + j for the Bartlett diagonal B_jj (j < r).
Gamma(alpha >= 1, 1) is Marsaglia & Tsang (2000): d = alpha - 1/3, c = 1 / sqrt(9 d); attempt j: x = normal, v = (1 + c x)^3,
accept d v when v > 0 and (u < 1 - 0.0331 x^4 or log u < x^2 / 2 + d (1 - v + log v)).  If all 64 attempts are rejected the
sampler returns d (the mode region; the acceptance rate is >= 0.95 for alpha >= 1, so this has probability < 1e-80).
"""
import numpy as np
from scipy.linalg import solve_triangular

from oracle import kalman_em as K
from oracle.dgp import rng_normal, rng_uniform
from simsmooth_oracle import psd_cholesky, normals as sim_normals

RNG_GB_NU, RNG_GB_W, RNG_GB_GN, RNG_GB_GU = 14, 15, 16, 17
GAMMA_TRIES = 64
CHAIN_SHIFT = 24


def gibbs_id(c, s):
    return (int(c) << CHAIN_SHIFT) + int(s)


def default_prior(r):
    return dict(kap_lam=0.01, a_R=3.0, b_R=1.0, kap_A=0.01, nu_Q=r + 2.0, s_Q=1.0)


# ------------------------------------------------------------------------------------------------------------ Gamma sampler
def gamma_mt(alpha, seed, rid, e):
    """Gamma(alpha, 1) numbers e (array) of replication id rid; returns (values, fallback flags)."""
    alpha = np.broadcast_to(np.asarray(alpha, float), np.shape(e)).ravel()
    e = np.asarray(e, np.uint64).ravel()
    el = (e[:, None] * np.uint64(GAMMA_TRIES) + np.arange(GAMMA_TRIES, dtype=np.uint64)[None, :]).ravel()
    x = rng_normal(seed, rid, RNG_GB_GN, el).reshape(-1, GAMMA_TRIES)
    u = rng_uniform(seed, rid, RNG_GB_GU, el).reshape(-1, GAMMA_TRIES)
    d = alpha - 1.0 / 3.0
    c = 1.0 / np.sqrt(9.0 * d)
    t = 1.0 + c[:, None] * x
    v = t * t * t
    with np.errstate(invalid="ignore", divide="ignore"):
        ok = (v > 0) & ((u < 1.0 - 0.0331 * (x * x) * (x * x)) | (np.log(u) < 0.5 * x * x + d[:, None] * (1.0 - v + np.log(v))))
    first = np.argmax(ok, axis=1)
    hit = ok[np.arange(len(e)), first]
    out = np.where(hit, d * v[np.arange(len(e)), first], d)
    return out, ~hit


# ------------------------------------------------------------------------------------------------------------ factor step
def prepare(Xp, Lam, R, A, Q, P0, p):
    """The simulation smoother's shared matrices (simsmooth_oracle.prepare) on an already padded panel, plus the loglik."""
    Tp, N = Xp.shape; r = Lam.shape[1]; k = r * p
    es = K.e_step(Xp, Lam, R, A, Q, P0, p)
    use, obs = es["use"], es["obs"]
    Lam0 = np.where(use[:, None], Lam, 0.0)
    W = Lam0 * np.where(use, 1.0 / np.where(use, R, 1.0), 0.0)[:, None]
    B = np.where(obs, Xp, 0.0) @ W
    Ct = np.stack([Lam0[obs[t]].T @ W[obs[t]] for t in range(Tp)])
    M = K.companion(A, r, p)
    J = [np.linalg.solve(es["Pp"][t + 1], M @ es["Pf"][t]).T for t in range(Tp - 1)]
    return dict(Xp=Xp, Lam=Lam, R=R, use=use, M=M, r=r, k=k, Tp=Tp, B=B, Ct=Ct, LC=np.stack([psd_cholesky(c) for c in Ct]),
                LP0=psd_cholesky(P0), LQ=psd_cholesky(Q), Pf=es["Pf"], J=J, loglik=float(es["loglik"]))


def draw_states(g, nu, eta, xi, eps):
    """simsmooth_oracle.draw_prepared, returning the whole state path z~ (Tp, k) as well."""
    r, k, Tp, M = g["r"], g["k"], g["Tp"], g["M"]
    zplus = np.zeros((Tp, k)); zplus[0] = g["LP0"] @ nu
    for t in range(1, Tp):
        zplus[t] = M @ zplus[t - 1]; zplus[t, :r] += g["LQ"] @ eta[t]
    zf = np.zeros((Tp, k))
    for t in range(Tp):
        c = g["B"][t] - g["Ct"][t] @ zplus[t, :r] - g["LC"][t] @ xi[t]
        zp = M @ zf[t - 1] if t > 0 else np.zeros(k)
        zf[t] = zp + g["Pf"][t][:, :r] @ (c - g["Ct"][t] @ zp[:r])
    zs = zf.copy()
    for t in range(Tp - 2, -1, -1):
        zs[t] = zf[t] + g["J"][t] @ (zs[t + 1] - M @ zf[t])
    Z = zplus + zs
    F = Z[:, :r]
    use, Lam, R = g["use"], g["Lam"], g["R"]
    Lam0 = np.where(use[:, None], Lam, 0.0)
    miss = F @ Lam0.T + np.sqrt(np.where(use, R, 0.0))[None, :] * np.asarray(eps).T
    Xd = np.where(np.isnan(g["Xp"]), miss, g["Xp"])
    Xd[:, ~use] = np.nan
    return Z, Xd


# ------------------------------------------------------------------------------------------------------------ parameter step
def in_model(Lam, R):
    return ~np.isnan(Lam).any(axis=1) & ~np.isnan(R)


def regression(Z, T, r, p):
    """(Y, Zl) of the transition step from the state path Z (Tp, k): rows t = 1 .. T-1, Zl_t = [f~_{t-1} .. f~_{t-p}] with
    f~_{-j} the j-th lag block of z~_0."""
    fext = np.vstack([Z[0, j * r:(j + 1) * r] for j in range(p - 1, 0, -1)] + [Z[:T, :r]]) if p > 1 else Z[:T, :r]
    o = p - 1                                                            # row of f~_0 in fext
    Zl = np.hstack([fext[o - l:o - l + T - 1] for l in range(p)])
    return Z[1:T, :r], Zl


def draw_params(X, Z, use, p, prior, seed, rid, return_fallback=False):
    """Steps 2-3 at the path Z (Tp, k) on the in-sample panel X (T, N).  Returns dict(Lam, R, A, Q)."""
    T, N = X.shape; r = Z.shape[1] // p; k = r * p
    F = Z[:T, :r]
    obs = ~np.isnan(X)
    Lam = np.full((N, r), np.nan); R = np.full(N, np.nan)
    nu = rng_normal(seed, rid, RNG_GB_NU, np.arange(N * r)).reshape(N, r)
    idx = np.flatnonzero(use)
    alphas, betas, Ls, ms = [], [], [], []
    for i in idx:
        o = obs[:, i]
        Fi = F[o]; xi = X[o, i]
        Si = Fi.T @ Fi; si = Fi.T @ xi; qi = xi @ xi
        Li = np.linalg.cholesky(prior["kap_lam"] * np.eye(r) + Si)
        mi = solve_triangular(Li, solve_triangular(Li, si, lower=True), lower=True, trans="T")
        alphas.append(prior["a_R"] + 0.5 * o.sum()); betas.append(prior["b_R"] + 0.5 * (qi - si @ mi)); Ls.append(Li); ms.append(mi)
    fb = np.zeros(0, bool)
    if len(idx):
        gam, fb = gamma_mt(np.array(alphas), seed, rid, idx)
        for j, i in enumerate(idx):
            R[i] = betas[j] / gam[j]
            Lam[i] = ms[j] + np.sqrt(R[i]) * solve_triangular(Ls[j], nu[i], lower=True, trans="T")
    # transition
    Y, Zl = regression(Z, T, r, p)
    G = prior["kap_A"] * np.eye(k) + Zl.T @ Zl
    LZ = np.linalg.cholesky(G)
    ZY = Zl.T @ Y
    Bh = solve_triangular(LZ, solve_triangular(LZ, ZY, lower=True), lower=True, trans="T")
    S = prior["s_Q"] * np.eye(r) + Y.T @ Y - Bh.T @ ZY
    S = 0.5 * (S + S.T)
    nuQ = prior["nu_Q"] + T - 1
    w = rng_normal(seed, rid, RNG_GB_W, np.arange(r * r + k * r))
    Bm = np.tril(w[:r * r].reshape(r, r).T, -1)                          # B_ij = w[i + r j], i > j
    chi, fb2 = gamma_mt(0.5 * (nuQ - np.arange(r)), seed, rid, N + np.arange(r))
    Bm[np.arange(r), np.arange(r)] = np.sqrt(2.0 * chi)
    LS = np.linalg.cholesky(S)
    U = solve_triangular(Bm, LS.T, lower=True).T                         # L B^-T
    Qn = U @ U.T
    Qn = 0.5 * (Qn + Qn.T)
    LQ = np.linalg.cholesky(Qn)
    Xi = w[r * r:].reshape(r, k).T                                       # Xi[a, b] = w[r^2 + a + k b]
    At = Bh + solve_triangular(LZ, Xi, lower=True, trans="T") @ LQ.T
    out = dict(Lam=Lam, R=R, A=np.ascontiguousarray(At.T), Q=Qn)
    if return_fallback:
        out["fallback"] = int(fb.sum() + fb2.sum())
    return out


# ------------------------------------------------------------------------------------------------------------ chains
def sweep(X, theta, p, H, prior, seed, rid):
    """One sweep at theta (dict Lam, R, A, Q, P0).  Returns (new theta, F (Tp, r), x~ (Tp, N), loglik of theta, z~_0)."""
    X = np.asarray(X, float); T, N = X.shape; r = theta["Lam"].shape[1]; k = r * p; Tp = T + H
    Xp = np.vstack([X, np.full((H, N), np.nan)])
    g = prepare(Xp, theta["Lam"], theta["R"], theta["A"], theta["Q"], theta["P0"], p)
    Z, Xd = draw_states(g, *sim_normals(seed, rid, k, r, Tp, N))
    new = draw_params(X, Z, in_model(theta["Lam"], theta["R"]), p, prior, seed, rid)
    new["P0"] = theta["P0"]
    return new, Z[:, :r].copy(), Xd, g["loglik"], Z[0].copy()


def chain(X, theta, p, prior, seed, c, sweep0, n_burn, n_keep, thin=1, H=0):
    """The records of chain c (dfm_gibbs' layout): kept Lam, R, A, Q, F, X, and the loglik trace of every sweep."""
    n_sweep = n_burn + n_keep * thin
    th = dict(theta)
    keep = {n: [] for n in ("Lam", "R", "A", "Q", "F", "X")}
    ll = []
    for j in range(n_sweep):
        s = sweep0 + j
        new, F, Xd, l, _ = sweep(X, th, p, H, prior, seed, gibbs_id(c, s))
        ll.append(l)
        if j >= n_burn and (j - n_burn + 1) % thin == 0:
            for n in ("Lam", "R", "A", "Q"):
                keep[n].append(new[n])
            keep["F"].append(F); keep["X"].append(Xd)
        th = new
    out = {n: np.stack(v) if v else None for n, v in keep.items()}
    out["loglik"] = np.array(ll)
    return out


# ------------------------------------------------------------------------------------------------------------ diagnostics
def split_rhat(draws):
    """Split-R^ (Gelman et al. 2013, BDA3 11.4) of draws (n_chain, n) along axis 1; trailing axes are kept."""
    d = np.asarray(draws, float)
    n = d.shape[1] // 2
    if n < 2:
        return np.full(d.shape[2:], np.nan)
    s = np.concatenate([d[:, :n], d[:, n:2 * n]], axis=0)
    m = s.shape[0]
    cm = s.mean(axis=1)
    B = n * cm.var(axis=0, ddof=1)
    W = s.var(axis=1, ddof=1).mean(axis=0)
    var = (n - 1) / n * W + B / n
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.sqrt(var / W)
