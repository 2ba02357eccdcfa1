"""Restatement of the reference's dfm_functions.ipynb (non-parametric DFM path).  ORACLE ONLY.

FP64 numpy/scipy; missing = NaN; arrays are (T, N) with the same orientation as the
Julia code.  Citations are raw JSON line numbers of dfm_functions.ipynb.  The
control flow deliberately mirrors the reference (per-series / per-period small
pivoted-QR least squares, `X\\y` -> LAPACK gelsy) so that it is also the honest
"restated-reference" CPU baseline.

PINNED by tests/test_oracle_golden.py against the stored outputs of
Stock_Watson.ipynb (Tables 2A/2B/2C/3/5).
"""
from dataclasses import dataclass, field
import numpy as np
import scipy.linalg as sla


# ----------------------------------------------------------------- helpers
def drop_missing_row(A):
    """:155-158"""
    keep = ~np.isnan(A).any(axis=1)
    return A[keep], keep


def drop_missing_col(A):
    """:167-170"""
    keep = ~np.isnan(A).any(axis=0)
    return A[:, keep], keep


def pca_score(X, nfac):
    """:179-183  full SVD, score = (X V)[:, :nfac]."""
    _, _, Vt = np.linalg.svd(X, full_matrices=False)
    return (X @ Vt.T)[:, :nfac]


def ols(y, X):
    """:205-210  b = X\\y (Julia: pivoted QR for non-square X) ; e = y - X b."""
    b = sla.lstsq(X, y, lapack_driver="gelsy", cond=None)[0]
    return b, y - X @ b


def ols_skipmissing_balanced(y, X):
    """:242-252  rows with any missing in [y X] are dropped."""
    y2 = y.reshape(len(y), -1)
    keep = ~(np.isnan(y2).any(axis=1) | np.isnan(X).any(axis=1))
    b, e = ols(y2[keep], X[keep])
    if y.ndim == 1:
        b, e = b[:, 0], e[:, 0]
    return b, e, keep


def ols_skipmissing_unbalanced(Y, X):
    """:271-286  column-by-column balanced OLS; e has NaN where dropped."""
    T, N = Y.shape
    b = np.empty((X.shape[1], N)); e = np.full((T, N), np.nan); used = np.zeros((T, N), bool)
    for i in range(N):
        bi, ei, keep = ols_skipmissing_balanced(Y[:, i], X)
        b[:, i] = bi; e[keep, i] = ei; used[:, i] = keep
    return b, e, used


def lagmat(X, lags):
    """:295-303"""
    X = X.reshape(len(X), -1)
    nc = X.shape[1]
    out = np.full((X.shape[0], nc * len(lags)), np.nan)
    for i, lag in enumerate(lags):
        if lag == 0:
            out[:, nc * i:nc * (i + 1)] = X
        else:
            out[lag:, nc * i:nc * (i + 1)] = X[:-lag]
    return out


def uar(y, n_lags):
    """:305-311  AR(n_lags) on a gap-free residual vector; ser uses len(y)-n_lags dof."""
    x = lagmat(y, list(range(1, n_lags + 1)))
    arcoef, ehat, _ = ols_skipmissing_balanced(y, x)
    ssr = float(ehat @ ehat)
    return arcoef, np.sqrt(ssr / (x.shape[0] - x.shape[1]))


def standardize_data(data):
    """:501-509  per-column mean / population std over non-missing."""
    mean = np.nanmean(data, axis=0)
    n = (~np.isnan(data)).sum(axis=0)
    std = np.nanstd(data, axis=0, ddof=1) * np.sqrt((n - 1) / n)
    return (data - mean) / std, std


def compute_r2(y, e):
    """:565-569"""
    ssr = float(e @ e); d = y - y.mean(); tss = float(d @ d)
    return 1 - ssr / tss, ssr, tss


# ----------------------------------------------------------------- constraints
@dataclass
class LambdaConstraint:
    """:1063-1068"""
    indices: np.ndarray      # 0-based series index per constraint row
    R: np.ndarray
    r: np.ndarray
    r_std: np.ndarray


def construct_constraint(varnames, used_varnames, R, r):
    """:1090-1102"""
    used = list(used_varnames)
    n_R = R.shape[0]
    idx = np.array([used.index(v) for v in varnames for _ in range(n_R)])
    return LambdaConstraint(idx, np.tile(R, (len(varnames), 1)), np.tile(r, len(varnames)),
                            np.zeros(len(varnames) * n_R))


def standardize_constraint(c, xdatastd):
    """:1182-1186"""
    if c is not None:
        c.r_std[:] = c.r / xdatastd[c.indices]


def impose_constraint(b, i, X, c, forwhat):
    """:1125-1141  restricted LS correction, in place on b."""
    if c is None:
        return
    used = c.indices == i
    if not used.any():
        # Julia: empty R_tmp -> 0-row algebra leaves b unchanged
        return
    if forwhat == "factor":
        R, r = c.R[used], c.r_std[used]
    else:
        R, r = np.hstack([c.R[used], np.zeros((used.sum(), 1))]), c.r[used]
    tmp = np.linalg.solve(X.T @ X, R.T)
    b -= tmp @ np.linalg.solve(R @ tmp, R @ b - r)


# ----------------------------------------------------------------- model containers
@dataclass
class VARModel:
    """:43-57, ctor :424-435.  `y` aliases DFMModel.factor."""
    y: np.ndarray
    nlag: int = 1
    withconst: bool = True
    initperiod: int = 1          # 1-based inclusive, as in the reference
    lastperiod: int = 0
    resid: np.ndarray = None
    betahat: np.ndarray = None
    M: np.ndarray = None
    Q: np.ndarray = None
    G: np.ndarray = None
    seps: np.ndarray = None

    def __post_init__(self):
        T, ns = self.y.shape
        if self.lastperiod == 0:
            self.lastperiod = T
        k = ns * self.nlag
        self.resid = np.full((T, ns), np.nan)
        self.betahat = np.full((k + int(self.withconst), ns), np.nan)
        self.M = np.full((k, k), np.nan); self.Q = np.full((ns, k), np.nan)
        self.G = np.full((k, ns), np.nan); self.seps = np.full((ns, ns), np.nan)


@dataclass
class FactorEstimateStats:
    """:66-73"""
    T: int
    ns: int
    nobs: float = np.nan
    tss: float = np.nan
    ssr: float = np.nan
    R2: np.ndarray = None
    iters: int = 0               # not in the reference (it is silent); kept for parity checks


class DFMModel:
    """:89-111, ctor :120-146."""

    def __init__(self, data, inclcode, nt_min_factor_estimation, nt_min_factorloading_estimation,
                 initperiod, lastperiod, nfac_o, nfac_u, tol, n_uarlag, n_factorlag):
        data = np.asarray(data, float); inclcode = np.asarray(inclcode).ravel()
        if data.shape[1] != len(inclcode):
            raise ValueError("length of inclcode must equal to number of data series")
        if not initperiod < lastperiod:
            raise ValueError("initperiod must be smaller than lastperiod")
        if not (n_uarlag > 0 and n_factorlag > 0):
            raise ValueError("n_uarlag and n_factorlag must be positive")
        self.data, self.inclcode = data, inclcode
        self.T, self.ns = data.shape
        self.nt_min_factor_estimation = nt_min_factor_estimation
        self.nt_min_factorloading_estimation = nt_min_factorloading_estimation
        self.initperiod, self.lastperiod = initperiod, lastperiod
        self.nfac_o, self.nfac_u, self.nfac_t = nfac_o, nfac_u, nfac_o + nfac_u
        self.tol, self.n_uarlag, self.n_factorlag = tol, n_uarlag, n_factorlag
        nest = int((inclcode == 1).sum())
        self.fes = FactorEstimateStats(lastperiod - initperiod + 1, nest, R2=np.full(nest, np.nan))
        self.factor = np.full((self.T, self.nfac_t), np.nan)
        self.lambda_ = np.full((self.ns, self.nfac_t), np.nan)
        self.uar_coef = np.full((self.ns, n_uarlag), np.nan)
        self.uar_ser = np.full(self.ns, np.nan)
        self.r2 = np.full(self.ns, np.nan)
        self.factor_var_model = VARModel(self.factor, n_factorlag, True, initperiod, lastperiod)
        self.lambda_est = None   # the loop-local lambda of estimate_factor! (:351), kept for checks


# ----------------------------------------------------------------- a7: ALS / least-squares EM
def estimate_factor(m, max_iter=100000000, computeR2=True, lam_constr=None, f_init=None):
    """estimate_factor!  :328-382."""
    i0, i1, nt_min, nfac_u, nfac_o, tol = (m.initperiod, m.lastperiod, m.nt_min_factor_estimation,
                                           m.nfac_u, m.nfac_o, m.tol)
    xdata = m.data[:, m.inclcode == 1][i0 - 1:i1]                       # :335-336
    xs, xstd = standardize_data(xdata)                                   # :339
    standardize_constraint(lam_constr, xstd)                             # :340
    m.fes.tss = float(np.nansum(xs ** 2)); m.fes.nobs = int((~np.isnan(xs)).sum())   # :342-343
    xbal, _ = drop_missing_col(xs)                                       # :345
    f = pca_score(xbal, nfac_u) if f_init is None else f_init.copy()     # :348
    m.fes.ssr = 0.0
    lam = np.full((m.fes.ns, m.nfac_t), np.nan)                          # :351 (undef Union -> missing)
    it = 0
    for it in range(1, max_iter + 1):                                    # :352
        ssr_old = m.fes.ssr
        for i in range(m.fes.ns):                                        # :355-362
            keep = ~(np.isnan(xs[:, i]) | np.isnan(f).any(axis=1))
            if keep.sum() >= nt_min:
                lam[i] = ols_skipmissing_balanced(xs[:, i], f)[0]
                impose_constraint(lam[i], i, f, lam_constr, "factor")
        b, ehat, _ = ols_skipmissing_unbalanced(xs.T, lam[:, nfac_o:])   # :364
        f = b.T
        m.fes.ssr = float(np.nansum(ehat ** 2))                          # :366
        if not abs(ssr_old - m.fes.ssr) >= tol * m.fes.T * m.fes.ns:     # :367-368
            break
    m.fes.iters = it
    m.factor[i0 - 1:i1] = f                                              # :371
    m.lambda_est = lam
    m.xs, m.xstd = xs, xstd
    if computeR2:                                                        # :372-380
        for i in range(m.fes.ns):
            tmp, _ = drop_missing_row(np.column_stack([xs[:, i], f]))
            if tmp.shape[0] >= nt_min:
                _, e = ols(tmp[:, 0], tmp[:, 1:])
                m.fes.R2[i] = compute_r2(tmp[:, 0], e)[0]


# ----------------------------------------------------------------- a9: loadings + idiosyncratic AR
def estimate_factor_loading(m, lam_constr=None):
    """estimate_factor_loading!  :391-415.  Series with < nt_min rows get NaN rows
    (the reference would raise UndefVarError / reuse stale values there: SURVEY 'bugs')."""
    i0, i1 = m.initperiod, m.lastperiod
    fac = m.factor[i0 - 1:i1]
    for s in range(m.ns):
        tmp, keep = drop_missing_row(np.column_stack([m.data[i0 - 1:i1, s], fac]))
        arcoef, ser = np.full(m.n_uarlag, np.nan), np.nan
        if keep.sum() >= m.nt_min_factorloading_estimation:
            X = np.column_stack([tmp[:, 1:], np.ones(keep.sum())])
            b, uhat = ols(tmp[:, 0], X)
            if lam_constr is not None and (lam_constr.indices == s).any():   # :401, :1167-1173
                impose_constraint(b, s, X, lam_constr, "loading")
                uhat = tmp[:, 0] - X @ b
            m.lambda_[s] = b[:-1]
            m.r2[s] = compute_r2(tmp[:, 0], uhat)[0]
            if m.r2[s] < 0.9999:
                arcoef, ser = uar(uhat, m.n_uarlag)
            else:
                arcoef, ser = np.zeros(m.n_uarlag), 0.0
        m.uar_coef[s] = arcoef; m.uar_ser[s] = ser


# ----------------------------------------------------------------- a10: factor VAR + companion
def estimate_var(v, compute_matrices=True):
    """estimate_var!  :444-468."""
    i0, i1 = v.initperiod, v.lastperiod
    y = v.y[i0 - 1:i1]
    x = lagmat(y, list(range(1, v.nlag + 1)))
    if v.withconst:
        x = np.column_stack([np.ones(i1 - i0 + 1), x])
    betahat, ehat, keep = ols_skipmissing_balanced(y, x)
    v.betahat[:] = betahat
    ndf = keep.sum() - x.shape[1]
    v.seps[:] = ehat.T @ ehat / ndf
    v.resid[i0 - 1 + np.flatnonzero(keep)] = ehat
    if compute_matrices:
        fill_matrices(v, betahat)


def fill_matrices(v, betahat):
    """fill_matrices!  :477-492.  (as in the reference, assumes withconst=True: drops row 1)."""
    ns, nlag = v.y.shape[1], v.nlag
    b = betahat[1:].T
    v.M[:] = 0; v.M[:ns] = b
    v.M[ns:, :ns * nlag - ns] = np.eye(ns * nlag - ns)
    v.Q[:] = 0; v.Q[:, :ns] = np.eye(ns)
    v.G[:] = 0; v.G[:ns] = np.linalg.cholesky(v.seps)          # cholesky(seps).U' = lower factor


def impulse_response(v, shock_ids, H):
    """:793-816  irf[:, h, j] = Q M^(h-1) G[:, shock_j]."""
    irfs = np.empty((v.Q.shape[0], H, len(shock_ids)))
    for j, sid in enumerate(shock_ids):
        x = v.G[:, sid].copy()
        for h in range(H):
            irfs[:, h, j] = v.Q @ x
            x = v.M @ x
    return irfs


def estimate(m, lam_constr_f=None, lam_constr_fl=None):
    """estimate!(m, ::NonParametric)  :530-543."""
    estimate_factor(m, lam_constr=lam_constr_f)
    estimate_factor_loading(m, lam_constr=lam_constr_fl)
    estimate_var(m.factor_var_model)


# ----------------------------------------------------------------- f1: number-of-factor criteria
def bai_ng_criterion(m):
    """:648-654"""
    fes = m.fes
    nbar = fes.nobs / fes.T
    g = np.log(min(nbar, fes.T)) * (nbar + fes.T) / fes.nobs
    return np.log(fes.ssr / fes.nobs) + m.nfac_t * g


def amengual_watson_test(m, nper=4):
    """:734-768"""
    T, ns, nstat = m.T, m.fes.ns, m.nfac_t
    nlag = m.factor_var_model.nlag
    est = m.data[:, m.inclcode == 1]
    x = np.column_stack([np.ones(T), lagmat(m.factor, list(range(1, nlag + 1)))])
    res = np.full((T, ns), np.nan)
    for s in range(ns):
        tmp, keep = drop_missing_row(np.column_stack([est[:, s], x]))
        if tmp.shape[0] - (tmp.shape[1] - 1) >= m.nt_min_factor_estimation:
            _, e = ols(tmp[:, 0], tmp[:, 1:])
            res[keep, s] = e
    aw = np.empty(nstat); ssr = np.empty(nstat); r2 = np.full((ns, nstat), np.nan)
    for nfac in range(1, nstat + 1):
        d = DFMModel(res, np.ones(ns, int), m.nt_min_factor_estimation, m.nt_min_factorloading_estimation,
                     m.initperiod + 4, m.lastperiod, 0, nfac, m.tol, m.n_uarlag, m.n_factorlag)
        estimate_factor(d)
        aw[nfac - 1] = bai_ng_criterion(d); ssr[nfac - 1] = d.fes.ssr; r2[:, nfac - 1] = d.fes.R2
    return aw, ssr, r2


def estimate_factor_numbers(m, max_nfac):
    """:698-725"""
    bn = np.full(max_nfac, np.nan); ssr_s = np.full(max_nfac, np.nan)
    R2_s = np.full((m.fes.ns, max_nfac), np.nan)
    aw = np.full((max_nfac, max_nfac), np.nan); ssr_d = np.full((max_nfac, max_nfac), np.nan)
    out = {}
    for i, nfac in enumerate(range(1, max_nfac + 1)):
        d = DFMModel(m.data, m.inclcode, m.nt_min_factor_estimation, m.nt_min_factorloading_estimation,
                     m.initperiod, m.lastperiod, m.nfac_o, nfac, m.tol, m.n_uarlag, m.n_factorlag)
        estimate_factor(d)
        bn[i] = bai_ng_criterion(d); ssr_s[i] = d.fes.ssr; R2_s[:, i] = d.fes.R2
        a, s, _ = amengual_watson_test(d, 4)
        aw[:nfac, i] = a; ssr_d[:nfac, i] = s
        out.update(tss=d.fes.tss, nobs=d.fes.nobs, T=d.fes.T)
    out.update(bn_icp=bn, ssr_static=ssr_s, R2_static=R2_s, aw_icp=aw, ssr_dynamic=ssr_d)
    return out


# ----------------------------------------------------------------- f4: instability tests (HAC / Chow / QLR)
def form_kernel(q):
    """form_kernel(q::Integer)  dfm_functions.ipynb (Bartlett weights 1 - i/(q+1), i = 0..q)."""
    return np.array([1.0 - i / (q + 1.0) for i in range(q + 1)])


def form_hscrc(z, X, kernel, q):
    """form_hscrc: HAC sandwich (X'X)^-1 [sum_i k_i (z'z_lag + z_lag'z)] (X'X)^-T."""
    k = X.shape[1]; T = z.shape[0]
    v = np.zeros((k, k))
    for i in range(-q, 1):
        r2 = T + i
        v = v + kernel[-i] * z[0:r2].T @ z[-i:r2 - i]
    for i in range(1, q + 1):
        v = v + kernel[i] * z[i:T].T @ z[0:T - i]
    XX = X.T @ X
    return np.linalg.solve(XX, np.linalg.solve(XX, v.T).T)          # XX \ v / XX'


def hac(u, X, q):
    z = X * u[:, None]
    vbeta = form_hscrc(z, X, form_kernel(q), q)
    return vbeta, np.sqrt(np.diag(vbeta))


def regress_hac(y, X, q):
    betahat, ehat = ols(y, X)
    vbeta, se = hac(ehat, X, q)
    return betahat, vbeta, se


def compute_chow(y, X, q, T_break):
    """compute_chow: Wald statistic of the break-dummy interactions with HAC(q) covariance."""
    k = X.shape[1]; T = len(y)
    D = np.concatenate([np.zeros(T_break), np.ones(T - T_break)])
    betahat, vbeta, _ = regress_hac(y, np.column_stack([X, X * D[:, None]]), q)
    gamma = betahat[k:]
    v1 = vbeta[k:, k:]
    return float(gamma @ np.linalg.solve(v1, gamma))


def compute_qlr(y, X2, ccut, q):
    """compute_qlr(y, nothing, X2, ccut, q): sup of the Chow statistics over the central break dates (q = 0 and HAC(q))."""
    T = len(y)
    n1t = int(np.floor(ccut * T)); n2t = T - n1t
    lr = [compute_chow(y, X2, 0, tb) for tb in range(n1t, n2t + 1)]
    lrr = [compute_chow(y, X2, q, tb) for tb in range(n1t, n2t + 1)]
    return max(lr), max(lrr)


def instability_tests(m, lastpre, q=6, ccut=0.15, min_obs=80):
    """The per-series loop of Stock_Watson.ipynb Table 4(a): Chow (break after `lastpre` rows of the rows that survive
    drop_missing_row -- the notebook's convention) and QLR statistics of the regression of each series on m.factor."""
    X = m.factor
    chow = np.full(m.ns, np.nan); qlr = np.full(m.ns, np.nan)
    for i in range(m.ns):
        y = m.data[:, i]
        if (~np.isnan(y[:lastpre])).sum() >= min_obs and (~np.isnan(y[lastpre:])).sum() >= min_obs:
            yx, _ = drop_missing_row(np.column_stack([y, X]))
            chow[i] = compute_chow(yx[:, 0], yx[:, 1:], q, lastpre)
            Td = yx.shape[0]; n1t = int(np.floor(ccut * Td))            # = compute_qlr(...)[2] (lmr); its q = 0 twin is not needed here
            qlr[i] = max(compute_chow(yx[:, 0], yx[:, 1:], q, tb) for tb in range(n1t, Td - n1t + 1))
    return chow, qlr


def fitted_value_correlations(m, m_alt, lastpre, min_obs=80):
    """Second half of the per-series loop of Table 4(a): correlation between the fitted values of the regression of each
    series on the full-sample factors (m.factor) and on the factors of another sample (m_alt.factor), over the rows where
    both exist (ols_skipmissing(y, X, Balanced()); yhat = X*bhat; drop_missing_row; cor)."""
    X, Xa = m.factor, m_alt.factor
    out = np.full(m.ns, np.nan)
    for i in range(m.ns):
        y = m.data[:, i]
        if (~np.isnan(y[:lastpre])).sum() >= min_obs and (~np.isnan(y[lastpre:])).sum() >= min_obs:
            yh = X @ ols_skipmissing_balanced(y, X)[0]
            ya = Xa @ ols_skipmissing_balanced(y, Xa)[0]
            both, _ = drop_missing_row(np.column_stack([yh, ya]))
            out[i] = np.corrcoef(both[:, 0], both[:, 1])[0, 1]
    return out
