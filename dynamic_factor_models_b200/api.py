"""Host-side mirror of the reference's `dfm_functions` interface (same names, argument meaning and
error behaviour; Julia's mutating `f!(m)` becomes `f(m)` that mutates `m`), every numerical step
delegated to the CUDA library through the C ABI.  Citations: dfm_functions.ipynb raw JSON lines.

Missing values are NaN (Julia `missing`).  Period indices (`initperiod`, `lastperiod`) are 1-based
and inclusive exactly as in the reference, so notebook code ports line by line.
"""
from dataclasses import dataclass

import numpy as np

from ._lib import Library

_default = None


def set_default_library(lib):
    global _default
    _default = lib


def get_library():
    """The process-wide Library (created lazily on cuda:0).  Raises DFMError when the CUDA library
    or device is missing: there is no CPU fallback."""
    global _default
    if _default is None:
        _default = Library()
    return _default


class NonParametric:      # dfm_functions.ipynb:22
    pass


class Parametric:         # dfm_functions.ipynb:23 (empty placeholder in the reference; implemented here)
    def __init__(self, max_iter=50, tol=1e-6, n_factorlag=None):
        self.max_iter, self.tol, self.n_factorlag = max_iter, tol, n_factorlag


@dataclass
class FactorEstimateStats:   # :66-73
    T: int
    ns: int
    nobs: float = np.nan
    tss: float = np.nan
    ssr: float = np.nan
    R2: np.ndarray = None
    iters: int = 0


class VARModel:              # :43-57, constructor :424-435
    def __init__(self, y, nlag=1, withconst=True, initperiod=1, lastperiod=None):
        self.y, self.nlag, self.withconst = y, nlag, withconst
        self.T, self.ns = y.shape
        self.initperiod, self.lastperiod = initperiod, (lastperiod or self.T)
        k = self.ns * nlag
        self.resid = np.full((self.T, self.ns), np.nan)
        self.betahat = np.full((k + int(withconst), self.ns), np.nan)
        self.M = np.full((k, k), np.nan); self.Q = np.full((self.ns, k), np.nan)
        self.G = np.full((k, self.ns), np.nan); self.seps = np.full((self.ns, self.ns), np.nan)


class DFMModel:              # :89-111, constructor :120-146
    def __init__(self, data, inclcode, nt_min_factor_estimation, nt_min_factorloading_estimation,
                 initperiod, lastperiod, nfac_o, nfac_u, tol, n_uarlag, n_factorlag):
        data = np.asarray(data, float); inclcode = np.asarray(inclcode).ravel()
        if data.shape[1] != len(inclcode):
            raise ValueError("length of inclcode must equal to number of data series")       # :124
        if not initperiod < lastperiod:
            raise ValueError("initperiod must be smaller than lastperiod")                   # :125
        if not (n_uarlag > 0 and n_factorlag > 0):
            raise ValueError("n_uarlag and n_factorlag must be positive")                    # :126
        if nfac_o != 0:
            raise ValueError("nfac_o > 0 is not supported (it cannot work in the reference either: :358)")
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
        self.lambda_est = None      # standardized-unit loadings of the ALS loop (:351), kept for the Parametric path
        self.em = None              # results of estimate(m, Parametric())


@dataclass
class LambdaConstraint:      # :1063-1068   (indices 0-based here)
    indices: np.ndarray
    R: np.ndarray
    r: np.ndarray


def construct_constraint(varnames, used_varnames, R, r):
    """:1090-1102"""
    used = list(used_varnames); R = np.asarray(R, float); r = np.asarray(r, float)
    n_R = R.shape[0]
    idx = np.array([used.index(v) for v in varnames for _ in range(n_R)], dtype=np.int32)
    return LambdaConstraint(idx, np.tile(R, (len(varnames), 1)), np.tile(r, len(varnames)))


def _constr(c):
    return None if c is None else (c.indices, c.R, c.r)


# ------------------------------------------------------------------ thin functional wrappers
def standardize_data(data, lib=None):
    """:501-509 -> (standardized, std)"""
    xs, _, sd = (lib or get_library()).standardize(data)
    return xs, sd


def pca_score(X, nfac_u, lib=None):
    """:179-183 (column signs: largest-magnitude entry of each right singular vector positive)."""
    return (lib or get_library()).pca_score(X, nfac_u)


def estimate_factor(m, max_iter=100000000, computeR2=True, lam_constr=None, lib=None, f_init=None):
    """estimate_factor!  :328-382"""
    lib = lib or get_library()
    i0, i1 = m.initperiod, m.lastperiod
    X = m.data[:, m.inclcode == 1][i0 - 1:i1]                               # :335-336
    out = lib.estimate_factor(X, m.nfac_u, nt_min=m.nt_min_factor_estimation, tol=m.tol, max_iter=max_iter,
                              compute_r2=computeR2, constr=_constr(lam_constr), F_init=f_init)
    st = out["stats"]
    if st["status"] in (2, 3):
        raise RuntimeError(f"estimate_factor: device status {st['status']}")
    m.fes.tss, m.fes.nobs, m.fes.ssr, m.fes.iters = st["tss"], st["nobs"], st["ssr"], st["iters"]
    m.factor[i0 - 1:i1] = out["F"]                                          # :371
    if computeR2:
        m.fes.R2[:] = out["R2"]
    m.lambda_est, m.xstd, m.xmean = out["Lam"], out["xstd"], out["xmean"]
    return None


def estimate_factor_loading(m, lam_constr=None, lib=None):
    """estimate_factor_loading!  :391-415"""
    lib = lib or get_library()
    i0, i1 = m.initperiod, m.lastperiod
    out = lib.estimate_loading(m.data[i0 - 1:i1], m.factor[i0 - 1:i1], nt_min=m.nt_min_factorloading_estimation,
                               n_uarlag=m.n_uarlag, constr=_constr(lam_constr))
    m.lambda_[:] = out["lam"]; m.r2[:] = out["r2"]; m.uar_coef[:] = out["uar_coef"]; m.uar_ser[:] = out["uar_ser"]
    return None


def estimate_var(varm, compute_matrices=True, lib=None):
    """estimate_var!  :444-468 (+ fill_matrices! :477-492)"""
    lib = lib or get_library()
    i0, i1 = varm.initperiod, varm.lastperiod
    out = lib.estimate_var(varm.y[i0 - 1:i1], varm.nlag, varm.withconst)
    varm.betahat[:] = out["betahat"]; varm.seps[:] = out["seps"]
    varm.resid[i0 - 1:i1] = out["resid"]
    if compute_matrices:
        varm.M[:] = out["M"]; varm.Q[:] = out["Q"]; varm.G[:] = out["G"]
    return None


def impulse_response(varm, shock_ids, T, lib=None):
    """:793-825.  shock_ids: iterable of 1-based ids as in the reference, or 'all'."""
    lib = lib or get_library()
    ids = list(range(1, varm.G.shape[1] + 1)) if isinstance(shock_ids, str) and shock_ids == "all" else list(shock_ids)
    return lib.irf(varm.M, varm.Q, varm.G, T, [i - 1 for i in ids])


def estimate(m, method=None, lam_constr_f=None, lam_constr_fl=None, lib=None):
    """estimate!(m, ::NonParametric) :530-543;  estimate!(m, ::Parametric) = the slot of :23."""
    method = method or NonParametric()
    estimate_factor(m, lam_constr=lam_constr_f, lib=lib)
    estimate_factor_loading(m, lam_constr=lam_constr_fl, lib=lib)
    estimate_var(m.factor_var_model, lib=lib)
    if isinstance(method, Parametric):
        _estimate_parametric(m, method, lib or get_library())
    return None


def _estimate_parametric(m, method, lib):
    """State-space EM initialised by the non-parametric estimates (SURVEY.md section 8 row a')."""
    i0, i1 = m.initperiod, m.lastperiod
    p = method.n_factorlag or m.n_factorlag
    X = m.data[:, m.inclcode == 1][i0 - 1:i1]
    Xs, _, _ = lib.standardize(X)
    Xs = np.where(np.isnan(m.lambda_est[:, :1].T), np.nan, Xs)      # series dropped by nt_min stay out of the model
    F0 = m.factor[i0 - 1:i1]
    Lam, R, A, Q = lib.em_init_from_factors(Xs, F0, p)
    m.em = lib.em_kalman(Xs, Lam, R, A, Q, p=p, max_iter=method.max_iter, tol=method.tol)
    m.factor[i0 - 1:i1] = m.em["F"]
    return None


def kalman_smooth(X, Lam, R, A, Q, p=1, P0=None, H=0, lib=None, **kw):
    """Smoothed factors, H-period forecasts and imputed values of a standardized panel at given state-space parameters
    (dfm_kalman_smooth).  See Library.kalman_smooth."""
    return (lib or get_library()).kalman_smooth(X, Lam, R, A, Q, p=p, P0=P0, H=H, **kw)


def forecast(m, H, lib=None):
    """Nowcasts, forecasts and imputed values from a model estimated with `estimate(m, Parametric())`.

    Runs the Kalman filter and smoother once at the EM estimates `m.em` over the estimation block (rows
    initperiod..lastperiod, series with inclcode == 1, standardized as `estimate` standardizes them) and H periods after it.
    Returns a dict, rows = periods initperiod .. lastperiod + H (1-based, in `periods`), columns = the estimation series
    (indices into m.data's columns in `series`):
      factor (T+H, r), factor_var (T+H, r, r)   E[f_t | data] and its covariance (standardized units, as m.factor);
      xhat (T+H, ns)   E[x_it | data] in data units: the data where observed, the nowcast / forecast / imputed value otherwise;
      xvar (T+H, ns)   Var[x_it | data] in data units: 0 where observed;
      common (T+H, ns) the common component lambda_i' E[f_t | data] in data units (xmean + xstd * common, as compute_series);
      loglik           log-likelihood of the observed cells at m.em's parameters.
    Series left out of the model (too few observations for the ALS step) have NaN columns."""
    b = _state_space_block(m, H, lib, "forecast")
    lib, e = b["lib"], b["em"]
    o = lib.kalman_smooth(b["Xs"], b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=H)
    if o["status"] != 0:
        raise RuntimeError(f"forecast: device status {o['status']}")
    xmean, xstd = b["xmean"], b["xstd"]
    return dict(periods=b["periods"], series=b["series"], factor=o["F"], factor_var=o["PF"],
                xhat=xmean + xstd * o["xhat"], xvar=xstd ** 2 * o["xvar"], common=xmean + xstd * o["common"],
                loglik=o["loglik"])


def _state_space_block(m, H, lib, what):
    """The estimation block of a model estimated with Parametric(), standardized as `estimate` standardizes it, with the
    series left out of the model (NaN ALS loadings) set to NaN, and the EM estimates with those series' loadings NaN."""
    if m.em is None:
        raise ValueError(f"{what} needs a model estimated with Parametric()")
    if H < 0:
        raise ValueError("H must be >= 0")
    lib = lib or get_library()
    i0, i1 = m.initperiod, m.lastperiod
    incl = np.flatnonzero(m.inclcode == 1)
    X = m.data[:, incl][i0 - 1:i1]
    Xs, xmean, xstd = lib.standardize(X)                               # the standardisation of _estimate_parametric
    out_model = np.isnan(m.lambda_est[:, 0])
    Xs = np.where(out_model[None, :], np.nan, Xs)
    e = m.em
    r = e["Lam"].shape[1]
    return dict(lib=lib, periods=np.arange(i0, i1 + H + 1), series=incl, Xs=Xs, xmean=xmean, xstd=xstd, em=e, p=e["A"].shape[1] // r,
                Lam=np.where(out_model[:, None], np.nan, e["Lam"]))


def posterior_draws(m, H, n_draw, seed, draw0=0, lib=None):
    """Draws from the JOINT posterior of the factor path and the missing / forecast values of a model estimated with
    `estimate(m, Parametric())`, at its EM estimates (simulation smoother, dfm_simulation_smoother).

    Same block as `forecast(m, H)` (rows `periods`, columns `series`).  Returns a dict with
      factor (n_draw, T+H, r)  draws of f_t (standardized units, as m.factor);
      x (n_draw, T+H, ns)      draws of the panel in data units: the data where observed, a draw where missing or forecast;
    draw j is draw id draw0 + j of stream `seed` (any split of a draw range gives the same draws).  Functions of a path --
    growth rates, averages, threshold probabilities -- take their posterior distribution from these draws; forecast's
    xhat / xvar are their means / variances cell by cell.  Series left out of the model have NaN columns."""
    b = _state_space_block(m, H, lib, "posterior_draws")
    lib, e = b["lib"], b["em"]
    o = lib.simulation_smoother(b["Xs"], b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=H, n_draw=n_draw, seed=seed,
                                draw0=draw0)
    if o["status"] != 0:
        raise RuntimeError(f"posterior_draws: device status {o['status']}")
    return dict(periods=b["periods"], series=b["series"], factor=o["F"], x=b["xmean"] + b["xstd"] * o["X"])


def news(m, data_new, targets, H=0, lib=None):
    """Why the nowcast moved: the news decomposition (Banbura & Modugno 2014) of the revision of each target between the
    data of a model estimated with `estimate(m, Parametric())` and a new vintage `data_new` (the shape of m.data), at the
    EM estimates m.em (dfm_news).

    targets: (column of m.data, 1-based period) pairs, period in initperiod .. lastperiod + H.  Both vintages are
    standardized with the mean and std of the estimation block of m.data, as `forecast` standardizes it.  The release window
    starts at the first row that holds a new cell.  Cells observed in both vintages with different values (data revisions)
    are handled first: `revision_effect` is the change of the estimate when the old cells take their new values, and the
    decomposition runs from that revised vintage.  A cell that disappears from the new vintage raises ValueError.
    Returns a dict, in data units:
      old, new (n_target)                E[y | old data], E[y | new data];
      revision_effect (n_target)         the part of new - old due to revised cells;
      news (news_rows, ns)               x_j - E[x_j | old] at the released cells, NaN elsewhere;
      weights, contributions (n_target, news_rows, ns)   w_qj (scaled by xstd_target / xstd_j) and w_qj news_j;
      by_series (n_target, ns)           contributions summed over the window rows:  by_series.sum(1) + revision_effect
                                         = new - old;
    and periods (the window rows, 1-based), series (columns of m.data), targets."""
    b = _state_space_block(m, H, lib, "news")
    lib, e = b["lib"], b["em"]
    i0, i1 = m.initperiod, m.lastperiod
    incl, xmean, xstd, Xs = b["series"], b["xmean"], b["xstd"], b["Xs"]
    data_new = np.asarray(data_new, float)
    if data_new.shape != m.data.shape:
        raise ValueError(f"news: data_new has shape {data_new.shape}, m.data {m.data.shape}")
    T, ns = Xs.shape
    col = {int(c): j for j, c in enumerate(incl)}
    tg = []
    for c, t in targets:
        if int(c) not in col:
            raise ValueError(f"news: target column {c} is not an estimation series")
        if not i0 <= t <= i1 + H:
            raise ValueError(f"news: target period {t} outside {i0} .. {i1 + H}")
        tg.append((col[int(c)], int(t) - i0))
    Xold = m.data[:, incl][i0 - 1:i1]
    Xnew = data_new[:, incl][i0 - 1:i1]
    inm = ~np.isnan(Xs)                                                 # old cells in the model
    if (inm & np.isnan(Xnew)).any():
        raise ValueError("news: a cell observed in m.data is missing in data_new")
    revised = inm & (Xnew != Xold)
    Xn_std = (Xnew - xmean) / xstd
    Xrev = np.where(revised, Xn_std, Xs)                                # the old cells at their new values
    out_model = np.isnan(b["Lam"][:, 0])
    Xn = np.where(inm, Xrev, np.where(out_model[None, :], np.nan, Xn_std))
    added = np.isnan(Xrev) & ~np.isnan(Xn)
    rows = np.flatnonzero(added.any(1))
    nr = T - int(rows[0]) if len(rows) else 1
    o = lib.news(Xrev, Xn, b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=H, targets=tg, news_rows=nr)
    if o["status"] != 0:
        raise RuntimeError(f"news: device status {o['status']}")
    ti = np.array([j for j, _ in tg], int)
    sd_t, mu_t = xstd[ti], xmean[ti]
    base = o["old_est"]
    if revised.any():
        ks = lib.kalman_smooth(Xs, b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=H, outputs=("xhat",))
        if ks["status"] != 0:
            raise RuntimeError(f"news: device status {ks['status']}")
        base = ks["xhat"][[t for _, t in tg], ti]
    w = np.transpose(o["weight"], (2, 0, 1)) * sd_t[:, None, None] / xstd[None, None, :]
    c = np.transpose(o["contrib"], (2, 0, 1)) * sd_t[:, None, None]
    return dict(old=mu_t + sd_t * base, new=mu_t + sd_t * o["new_est"], revision_effect=sd_t * (o["old_est"] - base),
                news=xstd[None, :] * o["news"], weights=w, contributions=c, by_series=c.sum(1),
                periods=np.arange(i0 + T - nr, i1 + 1), series=incl, targets=list(targets))


def forecast_bands(m, H, q, n_draw, seed, lib=None):
    """Percentile bands (numpy.percentile's linear interpolation, on the device through dfm_percentiles) of the panel draws
    of `posterior_draws(m, H, n_draw, seed)`, cell by cell.  Returns a dict with bands (len(q), T+H, ns) in data units, rows
    `periods`, columns `series` as forecast(m, H), and q.  n_draw <= 16384."""
    if not 1 <= n_draw <= 16384:
        raise ValueError("forecast_bands: n_draw must be in [1, 16384]")
    lib = lib or get_library()
    d = posterior_draws(m, H, n_draw, seed, lib=lib)
    x = d["x"]
    bands = lib.percentiles(x.reshape(n_draw, -1), q)
    return dict(periods=d["periods"], series=d["series"], q=np.asarray(q, float), bands=bands.reshape((len(q),) + x.shape[1:]))


def em_init_from_factors(Xs, F, p=1, lib=None):
    return (lib or get_library()).em_init_from_factors(Xs, F, p)


def em_kalman(X, Lam, R, A, Q, p=1, P0=None, max_iter=50, tol=0.0, lib=None, **kw):
    return (lib or get_library()).em_kalman(X, Lam, R, A, Q, p=p, P0=P0, max_iter=max_iter, tol=tol, **kw)


# ------------------------------------------------------------------ (f1) number-of-factor criteria
def bai_ng_criterion(m):
    """:648-654 (pure scalar arithmetic on the stats the device returned)."""
    fes = m.fes
    nbar = fes.nobs / fes.T
    g = np.log(min(nbar, fes.T)) * (nbar + fes.T) / fes.nobs
    return np.log(fes.ssr / fes.nobs) + m.nfac_t * g


def _lagmat(X, lags):
    X = X.reshape(len(X), -1); nc = X.shape[1]
    out = np.full((X.shape[0], nc * len(lags)), np.nan)
    for i, lag in enumerate(lags):
        out[lag:, nc * i:nc * (i + 1)] = X[:-lag]
    return out


def amengual_watson_test(m, nper=4, lib=None):
    """:734-768.  The residualisation on factor lags is one batched-over-series regression on the
    device (dfm_estimate_loading with the lagged factors as regressors); the nfac ALS solves are
    one batched dfm_estimate_factor call per nfac."""
    lib = lib or get_library()
    T, ns, nstat = m.T, m.fes.ns, m.nfac_t
    nlag = m.factor_var_model.nlag
    est = m.data[:, m.inclcode == 1]
    xl = _lagmat(m.factor, list(range(1, nlag + 1)))                     # [1, lags] regressors (:741)
    rows = ~np.isnan(xl).any(axis=1)
    res = np.full((T, ns), np.nan)
    # per-series OLS of est[:, s] on [lags, 1] over available rows (:743-752); constant last == first up to order
    yy = est[rows]; zz = xl[rows]
    K = zz.shape[1] + 1
    out = lib.estimate_loading(yy, zz, nt_min=m.nt_min_factor_estimation + K, n_uarlag=1)
    res[rows] = out["resid"]                       # device residuals e = y - [z 1] b, NaN where missing / not fitted
    aw = np.empty(nstat); ssr = np.empty(nstat); r2 = np.full((ns, nstat), np.nan)
    for nfac in range(1, nstat + 1):
        d = DFMModel(res, np.ones(ns, int), m.nt_min_factor_estimation, m.nt_min_factorloading_estimation,
                     m.initperiod + 4, m.lastperiod, 0, nfac, m.tol, m.n_uarlag, m.n_factorlag)
        estimate_factor(d, lib=lib)
        aw[nfac - 1] = bai_ng_criterion(d); ssr[nfac - 1] = d.fes.ssr; r2[:, nfac - 1] = d.fes.R2
    return aw, ssr, r2


def estimate_factor_numbers(m, max_nfac, lib=None):
    """:698-725"""
    lib = lib or get_library()
    bn = np.full(max_nfac, np.nan); ssr_s = np.full(max_nfac, np.nan)
    R2_s = np.full((m.fes.ns, max_nfac), np.nan)
    aw = np.full((max_nfac, max_nfac), np.nan); ssr_d = np.full((max_nfac, max_nfac), np.nan)
    out = {}
    for i, nfac in enumerate(range(1, max_nfac + 1)):
        d = DFMModel(m.data, m.inclcode, m.nt_min_factor_estimation, m.nt_min_factorloading_estimation,
                     m.initperiod, m.lastperiod, m.nfac_o, nfac, m.tol, m.n_uarlag, m.n_factorlag)
        estimate_factor(d, lib=lib)
        bn[i] = bai_ng_criterion(d); ssr_s[i] = d.fes.ssr; R2_s[:, i] = d.fes.R2
        a, s, _ = amengual_watson_test(d, 4, lib=lib)
        aw[:nfac, i] = a; ssr_d[:nfac, i] = s
        out.update(tss=d.fes.tss, nobs=d.fes.nobs, T=d.fes.T)
    out.update(bn_icp=bn, ssr_static=ssr_s, R2_static=R2_s, aw_icp=aw, ssr_dynamic=ssr_d)
    return out


# ---------------------------------------------------------------------------------------------- f4: instability tests
def instability_tests(m, lastpre, q=6, ccut=0.15, min_obs=80, lib=None, want_q0=False):
    """Chow and QLR statistics of every series of `m.data` regressed on `m.factor` (compute_chow / compute_qlr with
    regress_hac / hac / form_hscrc, dfm_functions.ipynb; the per-series loop of Stock_Watson.ipynb Table 4(a)): break after
    the first `lastpre` rows that survive drop_missing_row, Bartlett HAC with q lags, QLR over the central 1 - 2 ccut of
    the sample.  Series with fewer than min_obs observations on either side of row `lastpre` are NaN.  Returns (chow, qlr)
    or (chow, qlr, qlr0)."""
    lib = lib or get_library()
    out = lib.instability(m.data, m.factor, lastpre, q=q, ccut=ccut, min_obs=min_obs, want_q0=want_q0)
    return (out["chow"], out["qlr"], out["qlr0"]) if want_q0 else (out["chow"], out["qlr"])


def fitted_value_correlations(m, m_alt, lastpre, min_obs=80, lib=None):
    """cor(yhat, yhat_alt) per series: fitted values of `m.data` on `m.factor` and on `m_alt.factor` (Table 4(a), lower half)."""
    lib = lib or get_library()
    return lib.fit_correlation(m.data, m.factor, m_alt.factor, lastpre, min_obs=min_obs)
