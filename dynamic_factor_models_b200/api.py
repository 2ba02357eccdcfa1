"""Host-side mirror of the reference's `dfm_functions` interface (same names, argument meaning and
error behaviour; Julia's mutating `f!(m)` becomes `f(m)` that mutates `m`), every numerical step
delegated to the CUDA library through the C ABI.  Citations: dfm_functions.ipynb raw JSON lines.

Missing values are NaN (Julia `missing`).  Period indices (`initperiod`, `lastperiod`) are 1-based
and inclusive exactly as in the reference, so notebook code ports line by line.
"""
from dataclasses import dataclass

import numpy as np

from ._lib import Library, gibbs_default_prior as _gibbs_default_prior

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


def estimate(m, method=None, lam_constr_f=None, lam_constr_fl=None, lam_constr_em=None, lib=None):
    """estimate!(m, ::NonParametric) :530-543;  estimate!(m, ::Parametric) = the slot of :23.

    lam_constr_em (Parametric only): a LambdaConstraint on the estimation series (indices as lam_constr_f's, r in data units)
    under which the state-space EM runs, e.g. the named-factor normalisation of Figure 7.  Its r is divided by the estimation
    block's xstd (standardize_constraint!); the standardized restriction is kept in m.em["lam_constr"]."""
    method = method or NonParametric()
    estimate_factor(m, lam_constr=lam_constr_f, lib=lib)
    estimate_factor_loading(m, lam_constr=lam_constr_fl, lib=lib)
    estimate_var(m.factor_var_model, lib=lib)
    if isinstance(method, Parametric):
        _estimate_parametric(m, method, lib or get_library(), lam_constr_em)
    return None


def _estimate_parametric(m, method, lib, lam_constr_em=None):
    """State-space EM initialised by the non-parametric estimates (SURVEY.md section 8 row a'), restricted by lam_constr_em."""
    i0, i1 = m.initperiod, m.lastperiod
    p = method.n_factorlag or m.n_factorlag
    X = m.data[:, m.inclcode == 1][i0 - 1:i1]
    Xs, _, xstd = lib.standardize(X)
    Xs = np.where(np.isnan(m.lambda_est[:, :1].T), np.nan, Xs)      # series dropped by nt_min stay out of the model
    F0 = m.factor[i0 - 1:i1]
    Lam, R, A, Q = lib.em_init_from_factors(Xs, F0, p)
    constr = None
    if lam_constr_em is not None:
        idx = np.asarray(lam_constr_em.indices, dtype=np.int32)
        constr = (idx, np.asarray(lam_constr_em.R, float).reshape(len(idx), -1), np.asarray(lam_constr_em.r, float) / xstd[idx])
    m.em = lib.em_kalman(Xs, Lam, R, A, Q, p=p, max_iter=method.max_iter, tol=method.tol, constr=constr)
    if constr is not None:
        m.em["lam_constr"] = constr
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


def parametric_irf(m, H, lib=None):
    """Impulse responses of a model estimated with `estimate(m, Parametric())` at its EM estimates m.em, through dfm_irf:
    irf[:, h, j] = E M^h G e_j with M the companion matrix of m.em["A"] and G = [chol(Q); 0] (orthogonalized shocks).
    Returns (r, H, r) [variable, horizon, shock] in standardized factor units, as impulse_response.  The centre of the bands of
    parametric_bootstrap."""
    if m.em is None:
        raise ValueError("parametric_irf needs a model estimated with Parametric()")
    if H <= 0:
        raise ValueError("H must be > 0")
    lib = lib or get_library()
    A, Q = m.em["A"], m.em["Q"]
    r = Q.shape[0]; k = A.shape[1]
    M = np.zeros((k, k)); M[:r] = A; M[r:, :k - r] = np.eye(k - r)
    Qs = np.zeros((r, k)); Qs[:, :r] = np.eye(r)
    G = np.zeros((k, r)); G[:r] = np.linalg.cholesky(Q)
    return lib.irf(M, Qs, G, H, list(range(r)))


def series_irf(m, H, lib=None):
    """Responses of the estimation series to the orthogonalised factor shocks of `parametric_irf(m, H)`, in data units:
    (ns, H, r) [series, horizon, shock], out[i, h, j] = xstd_i lam_i' irf[:, h, j] with lam_i = m.em["Lam"][i] (series in the
    order of forecast's `series`; NaN for series out of the model).

    Identification: the factors of a state-space DFM are identified only up to f -> K f (Lam -> Lam K^-1, A_l -> K A_l K^-1,
    Q -> K Q K').  Under a named-factor restriction (lam_constr_em pinning some series' loadings to e_1', as Figure 7's oil
    series) the rotations left free have K's first row e_1'.  Then (K Q K')_11 = Q_11 and (K Q K') e_1 = K Q e_1, so the first
    column of chol(K Q K') is K times that of chol(Q): the factor responses to shock 1 become K times the old ones and the series
    responses lam_i' K^-1 K irf do not change.  The column of shock 1 is identified even though factors 2..r are not; the other
    shocks' columns depend on the rotation."""
    irf = parametric_irf(m, H, lib=lib)
    b = _state_space_block(m, 0, lib, "series_irf")
    return b["xstd"][:, None, None] * np.einsum("ia,ahj->ihj", b["Lam"], irf)


def variance_decomposition(m, H, lib=None):
    """Series responses and forecast-error variance decompositions of a model estimated with `estimate(m, Parametric())` at its
    EM estimates m.em (dfm_series_responses).  With L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L and c_{i,h} = lam_i' Psi_h:
      resp (ns, H, r)   xstd_i c_{i,h,j}: the response of series i in data units to the orthogonalised shock j (= series_irf);
      fevd (ns, H, r)   sum_{l<=h} c_{i,l,j}^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i): the share of the (h+1)-step forecast-error
                        variance of series i due to shock j; 1 - fevd.sum(-1) is the idiosyncratic share;
    and series (the order of forecast's `series`; NaN rows for series out of the model).

    Identification: as series_irf.  The factors are identified only up to f -> K f; under a named-factor restriction
    (lam_constr_em pinning some series' loadings to e_1') the columns of shock 1 of resp and fevd do not depend on the rotation
    left free, the other shocks' columns do (their sum, and so the idiosyncratic share, does not)."""
    if H <= 0:
        raise ValueError("H must be > 0")
    b = _state_space_block(m, 0, lib, "variance_decomposition")
    lib, e = b["lib"], b["em"]
    o = lib.series_responses(b["Lam"], e["R"], e["A"], e["Q"], H, scale=b["xstd"])
    if o["status"] != 0:
        raise RuntimeError(f"variance_decomposition: device status {o['status']}")
    return dict(resp=o["resp"], fevd=o["fevd"], series=b["series"])


def _named_factors(m):
    """The factors j (0-based) that m.em["lam_constr"] names: some series in the model has full-rank rows whose solution is
    c e_j, c != 0."""
    c = m.em.get("lam_constr") if m.em is not None else None
    if c is None:
        return set()
    idx, Hm, hv = c
    Lam = m.em["Lam"]
    r = Lam.shape[1]
    named = set()
    for i in set(int(v) for v in idx):
        if np.isnan(Lam[i]).any() or np.isnan(m.em["R"][i]) or np.isnan(m.lambda_est[i, 0]):
            continue
        sel = np.flatnonzero(np.asarray(idx) == i)
        Hi, hi = np.asarray(Hm, float)[sel], np.asarray(hv, float)[sel]
        if len(sel) < r or np.linalg.matrix_rank(Hi) < r:
            continue
        lam = np.linalg.lstsq(Hi, hi, rcond=None)[0]
        nz = np.flatnonzero(np.abs(lam) > 1e-12 * np.abs(lam).max()) if np.abs(lam).max() > 0 else []
        if len(nz) == 1:
            named.add(int(nz[0]))
    return named


def identified_responses(m, H, shocks=1, n_chain=4, n_burn=500, n_keep=1000, thin=1, prior=None, seed=20260922,
                         q=(5, 16, 50, 84, 95), chain0=0, sweep0=0, lib=None):
    """Posterior bands of the series responses and variance decompositions of the named shocks 1..`shocks` of a model estimated
    with `estimate(m, Parametric(), lam_constr_em=...)`, whose restriction names factors 1..shocks (factor j is named when some
    series in the model has r independent rows whose solution is c e_j, c != 0, as Figure 7's oil series).  Those columns are
    the ones the rotation left free by the restriction does not change (series_irf, variance_decomposition).

    Gibbs chains under the restriction (dfm_gibbs_constrained: the prior of gibbs with each restricted series' loadings
    conditioned on its rows) start at m.em; every kept draw's responses and decompositions come from dfm_series_responses.
    Returns a dict:
      resp, fevd (ns, H, shocks)                            at m.em (variance_decomposition's first `shocks` columns);
      resp_draws, fevd_draws (n_chain, n_keep, ns, H, shocks)  of every kept draw (NaN for a failed chain);
      resp_bands, fevd_bands (len(q), ns, H, shocks)        percentiles over the draws (dfm_percentiles; failed chains ignored);
      Lam, R, A, Q (n_chain, n_keep, ...)                   raw parameter draws (standardized units);
      loglik (n_chain, n_burn + n_keep thin), status (n_chain);
      rhat dict(loglik, resp (ns, H, shocks))               split-R^ over the kept draws;
    and prior, series, shocks, q.  n_chain n_keep <= 16384."""
    if m.em is None or m.em.get("lam_constr") is None:
        raise ValueError("identified_responses needs a model estimated with Parametric() under lam_constr_em")
    r = m.em["Q"].shape[0]
    if not 1 <= shocks <= r:
        raise ValueError(f"identified_responses: shocks must be in [1, {r}]")
    named = _named_factors(m)
    missing = [j + 1 for j in range(shocks) if j not in named]
    if missing:
        raise ValueError(f"identified_responses: the restriction of m does not name factor(s) {missing} (no series in the model "
                         "has r independent rows whose solution is a multiple of e_j), so their shocks are not identified")
    if H <= 0:
        raise ValueError("H must be > 0")
    if not 1 <= n_chain * n_keep <= 16384:
        raise ValueError("identified_responses: n_chain * n_keep must be in [1, 16384]")
    b = _state_space_block(m, 0, lib, "identified_responses")
    lib, e = b["lib"], b["em"]
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, prior=pr, outputs=("Lam", "R", "A", "Q"), constr=e["lam_constr"])
    n = n_chain * n_keep
    ns = b["Xs"].shape[1]
    sh = lambda a_: a_.reshape((n,) + a_.shape[2:])
    d = lib.series_responses(sh(o["Lam"]), sh(o["R"]), sh(o["A"]), sh(o["Q"]), H, n_shock=shocks, scale=b["xstd"])
    pt = lib.series_responses(b["Lam"], e["R"], e["A"], e["Q"], H, n_shock=shocks, scale=b["xstd"])
    if pt["status"] != 0:
        raise RuntimeError(f"identified_responses: device status {pt['status']}")
    qq = np.asarray(q, float)
    out = dict(resp=pt["resp"], fevd=pt["fevd"], Lam=o["Lam"], R=o["R"], A=o["A"], Q=o["Q"], loglik=o["loglik"], status=o["status"],
               prior=pr, series=b["series"], shocks=shocks, q=qq)
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    for nm in ("resp", "fevd"):
        dr = d[nm].reshape((n_chain, n_keep, ns, H, shocks))
        out[nm + "_draws"] = dr
        out[nm + "_bands"] = lib.percentiles(d[nm].reshape(n, -1), qq).reshape((len(qq), ns, H, shocks))
    out["rhat"] = dict(loglik=float(split_rhat(o["loglik"][:, kept])), resp=split_rhat(out["resp_draws"]))
    return out


def _history_rows(m, b, t0, what):
    """(t0 as a 1-based period, its row in the estimation block, the smoothed path F (T, r) at m.em)."""
    lo = m.initperiod + b["p"] - 1
    t0 = lo if t0 is None else int(t0)
    if not lo <= t0 <= m.lastperiod:
        raise ValueError(f"{what}: t0 must be a period in {lo} .. {m.lastperiod} (initperiod + p - 1 .. lastperiod)")
    e = b["em"]
    o = b["lib"].kalman_smooth(b["Xs"], b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=0, outputs=("F",))
    if o["status"] != 0:
        raise RuntimeError(f"{what}: device status {o['status']}")
    return t0, t0 - m.initperiod, o["F"]


def historical_decomposition(m, t0=None, lib=None):
    """Historical decomposition of a model estimated with `estimate(m, Parametric())` at its EM estimates m.em
    (dfm_historical_decomposition): each series' common component split, period by period, into the contributions of the r
    orthogonalised factor shocks since the base period t0 and the part carried over from the factors at t0.

    The path is the smoothed factor path E[f_t | data] at m.em (kalman_smooth over the estimation block, as forecast(m, 0)); all
    the pieces are linear in the path, so they are their own expectations given the data at m.em.  With L = chol(Q),
    Psi_h = [M^h]_{1:r,1:r} L (series_irf's responses) and the structural shocks eps_t = L^-1 (f_t - sum_l A_l f_{t-l}):
      contrib (ns, T, r)  xstd_i lam_i' sum_{s=t0+1..t} Psi_{t-s} e_j eps_{j,s}: the part of series i at period t due to shock
                          j since t0 (0 up to t0);
      base (ns, T)        xstd_i lam_i' [M^{t-t0} z_t0]_{1:r}: the path the factors at t0 and before would have taken without
                          shocks (the common component itself up to t0);
      resid (ns, T)       data - xmean - xstd_i lam_i' f_t (NaN where the data is missing);
      shocks (T, r)       eps_t (standardized; NaN for the first p periods, which have no lags in the sample);
    so xmean + base + contrib.sum(-1) + resid is the data at every observed cell.  Rows are the periods initperiod ..
    lastperiod (1-based, `periods`), columns the estimation series (`series`); series out of the model have NaN columns.
    t0: a 1-based period in initperiod + p - 1 .. lastperiod (default initperiod + p - 1, the first period whose p lags lie in
    the sample; returned as `t0`).

    Identification: as series_irf.  Under a named-factor restriction (lam_constr_em pinning some series' loadings to e_1') the
    rotations f -> K f left free have K's first row e_1'; then eps_1 and the column of shock 1 of contrib do not change, and
    neither do base and the sum of the other columns; the other shocks' individual columns do."""
    b = _state_space_block(m, 0, lib, "historical_decomposition")
    lib, e = b["lib"], b["em"]
    r = e["Q"].shape[0]
    t0, row, F = _history_rows(m, b, t0, "historical_decomposition")
    o = lib.historical_decomposition(b["Lam"], e["R"], e["A"], e["Q"], F, row, n_shock=r, scale=b["xstd"],
                                     outputs=("shocks", "contrib", "base"))
    if o["status"] != 0:
        raise RuntimeError(f"historical_decomposition: device status {o['status']}")
    X = m.data[:, b["series"]][m.initperiod - 1:m.lastperiod]
    resid = (X - b["xmean"] - b["xstd"] * (F @ b["Lam"].T)).T
    return dict(contrib=np.ascontiguousarray(o["contrib"]), base=np.ascontiguousarray(o["base"]), resid=np.ascontiguousarray(resid),
                shocks=np.ascontiguousarray(o["shocks"]), periods=b["periods"], series=b["series"], t0=t0)


def identified_history(m, shocks=1, t0=None, n_chain=4, n_burn=500, n_keep=1000, thin=1, prior=None, seed=20260922,
                       q=(5, 16, 50, 84, 95), chain0=0, sweep0=0, return_draws=False, lib=None):
    """Posterior bands of the historical decomposition by the named shocks 1..`shocks` of a model estimated with
    `estimate(m, Parametric(), lam_constr_em=...)`, whose restriction names factors 1..shocks (as identified_responses, whose
    preconditions and errors apply).  Those are the columns that the rotation left free by the restriction does not change
    (historical_decomposition).

    Gibbs chains under the restriction (dfm_gibbs_constrained, as identified_responses) start at m.em.  Kept draw j records the
    factor path drawn in its sweep at the parameters entering that sweep and the parameters drawn given that path: a joint
    posterior draw, decomposed as recorded (one dfm_historical_decomposition over all kept draws, n_shock = shocks).  Returns a
    dict, in data units, rows `periods`, columns `series`, t0 as historical_decomposition:
      contrib (ns, T, shocks), rest (ns, T), base (ns, T), shocks (T, shocks)   at m.em along the smoothed path
                          (historical_decomposition's; rest = the other shocks' columns summed);
      contrib_bands, rest_bands, base_bands, shocks_bands (len(q), ...)         percentiles over the kept draws
                          (dfm_percentiles; failed chains, whose draws are NaN, are ignored);
      contrib_draws, rest_draws, base_draws, shocks_draws (n_chain, n_keep, ...) only with return_draws=True: at the defaults
                          each is about 0.5 GB for Stock & Watson's Figure 7 block (139 series, 120 periods);
      rhat dict(loglik, contrib (ns, T, shocks))   split-R^ over the kept draws (NaN up to t0, where contrib is 0 in every draw);
      status (n_chain), loglik (n_chain, n_burn + n_keep thin);
    and prior, q, periods, series, t0.  n_chain n_keep <= 16384."""
    if m.em is None or m.em.get("lam_constr") is None:
        raise ValueError("identified_history needs a model estimated with Parametric() under lam_constr_em")
    r = m.em["Q"].shape[0]
    if not 1 <= shocks <= r:
        raise ValueError(f"identified_history: shocks must be in [1, {r}]")
    named = _named_factors(m)
    missing = [j + 1 for j in range(shocks) if j not in named]
    if missing:
        raise ValueError(f"identified_history: the restriction of m does not name factor(s) {missing} (no series in the model "
                         "has r independent rows whose solution is a multiple of e_j), so their shocks are not identified")
    if not 1 <= n_chain * n_keep <= 16384:
        raise ValueError("identified_history: n_chain * n_keep must be in [1, 16384]")
    b = _state_space_block(m, 0, lib, "identified_history")
    lib, e = b["lib"], b["em"]
    t0, row, F = _history_rows(m, b, t0, "identified_history")
    pt = lib.historical_decomposition(b["Lam"], e["R"], e["A"], e["Q"], F, row, n_shock=shocks, scale=b["xstd"])
    if pt["status"] != 0:
        raise RuntimeError(f"identified_history: device status {pt['status']}")
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, prior=pr, outputs=("Lam", "R", "A", "Q", "F"), constr=e["lam_constr"])
    n = n_chain * n_keep
    sh = lambda a_: a_.reshape((n,) + a_.shape[2:])
    d = lib.historical_decomposition(sh(o["Lam"]), sh(o["R"]), sh(o["A"]), sh(o["Q"]), sh(o["F"]), row, n_shock=shocks,
                                     scale=b["xstd"])
    qq = np.asarray(q, float)
    out = dict(contrib=np.ascontiguousarray(pt["contrib"]), rest=np.ascontiguousarray(pt["rest"]),
               base=np.ascontiguousarray(pt["base"]), shocks=np.ascontiguousarray(pt["shocks"][:, :shocks]), status=o["status"],
               loglik=o["loglik"], prior=pr, q=qq, periods=b["periods"], series=b["series"], t0=t0)
    # the records in the library's column-major layout, (n, d) row-major for dfm_percentiles, and back
    recs = dict(contrib=d["contrib"].transpose(0, 3, 2, 1), rest=d["rest"].transpose(0, 2, 1), base=d["base"].transpose(0, 2, 1),
                shocks=d["shocks"][:, :, :shocks].transpose(0, 2, 1))
    for nm, v in recs.items():
        bd = lib.percentiles(v.reshape(n, -1), qq).reshape((len(qq),) + v.shape[1:])
        out[nm + "_bands"] = np.ascontiguousarray(bd.transpose((0,) + tuple(range(bd.ndim - 1, 0, -1))))
        if return_draws:
            dr = d[nm][..., :shocks] if nm == "shocks" else d[nm]
            out[nm + "_draws"] = dr.reshape((n_chain, n_keep) + dr.shape[1:])
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    out["rhat"] = dict(loglik=float(split_rhat(o["loglik"][:, kept])),
                       contrib=split_rhat(d["contrib"].reshape((n_chain, n_keep) + d["contrib"].shape[1:])))
    return out


def _sign_rows(restrictions, ns, H, n_shock, what):
    """[(series, shock, sign, horizons)] -> (rows as four int arrays (series, horizon, shock, sign), n_shock).  horizons: an int
    or an inclusive (lo, hi); n_shock defaults to the last restricted shock."""
    rows = []
    for rs in restrictions:
        i, j, s, hz = rs
        lo, hi = (int(hz), int(hz)) if np.isscalar(hz) else (int(hz[0]), int(hz[1]))
        if not 0 <= int(i) < ns:
            raise ValueError(f"{what}: series {i} is not an estimation series (0 .. {ns - 1})")
        if int(j) < 1 or int(s) not in (1, -1):
            raise ValueError(f"{what}: a restriction needs a shock >= 1 and a sign of +1 or -1, got {rs}")
        if not 0 <= lo <= hi < H:
            raise ValueError(f"{what}: horizons {hz} outside 0 .. H-1 = {H - 1}")
        rows += [(int(i), h, int(j), int(s)) for h in range(lo, hi + 1)]
    if not rows:
        raise ValueError(f"{what}: no restrictions")
    top = max(j for _, _, j, _ in rows)
    n_shock = top if n_shock is None else int(n_shock)
    if top > n_shock:
        raise ValueError(f"{what}: a restriction on shock {top} > n_shock = {n_shock}")
    return [np.array([rw[q] for rw in rows], np.int64) for q in range(4)], n_shock


def _sign_block(m, restrictions, H, n_shock, what, lib):
    if H <= 0:
        raise ValueError("H must be > 0")
    b = _state_space_block(m, 0, lib, what)
    rows, n_shock = _sign_rows(restrictions, b["Xs"].shape[1], H, n_shock, what)
    r = b["em"]["Q"].shape[0]
    if n_shock > r:
        raise ValueError(f"{what}: n_shock = {n_shock} > r = {r}")
    out = [int(i) for i in set(rows[0].tolist()) if np.isnan(b["Lam"][i]).any() or np.isnan(b["em"]["R"][i])]
    if out:
        raise ValueError(f"{what}: restricted series {sorted(out)} are out of the model")
    return b, rows, n_shock


def sign_identified_set(m, restrictions, H, n_shock=None, n_rot=2 ** 20, n_keep=4096, seed=20260922, q=(5, 16, 50, 84, 95),
                        lib=None):
    """Shocks identified by sign restrictions on the series responses of a model estimated with `estimate(m, Parametric())`, at
    its EM estimates m.em (any Parametric fit, with or without lam_constr_em) (dfm_sign_restrictions).

    restrictions: [(series, shock, sign, horizons)]: series is the 0-based position among the estimation series (the index
    convention of LambdaConstraint.indices and of forecast's `series`), shock 1-based, sign +1 / -1, horizons an int or an
    inclusive (lo, hi) in 0 .. H-1.  With L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L and c_{i,h} = lam_i' Psi_h, candidate rotations
    Omega are drawn from the Haar measure on the orthogonal group (n_rot per call, counter-based: candidate c is the same
    rotation whatever n_rot); Omega is kept when, for every restricted shock j, sign * c_{i,h} omega_j is of one strict sign over
    the shock's rows (omega_j flipped when all are negative).  The accepted set of series responses does not depend on the
    normalisation of the factors (f -> K f), so no loading restriction is needed.

    Returns a dict:
      resp, fevd (n_kept, ns, H, n_shock)   the first n_kept = min(n_accept, n_keep) accepted rotations' series responses in data
                                             units (xstd_i c_{i,h} Omega e_j) and variance decompositions (variance_decomposition's
                                             on the rotated shocks);  rot (n_kept, r, r), cand (n_kept,) their Omega and ids;
      resp_bands, fevd_bands (len(q), ns, H, n_shock)   percentiles over the kept draws (dfm_percentiles);
      resp_lo, resp_hi, fevd_lo, fevd_hi (ns, H, n_shock)   min and max over the kept draws: an inner estimate of the identified
                                             set at m.em;
      n_accept, accept_rate (= n_accept / n_rot);  and series, n_shock, q, rows (the expanded (series, horizon, shock, sign)).
    The bands describe the distribution over the identified set that the Haar prior on Omega induces at m.em, not sampling
    uncertainty about the parameters (sign_restricted_responses adds that).  A uniform prior over rotations is not uniform over
    the responses (Baumeister & Hamilton 2015).  n_keep <= 16384."""
    if not 1 <= n_keep <= 16384:
        raise ValueError("sign_identified_set: n_keep must be in [1, 16384]")
    b, rows, n_shock = _sign_block(m, restrictions, H, n_shock, "sign_identified_set", lib)
    lib, e = b["lib"], b["em"]
    o = lib.sign_restrictions(b["Lam"], e["R"], e["A"], e["Q"], rows, H, n_rot, n_keep, n_shock=n_shock, seed=seed, scale=b["xstd"])
    if o["status"] != 0:
        raise RuntimeError(f"sign_identified_set: device status {o['status']}")
    nk = int(min(o["n_accept"], n_keep))
    qq = np.asarray(q, float)
    out = dict(resp=np.ascontiguousarray(o["resp"][:nk]), fevd=np.ascontiguousarray(o["fevd"][:nk]),
               rot=np.ascontiguousarray(o["rot"][:nk]), cand=o["cand"][:nk].copy(), n_accept=int(o["n_accept"]),
               accept_rate=float(o["n_accept"]) / n_rot, series=b["series"], n_shock=n_shock, q=qq,
               rows=np.stack(rows, axis=1))
    ns = b["Xs"].shape[1]
    for nm in ("resp", "fevd"):
        if nk:
            bd = lib.percentiles(out[nm].reshape(nk, -1), np.r_[qq, 0.0, 100.0]).reshape((len(qq) + 2, ns, H, n_shock))
        else:
            bd = np.full((len(qq) + 2, ns, H, n_shock), np.nan)
        out[nm + "_bands"], out[nm + "_lo"], out[nm + "_hi"] = bd[:len(qq)], bd[len(qq)], bd[len(qq) + 1]
    return out


def sign_restricted_responses(m, restrictions, H, n_shock=None, n_chain=4, n_burn=500, n_keep=1000, thin=1, rot_per_draw=4, prior=None,
                              seed=20260922, q=(5, 16, 50, 84, 95), chain0=0, sweep0=0, lib=None):
    """Posterior bands of the series responses and variance decompositions of shocks identified by sign restrictions, over the
    parameter draws of Gibbs chains (gibbs: dfm_gibbs, started at m.em, same prior and refusals: a lam_constr_em fit is refused)
    and, per kept draw, rot_per_draw Haar candidate rotations (dfm_sign_restrictions, candidate ids keyed on the draw's
    gibbs_id(chain, sweep)).  Every accepted (draw, rotation) pair is kept: a draw from the joint posterior under the Haar prior
    on the rotation truncated to the sign set (Arias, Rubio-Ramirez & Waggoner 2018).  restrictions, H, n_shock: as
    sign_identified_set.

    Returns a dict:
      resp_draws, fevd_draws (n_chain, n_keep, rot_per_draw, ns, H, n_shock)   NaN where the rotation was rejected;
      resp_bands, fevd_bands (len(q), ns, H, n_shock)    percentiles over the accepted pairs (dfm_percentiles, NaN ignored);
      accept (n_chain, n_keep)  accepted share of each draw's rotations;  accept_rate  over all pairs;
      n_empty  draws with no accepted rotation;  status (n_chain), loglik (n_chain, n_burn + n_keep thin);
      rhat dict(loglik, accept)  split-R^ over the kept draws;
    and prior, series, n_shock, q.  n_chain n_keep rot_per_draw <= 16384."""
    if m.em is not None and m.em.get("lam_constr") is not None:
        raise ValueError("sign_restricted_responses: the EM of m ran under restrictions on the loadings (lam_constr_em); the sampler "
                         "draws unrestricted loadings")
    if rot_per_draw < 1 or not 1 <= n_chain * n_keep * rot_per_draw <= 16384:
        raise ValueError("sign_restricted_responses: n_chain * n_keep * rot_per_draw must be in [1, 16384]")
    b, rows, n_shock = _sign_block(m, restrictions, H, n_shock, "sign_restricted_responses", lib)
    lib, e = b["lib"], b["em"]
    r = e["Q"].shape[0]
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, prior=pr, outputs=("Lam", "R", "A", "Q"))
    n = n_chain * n_keep
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    ids = ((np.arange(chain0, chain0 + n_chain, dtype=np.uint64)[:, None] << np.uint64(24)) +
           (np.uint64(sweep0) + kept.astype(np.uint64))[None, :]).ravel()              # gibbs_id(chain, kept sweep)
    sh = lambda a_: a_.reshape((n,) + a_.shape[2:])
    d = lib.sign_restrictions(sh(o["Lam"]), sh(o["R"]), sh(o["A"]), sh(o["Q"]), rows, H, rot_per_draw, rot_per_draw, n_shock=n_shock,
                              seed=seed, ids=ids, scale=b["xstd"], outputs=("resp", "fevd"))
    ns = b["Xs"].shape[1]
    qq = np.asarray(q, float)
    acc = d["n_accept"].reshape(n_chain, n_keep) / rot_per_draw
    out = dict(accept=acc, accept_rate=float(acc.mean()), n_empty=int((d["n_accept"] == 0).sum()), status=o["status"], loglik=o["loglik"],
               prior=pr, series=b["series"], n_shock=n_shock, q=qq,
               rhat=dict(loglik=float(split_rhat(o["loglik"][:, kept])), accept=float(split_rhat(acc))))
    for nm in ("resp", "fevd"):
        dr = d[nm]
        out[nm + "_draws"] = dr.reshape((n_chain, n_keep, rot_per_draw, ns, H, n_shock))
        out[nm + "_bands"] = lib.percentiles(dr.reshape(n * rot_per_draw, -1), qq).reshape((len(qq), ns, H, n_shock))
    return out


def _narr_rows(m, narrative, ns, H, p, what):
    """Narrative tuples -> six int arrays (kind, shock, series, row, h, sign) for the library, rows 0-based in the estimation
    block.  ("shock", shock, period, sign), ("most" | "overwhelming", shock, series, period, h), ("contrib", shock, series,
    period, h, sign); periods 1-based like historical_decomposition's t0."""
    from ._lib import NARR_KINDS
    out = []
    for row in narrative:
        kd = NARR_KINDS.get(row[0]) if len(row) else None
        size = {0: 4, 1: 5, 2: 5, 3: 6}.get(kd)
        if kd is None or len(row) != size:
            raise ValueError(f"{what}: narrative row {row} is not ('shock', j, period, sign), ('most' | 'overwhelming', j, series, "
                             "period, h) or ('contrib', j, series, period, h, sign)")
        if kd == 0:
            j, i, per, h, s = int(row[1]), 0, int(row[2]), 0, int(row[3])
        else:
            j, i, per, h = int(row[1]), int(row[2]), int(row[3]), int(row[4])
            s = int(row[5]) if kd == 3 else 1
            if not 0 <= i < ns:
                raise ValueError(f"{what}: narrative row {row}: series {i} is not an estimation series (0 .. {ns - 1})")
            if not 0 <= h < H:
                raise ValueError(f"{what}: narrative row {row}: h outside 0 .. H-1 = {H - 1}")
        if j < 1 or s not in (1, -1):
            raise ValueError(f"{what}: narrative row {row} needs a shock >= 1 and a sign of +1 or -1")
        lo = m.initperiod + p
        if per < lo or per + h > m.lastperiod:
            raise ValueError(f"{what}: narrative row {row}: periods {per} .. {per + h} outside {lo} .. {m.lastperiod} "
                             "(initperiod + p .. lastperiod)")
        out.append((kd, j, i, per - m.initperiod, h, s))
    return [np.array([rw[q] for rw in out], np.int64) for q in range(6)]


def _narr_block(m, restrictions, narrative, H, n_shock, what, lib):
    if H <= 0:
        raise ValueError("H must be > 0")
    b = _state_space_block(m, 0, lib, what)
    ns = b["Xs"].shape[1]
    rows, ns_sign = _sign_rows(restrictions, ns, H, None, what) if restrictions else ([np.zeros(0, np.int64)] * 4, 1)
    narr = _narr_rows(m, narrative, ns, H, b["p"], what)
    top = max([ns_sign] + ([int(narr[1].max())] if len(narr[1]) else []))
    n_shock = top if n_shock is None else int(n_shock)
    r = b["em"]["Q"].shape[0]
    if top > n_shock:
        raise ValueError(f"{what}: a restriction on shock {top} > n_shock = {n_shock}")
    if n_shock > r:
        raise ValueError(f"{what}: n_shock = {n_shock} > r = {r}")
    used = set(rows[0].tolist()) | set(narr[2][narr[0] != 0].tolist())
    out = [int(i) for i in used if np.isnan(b["Lam"][i]).any() or np.isnan(b["em"]["R"][i])]
    if out:
        raise ValueError(f"{what}: restricted series {sorted(out)} are out of the model")
    return b, rows, narr, n_shock


def _weighted_bands(lib, recs, w, q, shape):
    """Weighted percentile bands of recs (n, ...) with weights w (n,) (dfm_percentiles_weighted; NaN without a counted draw)."""
    n = recs.shape[0]
    if n == 0 or not ((w > 0) & np.isfinite(w)).any():
        return np.full((len(q),) + shape, np.nan)
    return lib.percentiles_weighted(recs.reshape(n, -1), w, q).reshape((len(q),) + shape)


def narrative_identified_set(m, restrictions, narrative, H, n_shock=None, n_rot=2 ** 20, n_keep=4096, n_sim=2 ** 14, seed=20260922,
                             q=(5, 16, 50, 84, 95), history=False, t0=None, return_draws=False, lib=None):
    """Shocks identified by sign restrictions plus narrative restrictions on dated episodes (Antolin-Diaz & Rubio-Ramirez 2018), at
    the EM estimates m.em of a model estimated with `estimate(m, Parametric())` (dfm_narrative_sign_restrictions).

    restrictions: sign_identified_set's (may be empty).  narrative: tuples, periods 1-based in initperiod + p .. lastperiod:
      ("shock", j, period, sign)                 sign * eps~_{j,period} > 0;
      ("most", j, series, period, h)             shock j contributes more than any other shock to the change of `series` over
                                                 period .. period + h that was not forecast at period - 1 (|H_j| > max |H_k|);
      ("overwhelming", j, series, period, h)     ... more than all the other shocks together (|H_j| > sum |H_k|);
      ("contrib", j, series, period, h, sign)    sign * H_j > 0;
    with H_k = historical_decomposition's contribution of shock k at period + h from base period - 1, on the rotated model.
    The path is the smoothed factor path at m.em, so the rows restrict E[eps | data, theta^], not the shocks themselves
    (narrative_restricted_responses restricts the path drawn with each parameter draw, a joint posterior draw).

    Each kept draw is weighted by 1 / w, w the probability of the narrative event under N(0, I) shocks estimated from n_sim
    simulations (weight = n_sim / n_ok).  Returns sign_identified_set's dict (resp, fevd, rot, cand, n_accept, accept_rate,
    resp_lo / hi, fevd_lo / hi: the inner estimate of the identified set, unweighted) with resp_bands / fevd_bands WEIGHTED
    (numpy's inverted_cdf rule with weights, cumulative weights exact: dfm_percentiles_weighted), plus:
      weight, n_ok (n_kept,);  ess = (sum w)^2 / sum w^2;  n_zero_omega: kept draws with n_ok = 0 (dropped from the bands);
      eps (n_kept, T, n_shock)   the identified shocks' paths eps~_t = Omega' L^-1 (f_t - sum A_l f_{t-l}) (NaN for the first p);
    and narrative (the library's rows: kind, shock, series, row, h, sign).

    history=True adds `history`, weighted bands of the identified shocks' historical decompositions over the kept draws:
    dfm_historical_decomposition of each kept draw's rotated model (loadings Lam L Omega, lags Omega' L^-1 A_l L Omega, Q = I
    exactly) along its rotated path Omega' L^-1 f, from base period t0 (historical_decomposition's t0 and default), in data
    units: contrib_bands (len(q), ns, T, n_shock), rest_bands (len(q), ns, T) (the other shocks summed), and t0, periods; with
    return_draws=True also contrib_draws (n_kept, ns, T, n_shock) and rest_draws (n_kept, ns, T).  With t0 = period - 1, contrib
    at `period` is the H_j of a ("most", j, series, period, 0) row times xstd.  The draws' decompositions are held in host
    memory while the bands are taken: about 1.1 GB at n_keep = 4096, n_shock = 1 on Stock & Watson's Figure 7 block (139 series,
    120 periods).  n_keep <= 16384."""
    if not 1 <= n_keep <= 16384:
        raise ValueError("narrative_identified_set: n_keep must be in [1, 16384]")
    b, rows, narr, n_shock = _narr_block(m, restrictions, narrative, H, n_shock, "narrative_identified_set", lib)
    lib, e = b["lib"], b["em"]
    t0, row0, F = _history_rows(m, b, t0, "narrative_identified_set")
    o = lib.narrative_sign_restrictions(b["Lam"], e["R"], e["A"], e["Q"], F, rows, narr, H, n_rot, n_keep, n_shock=n_shock, n_sim=n_sim,
                                        seed=seed, scale=b["xstd"])
    if o["status"] != 0:
        raise RuntimeError(f"narrative_identified_set: device status {o['status']}")
    nk = int(min(o["n_accept"], n_keep))
    qq = np.asarray(q, float)
    w = o["weight"][:nk].copy()
    fin = np.isfinite(w)
    out = dict(resp=np.ascontiguousarray(o["resp"][:nk]), fevd=np.ascontiguousarray(o["fevd"][:nk]),
               rot=np.ascontiguousarray(o["rot"][:nk]), cand=o["cand"][:nk].copy(), n_accept=int(o["n_accept"]),
               accept_rate=float(o["n_accept"]) / n_rot, weight=w, n_ok=o["n_ok"][:nk].copy(),
               ess=float(w[fin].sum() ** 2 / (w[fin] ** 2).sum()) if fin.any() else 0.0, n_zero_omega=int((~fin).sum()),
               eps=np.ascontiguousarray(o["eps"][:nk]), series=b["series"], n_shock=n_shock, q=qq,
               rows=np.stack(rows, axis=1), narrative=np.stack(narr, axis=1))
    ns = b["Xs"].shape[1]
    for nm in ("resp", "fevd"):
        shape = (ns, H, n_shock)
        out[nm + "_bands"] = _weighted_bands(lib, out[nm], w, qq, shape)
        lohi = lib.percentiles(out[nm].reshape(nk, -1), [0.0, 100.0]).reshape((2,) + shape) if nk else np.full((2,) + shape, np.nan)
        out[nm + "_lo"], out[nm + "_hi"] = lohi[0], lohi[1]
    if history:
        out["history"] = _narr_history(lib, b, F, row0, out["rot"], w, n_shock, qq, return_draws)
        out["history"].update(t0=t0, periods=b["periods"])
    return out


def _narr_history(lib, b, F, row0, rot, w, n_shock, qq, return_draws):
    """Weighted bands of the historical decompositions of the rotated models (Lam L Omega, Omega' L^-1 A_l L Omega, I) along the
    rotated paths Omega' L^-1 f of the kept draws rot (n, r, r), from base row row0."""
    e = b["em"]
    ns, T = b["Xs"].shape[1], F.shape[0]
    n, r = rot.shape[0], rot.shape[1]
    shape_c, shape_r = (ns, T, n_shock), (ns, T)
    if n == 0:
        return dict(contrib_bands=np.full((len(qq),) + shape_c, np.nan), rest_bands=np.full((len(qq),) + shape_r, np.nan))
    Lc = np.linalg.cholesky(e["Q"]); Li = np.linalg.inv(Lc)
    p = e["A"].shape[1] // r
    Lam = np.einsum("ia,ab,nbc->nic", b["Lam"], Lc, rot)
    A = np.concatenate([np.einsum("nba,bc,ncd->nad", rot, Li @ e["A"][:, l * r:(l + 1) * r] @ Lc, rot) for l in range(p)], axis=2)
    Fr = np.einsum("tc,nca->nta", F @ Li.T, rot)
    d = lib.historical_decomposition(Lam, np.broadcast_to(e["R"], (n, ns)), A, np.broadcast_to(np.eye(r), (n, r, r)), Fr, row0,
                                     n_shock=n_shock, scale=b["xstd"], outputs=("contrib", "rest"))
    if (d["status"] != 0).any():
        raise RuntimeError(f"narrative_identified_set: device status {d['status'][d['status'] != 0][0]} in the history")
    out = dict(contrib_bands=_weighted_bands(lib, d["contrib"], w, qq, shape_c), rest_bands=_weighted_bands(lib, d["rest"], w, qq, shape_r))
    if return_draws:
        out.update(contrib_draws=d["contrib"], rest_draws=d["rest"])
    return out


def narrative_restricted_responses(m, restrictions, narrative, H, n_shock=None, n_chain=4, n_burn=500, n_keep=1000, thin=1,
                                   rot_per_draw=4, n_sim=2 ** 14, prior=None, seed=20260922, q=(5, 16, 50, 84, 95), chain0=0, sweep0=0,
                                   lib=None):
    """Posterior bands under sign and narrative restrictions: Gibbs chains (gibbs: dfm_gibbs from m.em, same prior and refusals: a
    lam_constr_em fit is refused) record each kept draw's parameters and factor path; per kept draw, rot_per_draw Haar candidates
    (ids keyed on gibbs_id(chain, sweep), as sign_restricted_responses) are tested against the sign rows and the narrative rows
    evaluated on THAT draw's path, so the rows restrict the shocks of a joint posterior draw of parameters and path.  Every
    accepted pair is kept with importance weight n_sim / n_ok (narrative_identified_set).  restrictions, narrative, H, n_shock:
    as narrative_identified_set.

    Returns a dict:
      resp_draws, fevd_draws (n_chain, n_keep, rot_per_draw, ns, H, n_shock)   NaN where the rotation was rejected;
      weight (n_chain, n_keep, rot_per_draw)   NaN where rejected, +Inf where no simulation satisfied the rows;
      resp_bands, fevd_bands (len(q), ns, H, n_shock)   weighted percentiles over the accepted pairs (dfm_percentiles_weighted);
      ess, n_zero_omega;  accept (n_chain, n_keep), accept_rate, n_empty, status (n_chain), loglik;
      rhat dict(loglik, accept)  split-R^ over the kept draws;
    and prior, series, n_shock, q.  n_chain n_keep rot_per_draw <= 16384 (the defaults give 16 000)."""
    if m.em is not None and m.em.get("lam_constr") is not None:
        raise ValueError("narrative_restricted_responses: the EM of m ran under restrictions on the loadings (lam_constr_em); the "
                         "sampler draws unrestricted loadings")
    if rot_per_draw < 1 or not 1 <= n_chain * n_keep * rot_per_draw <= 16384:
        raise ValueError("narrative_restricted_responses: n_chain * n_keep * rot_per_draw must be in [1, 16384]")
    b, rows, narr, n_shock = _narr_block(m, restrictions, narrative, H, n_shock, "narrative_restricted_responses", lib)
    lib, e = b["lib"], b["em"]
    r = e["Q"].shape[0]
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, prior=pr, outputs=("Lam", "R", "A", "Q", "F"))
    n = n_chain * n_keep
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    ids = ((np.arange(chain0, chain0 + n_chain, dtype=np.uint64)[:, None] << np.uint64(24)) +
           (np.uint64(sweep0) + kept.astype(np.uint64))[None, :]).ravel()              # gibbs_id(chain, kept sweep)
    sh = lambda a_: a_.reshape((n,) + a_.shape[2:])
    d = lib.narrative_sign_restrictions(sh(o["Lam"]), sh(o["R"]), sh(o["A"]), sh(o["Q"]), sh(o["F"]), rows, narr, H, rot_per_draw,
                                        rot_per_draw, n_shock=n_shock, n_sim=n_sim, seed=seed, ids=ids, scale=b["xstd"],
                                        outputs=("resp", "fevd", "weight"))
    ns = b["Xs"].shape[1]
    qq = np.asarray(q, float)
    acc = d["n_accept"].reshape(n_chain, n_keep) / rot_per_draw
    w = d["weight"].reshape(-1)
    fin = np.isfinite(w)
    out = dict(accept=acc, accept_rate=float(acc.mean()), n_empty=int((d["n_accept"] == 0).sum()), status=o["status"], loglik=o["loglik"],
               weight=d["weight"].reshape(n_chain, n_keep, rot_per_draw), prior=pr, series=b["series"], n_shock=n_shock, q=qq,
               ess=float(w[fin].sum() ** 2 / (w[fin] ** 2).sum()) if fin.any() else 0.0,
               n_zero_omega=int(np.isinf(w).sum()),
               rhat=dict(loglik=float(split_rhat(o["loglik"][:, kept])), accept=float(split_rhat(acc))))
    for nm in ("resp", "fevd"):
        dr = d[nm]
        out[nm + "_draws"] = dr.reshape((n_chain, n_keep, rot_per_draw, ns, H, n_shock))
        out[nm + "_bands"] = _weighted_bands(lib, dr.reshape(n * rot_per_draw, -1), np.where(fin, w, 0.0), qq, (ns, H, n_shock))
    return out


def _proxy_inputs(m, b, z, normalize, H, block, what):
    """(Z (T, n_inst), instrument names, i0, block length) of proxy_identified_responses' arguments."""
    if H <= 0:
        raise ValueError("H must be > 0")
    T = m.lastperiod - m.initperiod + 1
    if isinstance(z, dict):
        names = [str(k) for k in z]
        Z = np.column_stack([np.asarray(v, float).reshape(-1) for v in z.values()]) if z else np.zeros((T, 0))
    else:
        Z = np.asarray(z, float)
        Z = Z.reshape(-1, 1) if Z.ndim == 1 else Z
        names = [str(k) for k in range(Z.shape[1])]
    if Z.ndim != 2 or Z.shape[0] != T or not 1 <= Z.shape[1] <= 8:
        raise ValueError(f"{what}: z must hold 1 .. 8 instruments over the estimation block's {T} rows, got shape {Z.shape}")
    ns = b["Xs"].shape[1]
    i0 = int(normalize)
    if not 0 <= i0 < ns:
        raise ValueError(f"{what}: normalize = {normalize} is not an estimation series (0 .. {ns - 1})")
    if np.isnan(b["Lam"][i0]).any() or np.isnan(b["em"]["R"][i0]):
        raise ValueError(f"{what}: the normalising series {i0} is out of the model")
    block = max(1, int(round(T ** (1.0 / 3.0)))) if block is None else int(block)
    if block < 1:
        raise ValueError(f"{what}: block must be >= 1")
    return Z, names, i0, block


def _proxy_bands(lib, d, recs, i0, qq, shape):
    """Percentile bands of resp, resp_unit (resp / resp[i0, 0] of the same record) and fevd over the record axis of d[...] (n_inst,
    n_rec, ns, H), returned (len(q), ns, H, n_inst)."""
    out = {}
    resp = d["resp"][:, recs]
    unit = resp / resp[:, :, i0:i0 + 1, :1]
    for nm, v in (("resp", resp), ("resp_unit", unit), ("fevd", d["fevd"][:, recs])):
        n = v.shape[1]
        bd = lib.percentiles(np.ascontiguousarray(v.transpose(1, 2, 3, 0)).reshape(n, -1), qq)
        out[nm + "_bands"] = bd.reshape((len(qq),) + shape)
    return out


def proxy_identified_responses(m, z, normalize, H, n_boot=4096, block=None, q=0, seed=20260922, q_bands=(5, 16, 50, 84, 95),
                               return_draws=False, lib=None):
    """Shocks identified by external instruments (proxy SVAR / SVAR-IV, Stock & Watson 2018) at the EM estimates m.em of a model
    estimated with `estimate(m, Parametric())`, with or without lam_constr_em (dfm_proxy_identification).

    z: an array (T,) or (T, n_inst), or a dict name -> (T,) array, over the estimation block's rows initperiod .. lastperiod (NaN
    where the instrument is unavailable); at most 8 instruments, each identifying its own shock.  normalize: the 0-based
    estimation series i0 (the index convention of sign_identified_set) whose impact response is the unit effect, e.g. an oil
    price.  With the smoothed factor path at m.em (kalman_smooth, as historical_decomposition), L = chol(Q), the innovations
    eta_t = f_t - sum_l A_l f_{t-l} and an instrument's periods T_k (z finite, t > p lags into the sample):
      omega_k = L^-1 Gamma_k / |L^-1 Gamma_k|, Gamma_k = mean over T_k of eta_t (z_t - zbar): the shock's column of the impact
      matrix is b_k = L omega_k, a one-standard-deviation shock covarying positively with its instrument.  None of the results
      depends on the normalisation of the factors (f -> K f; DESIGN.md 4.16), so no loading restriction is needed.
    Returns a dict (instruments on the last axis):
      resp, fevd (ns, H, n_inst)        xstd_i lam_i' Psi_h omega_k in data units, and the share of the (h+1)-step forecast-error
                                         variance (variance_decomposition's formula for one shock);
      resp_unit (ns, H, n_inst)         resp / resp[i0, 0]: the unit-effect normalisation (a shock moving series i0 by one unit
                                         on impact);
      eps (T, n_inst)                   the identified shock's path omega_k' L^-1 eta_t (NaN for the first p rows);
      omega (n_inst, r), reliability, first_stage_F, first_stage_pi, n_obs (n_inst,): reliability = |L^-1 Gamma_k|^2 / s^2_z,
                                         the squared correlation of the instrument with the shock under the model's Q, reported as
                                         computed (along the smoothed path, whose innovations are shrunk, it can exceed 1);
                                         first_stage_F: Stock & Watson's HAC(q) first-stage F of lam_i0' eta_t on [1, z_t];
      shock_corr (n_inst, n_inst)       omega_k' omega_l: the correlation of the shocks two instruments identify (1 when they
                                         identify the same shock);
      resp_bands, resp_unit_bands, fevd_bands (len(q_bands), ns, H, n_inst)   percentiles over the n_boot moving-block bootstrap
                                         replicates of the instrument moments (dfm_percentiles);
      resp_draws, resp_unit_draws, fevd_draws (n_boot, ns, H, n_inst)   only with return_draws=True: the replicates' records;
    and status (n_inst,), names, series, q, block, periods.
    The bands hold theta = m.em and the path fixed: they describe the instrument-side sampling uncertainty only
    (proxy_restricted_responses adds parameter and path uncertainty).  block: the bootstrap's block length, default
    round(T^(1/3)) (the rate that balances the bias and variance of a block bootstrap variance estimate); the periods where an
    instrument is missing are skipped, so a block may join periods across a gap.  n_boot <= 16384."""
    if not 1 <= n_boot <= 16384:
        raise ValueError("proxy_identified_responses: n_boot must be in [1, 16384]")
    b = _state_space_block(m, 0, lib, "proxy_identified_responses")
    lib, e = b["lib"], b["em"]
    Z, names, i0, block = _proxy_inputs(m, b, z, normalize, H, block, "proxy_identified_responses")
    o = lib.kalman_smooth(b["Xs"], b["Lam"], e["R"], e["A"], e["Q"], p=b["p"], P0=e["P0"], H=0, outputs=("F",))
    if o["status"] != 0:
        raise RuntimeError(f"proxy_identified_responses: device status {o['status']}")
    d = lib.proxy_identification(b["Lam"], e["R"], e["A"], e["Q"], o["F"], Z, i0, H, n_boot=n_boot, block=block, q=q, seed=seed,
                                 scale=b["xstd"])
    bad = np.flatnonzero(d["status"] != 0)
    if len(bad):
        raise RuntimeError(f"proxy_identified_responses: instrument(s) {[names[k] for k in bad]} failed with status "
                           f"{d['status'][bad].tolist()} (3: a failed model, fewer than 3 usable periods or no covariance with the "
                           "innovations)")
    qq = np.asarray(q_bands, float)
    ns = b["Xs"].shape[1]
    mv = lambda a_: np.ascontiguousarray(np.moveaxis(a_, 0, -1))
    om = d["omega"][:, 0]
    resp = d["resp"][:, 0]
    out = dict(resp=mv(resp), resp_unit=mv(resp / resp[:, i0:i0 + 1, :1]), fevd=mv(d["fevd"][:, 0]), eps=mv(d["eps"]),
               omega=np.ascontiguousarray(om), reliability=d["reliability"].copy(), first_stage_F=d["fs_F"].copy(),
               first_stage_pi=d["fs_pi"].copy(), n_obs=d["n_obs"].astype(int), shock_corr=om @ om.T, status=d["status"].copy(),
               names=names, series=b["series"], q=qq, block=block, periods=b["periods"])
    out.update(_proxy_bands(lib, d, slice(1, None), i0, qq, (ns, H, len(names))))
    if return_draws:
        rr = d["resp"][:, 1:]
        for nm, v in (("resp", rr), ("resp_unit", rr / rr[:, :, i0:i0 + 1, :1]), ("fevd", d["fevd"][:, 1:])):
            out[nm + "_draws"] = np.ascontiguousarray(np.moveaxis(v, 0, -1))
    return out


def proxy_restricted_responses(m, z, normalize, H, n_chain=4, n_burn=500, n_keep=1000, thin=1, boot_per_draw=1, block=None, q=0,
                               prior=None, seed=20260922, q_bands=(5, 16, 50, 84, 95), chain0=0, sweep0=0, lib=None):
    """Bands of the instrument-identified responses over Gibbs parameter and path draws: gibbs (dfm_gibbs from m.em, same prior and
    refusals: a lam_constr_em fit is refused, the sampler draws unrestricted loadings) records each kept draw's parameters and
    factor path, and one dfm_proxy_identification over all kept draws identifies each draw's shocks along its own path, with
    boot_per_draw moving-block bootstrap replicates of the instrument moments per draw (ids gibbs_id(chain, kept sweep), as
    sign_restricted_responses).  z, normalize, H, block, q: as proxy_identified_responses.

    This combines posterior draws of the parameters and the path with a block bootstrap of the instrument moments; it is not a
    fully Bayesian proxy model (the instrument's own likelihood, as in Caldara & Herbst 2019, is not part of the posterior).

    Returns a dict:
      resp_bands, resp_unit_bands, fevd_bands (len(q_bands), ns, H, n_inst)   percentiles over every (draw, replicate) record
                   (replicates 1 .. boot_per_draw of every draw; with boot_per_draw = 0, replicate 0, the draw's own sample);
      reliability, first_stage_F (n_chain, n_keep, n_inst)   of each draw (replicate 0);
      proxy_status (n_chain, n_keep, n_inst)   dfm_proxy_identification's status (a failed chain's draws are 3);
      status (n_chain), loglik (n_chain, n_burn + n_keep thin), rhat dict(loglik)   split-R^ over the kept draws;
    and prior, names, series, q, block.  n_chain n_keep max(1, boot_per_draw) <= 16384."""
    if m.em is not None and m.em.get("lam_constr") is not None:
        raise ValueError("proxy_restricted_responses: the EM of m ran under restrictions on the loadings (lam_constr_em); the sampler "
                         "draws unrestricted loadings")
    nrb = max(1, int(boot_per_draw))
    if boot_per_draw < 0 or not 1 <= n_chain * n_keep * nrb <= 16384:
        raise ValueError("proxy_restricted_responses: n_chain * n_keep * max(1, boot_per_draw) must be in [1, 16384]")
    b = _state_space_block(m, 0, lib, "proxy_restricted_responses")
    lib, e = b["lib"], b["em"]
    Z, names, i0, block = _proxy_inputs(m, b, z, normalize, H, block, "proxy_restricted_responses")
    r = e["Q"].shape[0]
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, prior=pr, outputs=("Lam", "R", "A", "Q", "F"))
    n = n_chain * n_keep
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    ids = ((np.arange(chain0, chain0 + n_chain, dtype=np.uint64)[:, None] << np.uint64(24)) +
           (np.uint64(sweep0) + kept.astype(np.uint64))[None, :]).ravel()              # gibbs_id(chain, kept sweep)
    sh = lambda a_: a_.reshape((n,) + a_.shape[2:])
    d = lib.proxy_identification(sh(o["Lam"]), sh(o["R"]), sh(o["A"]), sh(o["Q"]), sh(o["F"]), Z, i0, H, n_boot=int(boot_per_draw),
                                 block=block, q=q, seed=seed, ids=ids, scale=b["xstd"], outputs=("resp", "fevd", "reliability", "fs_F"))
    ns, ni = b["Xs"].shape[1], Z.shape[1]
    # records (n_inst, n_draw * nrb, ns, H): the draws' replicates 1 .. boot_per_draw (or replicate 0)
    sel = slice(1, None) if boot_per_draw > 0 else slice(0, 1)
    dd = {nm: np.moveaxis(d[nm][:, :, sel], 1, 0).reshape((ni, n * nrb, ns, H)) for nm in ("resp", "fevd")}
    qq = np.asarray(q_bands, float)
    out = dict(reliability=d["reliability"].reshape(n_chain, n_keep, ni), first_stage_F=d["fs_F"].reshape(n_chain, n_keep, ni),
               proxy_status=d["status"].reshape(n_chain, n_keep, ni), status=o["status"], loglik=o["loglik"], prior=pr, names=names,
               series=b["series"], q=qq, block=block, rhat=dict(loglik=float(split_rhat(o["loglik"][:, kept]))))
    out.update(_proxy_bands(lib, dd, slice(None), i0, qq, (ns, H, ni)))
    return out


def parametric_bootstrap(m, n_rep, H_irf=24, H_fc=0, fc_rows=None, seed=20260922, q=(5, 16, 50, 84, 95), max_iter=50, tol=0.0, rep0=0,
                         lib=None):
    """Parametric bootstrap of a model estimated with `estimate(m, Parametric())` (dfm_ss_bootstrap): n_rep panels are drawn
    from the state-space model at m.em (with the estimation block's missing pattern and ragged edge), the EM re-runs on all of
    them from m.em (max_iter / tol as Parametric), and every replicate is rotated back onto m.em's factors.  Bands over the
    replicates carry the estimation uncertainty of the parameters, which forecast / forecast_bands / posterior_draws leave out.

    Same block as `forecast(m, H_fc)`.  fc_rows: trailing rows of the T + H_fc forecast rows returned per replicate (default
    H_fc; more rows include the ragged edge).  Returns a dict:
      Lam (n_rep, ns, r), R (n_rep, ns), A (n_rep, r, k), Q (n_rep, r, r)   aligned parameter draws (standardized units);
      irf (n_rep, r, H_irf, r)          impulse responses [variable, horizon, shock];  irf_point = parametric_irf(m, H_irf);
      irf_bands (len(q), r, H_irf, r)   percentiles of irf over the replicates (device, dfm_percentiles; failed replicates
                                        ignored);
      xhat (n_rep, fc_rows, ns)         E[x | data] at each replicate's parameters, data units;  xhat_bands (len(q), fc_rows, ns);
      xvar (n_rep, fc_rows, ns)         Var[x | data] at each replicate's parameters, data units;
      total_var (fc_rows, ns)           mean_b xvar_b + var_b xhat_b (law of total variance: filtering and parameter uncertainty);
      loglik, iters, status (n_rep)     the replicates' EM results (status != 0: failed, NaN records);
    and periods (the fc_rows rows, 1-based), series, q.  Series left out of the model have NaN columns.  n_rep <= 16384."""
    if m.em is not None and m.em.get("lam_constr") is not None:
        raise ValueError("parametric_bootstrap: the EM of m ran under restrictions on the loadings (lam_constr_em); the bootstrap "
                         "re-estimates without them and its rotation onto m.em would undo them")
    if not 1 <= n_rep <= 16384:
        raise ValueError("parametric_bootstrap: n_rep must be in [1, 16384]")
    if H_irf <= 0:
        raise ValueError("parametric_bootstrap: H_irf must be > 0")
    b = _state_space_block(m, H_fc, lib, "parametric_bootstrap")
    lib, e = b["lib"], b["em"]
    T = b["Xs"].shape[0]
    fc_rows = H_fc if fc_rows is None else int(fc_rows)
    if not 0 <= fc_rows <= T + H_fc:
        raise ValueError(f"parametric_bootstrap: fc_rows must be in [0, {T + H_fc}]")
    o = lib.ss_bootstrap(b["Xs"], b["Lam"], e["R"], e["A"], e["Q"], e["P0"], p=b["p"], n_rep=n_rep, seed=seed, rep0=rep0, H_irf=H_irf,
                         H_fc=H_fc, fc_rows=fc_rows, max_iter=max_iter, tol=tol)
    qq = np.asarray(q, float)
    r = e["Q"].shape[0]
    out = dict(Lam=o["Lam"], R=o["R"], A=o["A"], Q=o["Q"], irf=o["irf"], irf_point=parametric_irf(m, H_irf, lib=lib),
               irf_bands=lib.percentiles(o["irf"].reshape(n_rep, -1), qq).reshape(len(qq), r, H_irf, r),
               loglik=o["loglik"], iters=o["iters"], status=o["status"], periods=b["periods"][len(b["periods"]) - fc_rows:],
               series=b["series"], q=qq)
    if fc_rows > 0:
        xstd, ok = b["xstd"], o["status"] == 0
        xh = b["xmean"] + xstd * o["xhat"]
        xv = xstd ** 2 * o["xvar"]
        out.update(xhat=xh, xvar=xv, xhat_bands=lib.percentiles(xh.reshape(n_rep, -1), qq).reshape((len(qq),) + xh.shape[1:]),
                   total_var=xv[ok].mean(0) + xh[ok].var(0) if ok.any() else np.full(xh.shape[1:], np.nan))
    return out


def split_rhat(draws):
    """Split-R^ (Gelman et al. 2013, Bayesian Data Analysis 3rd ed., section 11.4) of draws (n_chain, n, ...): every chain cut in
    two halves, R^ = sqrt(((n'-1)/n' W + B/n') / W) over the 2 n_chain half-chains of length n'.  NaN when n < 4 or a chain
    failed (NaN draws)."""
    d = np.asarray(draws, float)
    h = d.shape[1] // 2
    if h < 2:
        return np.full(d.shape[2:], np.nan)
    s = np.concatenate([d[:, :h], d[:, h:2 * h]], axis=0)
    W = s.var(axis=1, ddof=1).mean(axis=0)
    B = h * s.mean(axis=1).var(axis=0, ddof=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.sqrt(((h - 1) / h * W + B / h) / W)


def gibbs(m, n_chain=4, n_burn=500, n_keep=1000, thin=1, H_irf=24, H_fc=0, fc_rows=None, prior=None, seed=20260922,
          q=(5, 16, 50, 84, 95), chain0=0, sweep0=0, lib=None):
    """Bayesian estimation of a model estimated with `estimate(m, Parametric())` by Gibbs sampling (dfm_gibbs): n_chain chains,
    all started at m.em, alternate a joint draw of the factor path (the simulation smoother) with conjugate draws of the
    parameters.  Prior (standardized units; `prior` overrides entries of the default, which is weak next to T of a few hundred):
      lam_i | R_i ~ N(0, R_i / kap_lam I),  R_i ~ IG(a_R, b_R),  A' | Q ~ MN(0, I / kap_A, Q),  Q ~ IW(nu_Q, s_Q I);
      defaults kap_lam = kap_A = 0.01, a_R = 3, b_R = 1, nu_Q = r + 2, s_Q = 1.  P0 stays at m.em's; A is not restricted to be
      stationary.
    Same block as `forecast(m, H_fc)`; fc_rows: trailing rows of the T + H_fc rows whose predictive draws are returned (default
    H_fc).  Returns a dict:
      Lam (n_chain, n_keep, ns, r), R (.., ns), A (.., r, k), Q (.., r, r)   raw parameter draws (standardized units);
      irf (n_chain, n_keep, r, H_irf, r)   impulse responses [variable, horizon, shock] of each draw rotated onto m.em
                                           (parametric_bootstrap's alignment);  irf_bands (len(q), r, H_irf, r);
      x (n_chain, n_keep, fc_rows, ns)     predictive draws in data units (the data where observed);  x_bands (len(q), fc_rows, ns);
      loglik (n_chain, n_burn + n_keep thin)  log-likelihood of the parameters entering each sweep;  status (n_chain);
      rhat dict(loglik, R (ns), x (fc_rows, ns))  split-R^ over the kept draws (the loglik of kept sweeps);
    and periods (the fc_rows rows, 1-based), series, q.  Bands through dfm_percentiles (n_chain n_keep <= 16384)."""
    if m.em is not None and m.em.get("lam_constr") is not None:
        raise ValueError("gibbs: the EM of m ran under restrictions on the loadings (lam_constr_em); the sampler draws unrestricted "
                         "loadings")
    if not 1 <= n_chain * n_keep <= 16384:
        raise ValueError("gibbs: n_chain * n_keep must be in [1, 16384]")
    b = _state_space_block(m, H_fc, lib, "gibbs")
    lib, e = b["lib"], b["em"]
    T = b["Xs"].shape[0]
    fc_rows = H_fc if fc_rows is None else int(fc_rows)
    if not 0 <= fc_rows <= T + H_fc:
        raise ValueError(f"gibbs: fc_rows must be in [0, {T + H_fc}]")
    r = e["Q"].shape[0]
    pr = dict(_gibbs_default_prior(r)); pr.update(prior or {})
    init = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"])
    ref = dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"])
    outs = ("Lam", "R", "A", "Q") + (("irf",) if H_irf > 0 else ()) + (("X",) if fc_rows > 0 else ())
    o = lib.gibbs(b["Xs"], init, p=b["p"], n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin,
                  seed=seed, H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, prior=pr, ref=ref if H_irf > 0 else None, outputs=outs)
    qq = np.asarray(q, float)
    n = n_chain * n_keep
    kept = n_burn + thin * np.arange(1, n_keep + 1) - 1
    out = dict(Lam=o["Lam"], R=o["R"], A=o["A"], Q=o["Q"], loglik=o["loglik"], status=o["status"], prior=pr,
               periods=b["periods"][len(b["periods"]) - fc_rows:], series=b["series"], q=qq,
               rhat=dict(loglik=float(split_rhat(o["loglik"][:, kept])), R=split_rhat(o["R"])))
    if H_irf > 0:
        out["irf"] = o["irf"]
        out["irf_bands"] = lib.percentiles(o["irf"].reshape(n, -1), qq).reshape((len(qq),) + o["irf"].shape[2:])
    if fc_rows > 0:
        x = b["xmean"] + b["xstd"] * o["X"]
        out["x"] = x
        out["x_bands"] = lib.percentiles(x.reshape(n, -1), qq).reshape((len(qq),) + x.shape[2:])
        out["rhat"]["x"] = split_rhat(x)
    return out


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
