"""Parity checks: library (CUDA on the GPU box / host-emulation harness here) vs the oracle.
Each function takes a `Library`.  Tolerances are written next to each comparison; all arithmetic
is FP64 on both sides, the bar from BASELINE.json is factor RMSE <= 1e-5."""
import numpy as np

from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel
import dynamic_factor_models_b200 as D

CFG = dict(nt_min_f=20, nt_min_fl=40, tol=1e-8, n_uarlag=4, n_factorlag=4)   # Stock_Watson.ipynb:245-251


def sign_align(F, Fref):
    s = np.sign(np.nansum(F * Fref, axis=0)); s[s == 0] = 1
    return F * s, s


def rmse(a, b):
    d = (a - b)[~np.isnan(a - b)]
    return float(np.sqrt(np.mean(d ** 2)))


def ref_model(data, incl, r, i0=3, i1=224):
    return R.DFMModel(data, incl, CFG["nt_min_f"], CFG["nt_min_fl"], i0, i1, 0, r, CFG["tol"], CFG["n_uarlag"], CFG["n_factorlag"])


def gpu_model(data, incl, r, i0=3, i1=224):
    return D.DFMModel(data, incl, CFG["nt_min_f"], CFG["nt_min_fl"], i0, i1, 0, r, CFG["tol"], CFG["n_uarlag"], CFG["n_factorlag"])


def check_standardize(lib, rng=None):
    X, _ = simulate_panel(17, 3, 41, rep=1, missing_frac=0.1, standardize=False)
    xs, sd = R.standardize_data(X)
    gxs, gmu, gsd = lib.standardize(X)
    np.testing.assert_allclose(gsd, sd, rtol=1e-13)
    np.testing.assert_allclose(gxs, xs, rtol=1e-12, atol=1e-13)
    assert (np.isnan(gxs) == np.isnan(xs)).all()


def separated_panel(T, N, decay=0.93, rep=2):
    """T x N panel U diag(s) V' with s_j = decay^j and a V whose column j has its largest entry in row j, well above the
    others: distinct singular values and an unambiguous sign rule (see pca_sign_rule)."""
    rng = np.random.default_rng(rep)
    n = min(T, N)
    U, _ = np.linalg.qr(rng.standard_normal((T, n)))
    M = 0.1 * rng.standard_normal((N, n))
    M[np.arange(n), np.arange(n)] += rng.choice([-1.0, 1.0], n)
    V, _ = np.linalg.qr(M)
    return (U * decay ** np.arange(n)) @ V.T


def pca_sign_rule(X, r):
    """X V_r with numpy's SVD and the library's documented sign rule: the entry of largest magnitude of each right singular
    vector is positive.  Asserts that the top r + 1 singular values and each column's two largest |entries| are apart, so
    that the rule and the columns are well defined."""
    _, s, Vt = np.linalg.svd(X, full_matrices=False)
    s = np.append(s, 0.0)
    assert (s[:r] > 1.01 * s[1:r + 1]).all(), "singular values too close"
    V = Vt[:r].T.copy()
    a = np.sort(np.abs(V), axis=0)
    assert (a[-1] - a[-2] > 1e-4).all(), "largest entries too close"      # (the vectors have unit norm)
    j = np.argmax(np.abs(V), axis=0)
    V *= np.sign(V[j, np.arange(r)])
    return X @ V


def check_pca(lib, T=60, N=25, r=4, sizes=None, sign_rule=False, batch=1):
    """sign_rule: raw scores of separated_panel data against pca_sign_rule, no sign alignment; batch > 1: also a batched
    call against one call per panel."""
    for (t, n) in (sizes or ((T, N), (N, T))):          # both Gram modes (X'X and XX')
        if not sign_rule:
            X, _ = simulate_panel(n, r, t, rep=2)
            ref = R.pca_score(X, r)
            got = lib.pca_score(X, r)
            got, _ = sign_align(got, ref)
            assert rmse(got, ref) < 1e-10 * max(1.0, np.abs(ref).max())
            continue
        Xb = np.stack([separated_panel(t, n, rep=2 + b) for b in range(batch)])
        got = lib.pca_score(Xb, r)
        for b in range(batch):
            ref = pca_sign_rule(Xb[b], r)
            assert np.abs(got[b] - ref).max() < 1e-9 * np.abs(ref).max(), np.abs(got[b] - ref).max()
            if batch > 1:
                np.testing.assert_allclose(got[b], lib.pca_score(Xb[b], r), rtol=1e-13, atol=1e-13 * np.abs(ref).max())


def check_estimate_factor_c1(lib, panels, r=8):
    """C1: hom_fac_1 'All' panel, T=222 x N=139, r=8 (Stock_Watson.ipynb:1266-1272)."""
    m = ref_model(panels["all_bpdata"], panels["all_inclcode"], r); R.estimate_factor(m)
    g = gpu_model(panels["all_bpdata"], panels["all_inclcode"], r); D.estimate_factor(g, lib=lib)
    assert g.fes.nobs == m.fes.nobs
    np.testing.assert_allclose(g.fes.tss, m.fes.tss, rtol=1e-12)
    assert g.fes.iters == m.fes.iters, (g.fes.iters, m.fes.iters)
    np.testing.assert_allclose(g.fes.ssr, m.fes.ssr, rtol=1e-9)
    F, s = sign_align(g.factor[2:224], m.factor[2:224])
    e = rmse(F, m.factor[2:224])
    assert e < 1e-7, e                       # north-star bar: 1e-5
    lam = g.lambda_est * s
    assert (np.isnan(lam) == np.isnan(m.lambda_est)).all()
    assert rmse(lam, m.lambda_est) < 1e-7
    np.testing.assert_allclose(g.fes.R2, m.fes.R2, rtol=1e-7, atol=1e-9)
    # golden Table 2B row r=8 (Stock_Watson.ipynb:626): trace R2 0.501, BN-ICp2 -0.223
    if r == 8:
        assert abs((1 - g.fes.ssr / g.fes.tss) - 0.501) < 6e-4
        assert abs(D.bai_ng_criterion(g) - (-0.223)) < 6e-4
    return e


def check_estimate_factor_same_init(lib, N=30, r=3, T=80, miss=0.08, iters=(1, 7), short_series=True, constr=None,
                                    pca_start=False):
    """Same starting factors on both sides -> no sign ambiguity, tight tolerance; fixed sweeps.  miss = 0 with
    short_series=False: a balanced panel.  constr = (index, R, r) rows of a :factor constraint (r unstandardized).
    pca_start: the library starts from its own PCA, the oracle from pca_sign_rule (the sign rule the library documents)."""
    X, _ = simulate_panel(N, r, T, rep=4, standardize=False)
    rng = np.random.default_rng(4)
    hole = rng.uniform(size=(T, N // 2)) < 2 * miss                 # missing data only in half of the columns
    X[:, :N // 2][hole] = np.nan
    if short_series:
        X[:, 0] = np.nan; X[:15, 0] = 1.0 + np.arange(15) * 0.1    # a series with < nt_min obs
    m = R.DFMModel(X, np.ones(N, int), 20, 40, 1, T, 0, r, 1e-8, 4, 2)
    xs, _ = R.standardize_data(X)
    f0 = (pca_sign_rule if pca_start else R.pca_score)(R.drop_missing_col(xs)[0], r)
    lc = None
    if constr is not None:
        lc = R.LambdaConstraint(np.asarray(constr[0]), np.asarray(constr[1], float), np.asarray(constr[2], float),
                                np.zeros(len(constr[0])))
    for max_iter in iters:
        R.estimate_factor(m, max_iter=max_iter, f_init=f0, lam_constr=lc)
        out = lib.estimate_factor(X, r, nt_min=20, tol=1e-8, max_iter=max_iter, F_init=None if pca_start else f0, constr=constr)
        assert out["stats"]["iters"] == m.fes.iters
        np.testing.assert_allclose(out["F"], m.factor, rtol=1e-9, atol=1e-10)
        np.testing.assert_allclose(out["Lam"], m.lambda_est, rtol=1e-9, atol=1e-10)
        if short_series:
            assert np.isnan(out["Lam"][0]).all()
        np.testing.assert_allclose(out["stats"]["ssr"], m.fes.ssr, rtol=1e-11)
        np.testing.assert_allclose(out["R2"], m.fes.R2, rtol=1e-8, atol=1e-10)
        if constr is not None:                                         # the restriction holds (standardized units)
            for q, i in enumerate(constr[0]):
                np.testing.assert_allclose(np.asarray(constr[1])[q] @ out["Lam"][i], constr[2][q] / out["xstd"][i], rtol=1e-9, atol=1e-11)


def check_constraint(lib, panels):
    """Figure-7 configuration (Stock_Watson.ipynb:1326-1344): oil-price loadings restricted."""
    data, incl = panels["all_bpdata"], panels["all_inclcode"]
    names = [str(s) for s in panels["all_names"]]
    calds = [tuple(x) for x in panels["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    r = 8
    varnames = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]
    Rm = np.eye(r); rv = np.r_[1.0, np.zeros(r - 1)]
    used = [n for n, c in zip(names, incl) if c == 1]
    m = ref_model(data, incl, r, i0, i1)
    cf = R.construct_constraint(varnames, used, Rm, rv); cfl = R.construct_constraint(varnames, names, Rm, rv)
    R.estimate(m, lam_constr_f=cf, lam_constr_fl=cfl)
    g = gpu_model(data, incl, r, i0, i1)
    gf = D.construct_constraint(varnames, used, Rm, rv); gfl = D.construct_constraint(varnames, names, Rm, rv)
    # a constrained fit is NOT invariant to the (LAPACK-arbitrary) signs of the PCA start, so both
    # sides start from the oracle's PCA scores
    xs, _ = R.standardize_data(data[:, incl == 1][i0 - 1:i1])
    f0 = R.pca_score(R.drop_missing_col(xs)[0], r)
    D.estimate_factor(g, lam_constr=gf, lib=lib, f_init=f0)
    D.estimate_factor_loading(g, lam_constr=gfl, lib=lib)
    D.estimate_var(g.factor_var_model, lib=lib)
    assert g.fes.iters == m.fes.iters
    F, s = sign_align(g.factor[i0 - 1:i1], m.factor[i0 - 1:i1])
    assert rmse(F, m.factor[i0 - 1:i1]) < 1e-7
    assert rmse(g.lambda_ * s, m.lambda_) < 1e-7
    np.testing.assert_allclose(g.r2, m.r2, rtol=1e-6, atol=1e-8)
    for nme in varnames:                       # the restriction holds on the constrained series
        j = names.index(nme)
        if not np.isnan(g.lambda_[j, 0]):
            np.testing.assert_allclose(g.lambda_[j] * s, rv, atol=1e-9)


def check_full_nonparametric_c1(lib, panels, r=8):
    """estimate!(m, NonParametric()) end to end: factors, loadings, uar, VAR, companion, IRF."""
    m = ref_model(panels["all_bpdata"], panels["all_inclcode"], r); R.estimate(m)
    g = gpu_model(panels["all_bpdata"], panels["all_inclcode"], r); D.estimate(g, lib=lib)
    F, s = sign_align(g.factor[2:224], m.factor[2:224])
    assert rmse(F, m.factor[2:224]) < 1e-7
    assert (np.isnan(g.lambda_) == np.isnan(m.lambda_)).all()
    assert rmse(g.lambda_ * s, m.lambda_) < 1e-7
    np.testing.assert_allclose(g.r2, m.r2, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(g.uar_coef, m.uar_coef, rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(g.uar_ser, m.uar_ser, rtol=1e-7, atol=1e-10)
    # VAR pieces transform with the sign matrix S = diag(s): compare sign-invariant forms
    gv, mv = g.factor_var_model, m.factor_var_model
    S4 = np.tile(s, mv.nlag)
    np.testing.assert_allclose(gv.M * S4[:, None] * S4[None, :], mv.M, rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(gv.seps * s[:, None] * s[None, :], mv.seps, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(gv.betahat[1:] * S4[:, None] * s[None, :], mv.betahat[1:], rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(gv.resid[6:224] * s, mv.resid[6:224], rtol=1e-6, atol=1e-8)
    assert np.isnan(gv.resid[:6]).all()
    np.testing.assert_allclose(gv.G @ gv.G.T * S4[:, None] * S4[None, :], mv.G @ mv.G.T, rtol=1e-6, atol=1e-9)
    # table 3 golden (Stock_Watson.ipynb:991-1017), column r=8, visible rows
    return g, m, s


def check_var_irf(lib, r=3, p=2, T=120, withconst=True, shocks=(0, 2), H=12, batch=1, rtol=1e-9):
    """withconst=False: M, Q, G against a companion form built here (the oracle's fill_matrices assumes a constant).
    batch > 1: the IRF of a batch of that many perturbed models against one oracle IRF per model."""
    _, tr = simulate_panel(10, r, T, rep=6)
    Fm = np.full((T + 3, r), np.nan); Fm[3:] = tr["F"]
    v = R.VARModel(Fm, p, withconst, 4, T + 3); R.estimate_var(v, compute_matrices=withconst)
    out = lib.estimate_var(Fm[3:], p, withconst)
    np.testing.assert_allclose(out["betahat"], v.betahat, rtol=rtol, atol=1e-11)
    np.testing.assert_allclose(out["seps"], v.seps, rtol=rtol)
    if not withconst:
        k = r * p
        v.M = np.zeros((k, k)); v.M[:r] = v.betahat.T; v.M[r:, :k - r] = np.eye(k - r)
        v.Q = np.zeros((r, k)); v.Q[:, :r] = np.eye(r)
        v.G = np.zeros((k, r)); v.G[:r] = np.linalg.cholesky(v.seps)
    np.testing.assert_allclose(out["M"], v.M, rtol=rtol, atol=1e-11)
    np.testing.assert_allclose(out["Q"], v.Q, atol=0)
    np.testing.assert_allclose(out["G"], v.G, rtol=rtol, atol=1e-12)
    np.testing.assert_allclose(out["resid"][p:], v.resid[3 + p:], rtol=1e-8, atol=1e-10)
    assert np.isnan(out["resid"][:p]).all()
    irf_ref = R.impulse_response(v, list(shocks), H)
    irf = lib.irf(out["M"], out["Q"], out["G"], H, list(shocks))
    np.testing.assert_allclose(irf, irf_ref, rtol=1e-9, atol=1e-12)
    if batch > 1:
        scale = 1.0 - 0.1 * np.arange(batch)                           # damped copies: a different IRF per model
        Mb = np.stack([out["M"] * s for s in scale]); Qb = np.stack([out["Q"]] * batch); Gb = np.stack([out["G"] * (1 + s) for s in scale])
        got = lib.irf(Mb, Qb, Gb, H, list(shocks))
        for b in range(batch):
            vb = R.VARModel(Fm, p, withconst, 4, T + 3); vb.M, vb.Q, vb.G = Mb[b], Qb[b], Gb[b]
            np.testing.assert_allclose(got[b], R.impulse_response(vb, list(shocks), H), rtol=1e-9, atol=1e-12)


def check_loading(lib, N=12, r=3, T=120, n_uarlag=4, nt_min=40, F_holes=(), edge_series=False, exact=False, batch=1):
    """estimate_loading (loadings, R2, idiosyncratic AR, constant, residuals) vs oracle.estimate_factor_loading and a
    numpy OLS of each series on [F 1] over the rows where the series and every factor are observed.  F_holes: rows of F
    set missing; edge_series: series 1 with exactly nt_min usable rows, series 2 with nt_min - 1; exact: series 3 an exact
    linear combination of the factors (R2 >= 0.9999: zero AR coefficients, ser 0).  batch > 1: that many panels in one
    call, each also against a one-panel call."""
    outs, Xs, Fs = [], [], []
    for b in range(batch):
        X, tr = simulate_panel(N, r, T, rep=3 + b, standardize=False)
        F = tr["F"].copy()
        F[list(F_holes)] = np.nan
        X[:10, 2 % N] = np.nan
        use = ~np.isnan(F).any(axis=1)
        if edge_series:
            for i, n_use in ((1, nt_min), (2, nt_min - 1)):
                rows = np.flatnonzero(use & ~np.isnan(X[:, i]))
                X[rows[n_use:], i] = np.nan
        if exact:
            X[:, 3] = 0.5 + F @ (1.0 + np.arange(r)) / r
        Xs.append(X); Fs.append(F)
    got = lib.estimate_loading(np.stack(Xs), np.stack(Fs), nt_min=nt_min, n_uarlag=n_uarlag) if batch > 1 else \
        lib.estimate_loading(Xs[0], Fs[0], nt_min=nt_min, n_uarlag=n_uarlag)
    for b in range(batch):
        X, F = Xs[b], Fs[b]
        g = {k: (v[b] if batch > 1 else v) for k, v in got.items()}
        if batch > 1:
            one = lib.estimate_loading(X, F, nt_min=nt_min, n_uarlag=n_uarlag)
            for k in ("lam", "r2", "uar_coef", "uar_ser", "constant", "resid"):
                np.testing.assert_allclose(g[k], one[k], rtol=1e-13, atol=1e-14, err_msg=k)
        assert g["status"] == 0
        m = R.DFMModel(X, np.ones(N, int), 20, nt_min, 1, T, 0, r, 1e-8, n_uarlag, 2)
        m.factor[:] = F
        R.estimate_factor_loading(m)
        for k, ref, rt in (("lam", m.lambda_, 1e-9), ("r2", m.r2, 1e-9), ("uar_coef", m.uar_coef, 1e-8), ("uar_ser", m.uar_ser, 1e-8)):
            assert np.array_equal(np.isnan(g[k]), np.isnan(ref)), k
            np.testing.assert_allclose(g[k], ref, rtol=rt, atol=1e-10, err_msg=k)
        use = ~np.isnan(F).any(axis=1)
        for i in range(N):
            keep = use & ~np.isnan(X[:, i])
            if keep.sum() < nt_min:
                assert np.isnan(g["lam"][i]).all() and np.isnan(g["constant"][i]) and np.isnan(g["resid"][:, i]).all()
                continue
            Z = np.column_stack([F[keep], np.ones(keep.sum())])
            beta = np.linalg.lstsq(Z, X[keep, i], rcond=None)[0]
            np.testing.assert_allclose(g["constant"][i], beta[-1], rtol=1e-9, atol=1e-10)
            assert np.array_equal(np.isnan(g["resid"][:, i]), ~keep)
            np.testing.assert_allclose(g["resid"][keep, i], X[keep, i] - Z @ beta, rtol=1e-8, atol=1e-9)
        if edge_series:
            assert np.isfinite(g["lam"][1]).all() and np.isnan(g["lam"][2]).all()
        if exact:
            assert g["r2"][3] >= 0.9999 and (g["uar_coef"][3] == 0).all() and g["uar_ser"][3] == 0


def check_var_missing_rows(lib, r=3, p=2, T=120):
    """estimate_var! drops every row with a missing y_t or lag (ols_skipmissing Balanced, dfm_functions.ipynb:242-252,
    452): NaNs INSIDE [initperiod, lastperiod] must give the oracle's fit, NaN residuals on the dropped rows."""
    _, tr = simulate_panel(10, r, T, rep=8)
    Fm = tr["F"].copy()
    Fm[17, 1] = np.nan; Fm[60:62, :] = np.nan; Fm[T - 1, 0] = np.nan
    v = R.VARModel(Fm.copy(), p, True, 1, T); R.estimate_var(v)
    out = lib.estimate_var(Fm, p, True)
    np.testing.assert_allclose(out["betahat"], v.betahat, rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(out["seps"], v.seps, rtol=1e-9)
    np.testing.assert_allclose(out["G"], v.G, rtol=1e-9, atol=1e-12)
    assert np.array_equal(np.isnan(out["resid"]), np.isnan(v.resid))
    ok = ~np.isnan(v.resid)
    np.testing.assert_allclose(out["resid"][ok], v.resid[ok], rtol=1e-8, atol=1e-10)
    # batched call: a panel without enough complete rows comes back as NaN, the others are fitted
    Fb = np.stack([tr["F"], np.full_like(tr["F"], np.nan), Fm])
    ob = lib.estimate_var(Fb, p, True)
    assert np.isnan(ob["betahat"][1]).all() and np.isnan(ob["M"][1]).all()
    np.testing.assert_allclose(ob["betahat"][2], v.betahat, rtol=1e-9, atol=1e-11)
    assert np.isfinite(ob["betahat"][0]).all()


def ll_atol(X, per_cell):
    """Absolute log-likelihood bar per_cell * (observed cells of X).  The log-likelihood is a sum of one term of order one
    per observed cell; on a well-fitted panel with many factors those terms cancel to a total near zero, so a bar relative
    to |ll| alone would ask for more digits than the sum has."""
    return per_cell * float(np.count_nonzero(~np.isnan(X)))


def check_em(lib, N=24, r=3, T=70, p=1, miss=0.0, iters=6, path=0, rep=9, holes=(), ll_cell_tol=0.0):
    """E-step + M-step vs the spec oracle, same initial parameters, fixed iterations.  holes: (t0, t1, i) blocks X[t0:t1, i]
    set missing (the observation pattern then stays constant between block edges); ll_cell_tol: see ll_atol."""
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    for t0, t1, i in holes:
        X[t0:t1, i] = np.nan
    F0 = R.pca_score(np.nan_to_num(X), r)
    Lam, Rv, A, Q = K.init_from_factors(X, F0, p)
    compare_em_init(lib.em_init_from_factors(X, F0, p), (Lam, Rv, A, Q))
    ref = K.em_kalman(X, Lam, Rv, A, Q, p=p, max_iter=iters, tol=0.0)
    got = lib.em_kalman(X, Lam, Rv, A, Q, p=p, max_iter=iters, tol=0.0, path=path)
    assert got["status"] == 0 and got["iters"] == iters
    compare_em(got, ref, ll_atol(X, ll_cell_tol))


def compare_em_init(got, ref):
    """(Lam, R, A, Q) of em_init_from_factors vs oracle.kalman_em.init_from_factors."""
    gL, gR, gA, gQ = got
    Lam, Rv, A, Q = ref
    np.testing.assert_allclose(gL, Lam, rtol=1e-9, atol=1e-11); np.testing.assert_allclose(gR, Rv, rtol=1e-9)
    np.testing.assert_allclose(gA, A, rtol=1e-8, atol=1e-10); np.testing.assert_allclose(gQ, Q, rtol=1e-8, atol=1e-10)


def compare_em(got, ref, ll_abs=0.0):
    """One panel's em_kalman results vs oracle.kalman_em.em_kalman from the same start; ll_abs: absolute log-likelihood bar."""
    np.testing.assert_allclose(got["P0"], ref["P0"], rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=1e-10, atol=ll_abs)
    assert (np.diff(got["loglik"]) > -1e-8 * np.abs(got["loglik"][:-1])).all()      # EM invariant
    assert rmse(got["F"], ref["F"]) < 1e-8
    np.testing.assert_allclose(got["PF"], ref["PsF"], rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(got["Lam"], ref["Lam"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(got["R"], ref["R"], rtol=1e-7)
    np.testing.assert_allclose(got["A"], ref["A"], rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(got["Q"], ref["Q"], rtol=1e-6, atol=1e-8)


def check_em_convergence_rule(lib, path=0):
    X, _ = simulate_panel(20, 2, 60, rep=12)
    F0 = R.pca_score(X, 2)
    Lam, Rv, A, Q = K.init_from_factors(X, F0, 1)
    ref = K.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=200, tol=1e-5)
    got = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=200, tol=1e-5, path=path)
    assert got["iters"] == ref["iters"] and ref["iters"] < 200
    n = ref["iters"]
    np.testing.assert_allclose(got["loglik"][:n], ref["loglik"], rtol=1e-10)
    assert np.isnan(got["loglik"][n:]).all()
    assert rmse(got["F"], ref["F"]) < 1e-8


def check_em_batch(lib, B=3, N=16, r=2, T=40, p=1, path=0):
    """Batched call == the same panels one at a time (replication independence)."""
    Xb = np.stack([simulate_panel(N, r, T, rep=20 + b, missing_frac=0.05 * (b % 2))[0] for b in range(B)])
    inits = [K.init_from_factors(Xb[b], R.pca_score(np.nan_to_num(Xb[b]), r), p) for b in range(B)]
    Lam = np.stack([i[0] for i in inits]); Rv = np.stack([i[1] for i in inits])
    A = np.stack([i[2] for i in inits]); Q = np.stack([i[3] for i in inits])
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=p, max_iter=4, path=path)
    for b in range(B):
        one = lib.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=p, max_iter=4, path=path)
        np.testing.assert_allclose(got["F"][b], one["F"], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(got["loglik"][b], one["loglik"], rtol=1e-13)
        ref = K.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=p, max_iter=4)
        assert rmse(got["F"][b], ref["F"]) < 1e-8


def check_em_batch_balanced(lib, B=5, N=16, r=2, T=40, path=0, ll_cell_tol=0.0):
    Xb = np.stack([simulate_panel(N, r, T, rep=40 + b)[0] for b in range(B)])
    inits = [K.init_from_factors(Xb[b], R.pca_score(Xb[b], r), 1) for b in range(B)]
    Lam = np.stack([i[0] for i in inits]); Rv = np.stack([i[1] for i in inits])
    A = np.stack([i[2] for i in inits]); Q = np.stack([i[3] for i in inits])
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=4, path=path)
    for b in range(B):
        ref = K.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=1, max_iter=4)
        assert rmse(got["F"][b], ref["F"]) < 1e-8
        np.testing.assert_allclose(got["loglik"][b], ref["loglik"], rtol=1e-10, atol=ll_atol(Xb[b], ll_cell_tol))
        np.testing.assert_allclose(got["PF"][b], ref["PsF"], rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(got["Lam"][b], ref["Lam"], rtol=1e-7, atol=1e-9)


def check_als_balanced(lib, N=30, r=3, T=80, B=4, per_panel=False):
    """Balanced panels -> fused ALS kernel (one launch for all sweeps): vs the oracle, from a perturbed
    start so that several sweeps are needed; also PCA start, iteration cap and batch.  per_panel: the batched call also
    against one call per panel, and the panels must stop after different numbers of sweeps."""
    rng = np.random.default_rng(3)
    Xb = np.stack([simulate_panel(N, r, T, rep=60 + b, standardize=False)[0] * (1 + 0.3 * b) + b for b in range(B)])
    f0s = []
    for b in range(B):
        xs, _ = R.standardize_data(Xb[b])
        wide = 1 + 3 * b if per_panel else 1                             # per_panel: starts further off, panel by panel
        f0s.append(R.pca_score(xs, r) @ (np.eye(r) + 0.3 * wide * rng.standard_normal((r, r))) + 0.5 * wide * rng.standard_normal((T, r)))
    f0s = np.stack(f0s)
    for max_iter in (1, 4, 100000):
        got = lib.estimate_factor(Xb, r, nt_min=20, tol=1e-8, max_iter=max_iter, F_init=f0s)
        for b in range(B):
            m = R.DFMModel(Xb[b], np.ones(N, int), 20, 40, 1, T, 0, r, 1e-8, 4, 2)
            R.estimate_factor(m, max_iter=max_iter, f_init=f0s[b])
            assert got["stats"][b]["iters"] == m.fes.iters, (max_iter, b, got["stats"][b]["iters"], m.fes.iters)
            np.testing.assert_allclose(got["F"][b], m.factor, rtol=1e-8, atol=1e-9)
            np.testing.assert_allclose(got["Lam"][b], m.lambda_est, rtol=1e-8, atol=1e-9)
            np.testing.assert_allclose(got["stats"][b]["ssr"], m.fes.ssr, rtol=1e-9)
            np.testing.assert_allclose(got["stats"][b]["tss"], m.fes.tss, rtol=1e-12)
            np.testing.assert_allclose(got["R2"][b], m.fes.R2, rtol=1e-7, atol=1e-9)
            if per_panel:
                one = lib.estimate_factor(Xb[b], r, nt_min=20, tol=1e-8, max_iter=max_iter, F_init=f0s[b])
                assert one["stats"]["iters"] == got["stats"][b]["iters"]
                np.testing.assert_allclose(got["F"][b], one["F"], rtol=1e-12, atol=1e-13)
        if per_panel and max_iter == 100000:
            assert len({s["iters"] for s in got["stats"]}) > 1, [s["iters"] for s in got["stats"]]
    # PCA start (sign-aligned)
    got = lib.estimate_factor(Xb[0], r, nt_min=20, tol=1e-8)
    m = R.DFMModel(Xb[0], np.ones(N, int), 20, 40, 1, T, 0, r, 1e-8, 4, 2); R.estimate_factor(m)
    assert got["stats"]["iters"] == m.fes.iters
    F, _ = sign_align(got["F"], m.factor)
    assert rmse(F, m.factor) < 1e-8


def check_als_batch(lib, B=3, N=20, r=2, T=50):
    Xb = np.stack([simulate_panel(N, r, T, rep=30 + b, standardize=False)[0] for b in range(B)])
    Xb[:, 5:9, 3:8] = np.nan; Xb[1, 20:30, 0] = np.nan
    got = lib.estimate_factor(Xb, r, nt_min=10, tol=1e-8)
    for b in range(B):
        m = R.DFMModel(Xb[b], np.ones(N, int), 10, 10, 1, T, 0, r, 1e-8, 4, 2); R.estimate_factor(m)
        assert got["stats"][b]["iters"] == m.fes.iters
        F, _ = sign_align(got["F"][b], m.factor)
        assert rmse(F, m.factor) < 1e-8
        np.testing.assert_allclose(got["stats"][b]["ssr"], m.fes.ssr, rtol=1e-10)


def check_parametric_c1(lib, panels, iters=3):
    """C1 with VAR(4) state (k = 32) and 5.7% missing data: general path vs oracle."""
    m = ref_model(panels["all_bpdata"], panels["all_inclcode"], 8); R.estimate_factor(m, computeR2=False)
    Xs = m.xs.copy(); Xs[:, np.isnan(m.lambda_est[:, 0])] = np.nan
    F0 = m.factor[2:224]
    Lam, Rv, A, Q = K.init_from_factors(Xs, F0, 4)
    Lam[np.isnan(m.lambda_est[:, 0])] = np.nan
    ref = K.em_kalman(Xs, Lam, Rv, A, Q, p=4, max_iter=iters)
    got = lib.em_kalman(Xs, Lam, Rv, A, Q, p=4, max_iter=iters, path=1)
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=1e-9)
    assert rmse(got["F"], ref["F"]) < 1e-7
    np.testing.assert_allclose(got["A"], ref["A"], rtol=1e-5, atol=1e-7)


def check_nile_published(lib, path=0):
    """The product's filter / smoother on the published local-level example (Durbin & Koopman 2012, ch. 2; see
    tests/test_oracle_kalman_published.py): diffuse log-likelihood -632.54 at the published ML estimates."""
    import json
    import os
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nile_local_level.json")))
    y = np.array(g["nile"], float)[:, None]; pub = g["published"]; P1 = 1e7
    s2e, s2n = pub["sigma2_eps"], pub["sigma2_eta"]
    out = lib.em_kalman(y, np.ones((1, 1)), np.array([s2e]), np.ones((1, 1)), np.array([[s2n]]), p=1, P0=np.array([[P1]]), max_iter=1,
                        path=path)
    first = -0.5 * np.log(2 * np.pi) - 0.5 * np.log(P1 + s2e) - 0.5 * y[0, 0] ** 2 / (P1 + s2e)
    assert abs((out["loglik"][0] - first) - pub["loglik_diffuse"]) < 0.01
    es = K.e_step(y, np.ones((1, 1)), np.array([s2e]), np.ones((1, 1)), np.array([[s2n]]), np.array([[P1]]), 1)
    np.testing.assert_allclose(out["F"][:, 0], es["zs"][:, 0], rtol=1e-9)
    np.testing.assert_allclose(out["loglik"][0], es["loglik"], rtol=1e-11)


def check_simulate_panels(lib, N=24, r=3, T=70, B=3, rep0=5):
    """Device generator (K9) vs its numpy restatement: same counter-based Philox stream, same DGP; panels are a function
    of the replication id only (any batch split gives the same bits)."""
    from oracle import dgp
    X, F = lib.simulate_panels(rep0, B, N, r, T, dgp.SEED, want_F=True)
    for b in range(B):
        Xr, tr = dgp.simulate_panel_device_stream(N, r, T, rep=rep0 + b)
        np.testing.assert_allclose(F[b], tr["F"], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(X[b], Xr, rtol=1e-10, atol=1e-12)
    assert abs(X.mean(axis=1)).max() < 1e-12 and abs(X.std(axis=1) - 1).max() < 1e-12      # standardised columns
    X2 = lib.simulate_panels(rep0 + 1, 1, N, r, T, dgp.SEED)
    assert np.array_equal(X2[0], X[1])                                                     # independent of the batch split
    assert not np.allclose(lib.simulate_panels(rep0, 1, N, r, T, dgp.SEED + 1)[0], X[0])


def check_simulate_panels_statistics(lib, N=60, r=4, T=400, B=8):
    """The device DGP has the frozen distributions: factor AR(1) coefficients in [.2,.8], unit innovation variance,
    and a dominant r-factor structure (moments over B panels)."""
    from oracle import dgp
    X, F = lib.simulate_panels(100, B, N, r, T, dgp.SEED, want_F=True)
    a_hat = np.array([[np.dot(F[b, 1:, j], F[b, :-1, j]) / np.dot(F[b, :-1, j], F[b, :-1, j]) for j in range(r)] for b in range(B)])
    assert a_hat.min() > 0.05 and a_hat.max() < 0.92
    innov = F[:, 1:, :] - a_hat[:, None, :] * F[:, :-1, :]
    assert abs(innov.var() - 1.0) < 0.05
    # common component share: var(Lam f) / var(x) with E|lam|^2 = r, var f_j = 1/(1-a^2) >= 1, s2 ~ 1  ->  well above 1/2
    ev = np.linalg.eigvalsh(np.corrcoef(X[0].T))[::-1]
    assert ev[:r].sum() / N > 0.5 and ev[r] < ev[r - 1]


def check_bootstrap_panels(lib, panels, B=2):
    """Device residual bootstrap (C4) vs its numpy restatement on the fitted C1 model."""
    from oracle import dgp
    m = ref_model(panels["all_bpdata"], panels["all_inclcode"], 4)
    R.estimate(m)
    i0, i1 = m.initperiod, m.lastperiod
    v = m.factor_var_model; p = v.nlag
    F0 = m.factor[i0 - 1:i1]; resid = v.resid[i0 - 1:i1][p:]
    data = m.data[i0 - 1:i1]
    X = lib.bootstrap_panels(F0, resid, v.betahat, m.lambda_, m.uar_coef, m.uar_ser, data, 7, B, dgp.SEED, burn=50)
    for b in range(B):
        Xr = dgp.bootstrap_panel_device_stream(F0, resid, v.betahat, m.lambda_, m.uar_coef, m.uar_ser, data, 7 + b, burn=50)
        assert np.array_equal(np.isnan(X[b]), np.isnan(Xr))
        ok = ~np.isnan(Xr)
        np.testing.assert_allclose(X[b][ok], Xr[ok], rtol=1e-9, atol=1e-10)
    assert np.array_equal(np.isnan(X[0]) | np.isnan(data), np.isnan(X[0]))                 # original missing pattern re-imposed


def check_percentiles(lib, n=37, d=11, q=(5, 16, 50, 84, 95, 0, 100), odd_columns=False):
    """odd_columns: column 0 all NaN (result NaN) and column d - 1 with one finite record (every percentile is that record)."""
    import warnings
    rng = np.random.default_rng(3)
    recs = rng.standard_normal((n, d)); recs[5 % n] = np.nan; recs[20 % n] = np.nan      # two failed replications
    if odd_columns:
        recs[:, 0] = np.nan
        recs[:, d - 1] = np.nan; recs[n // 2, d - 1] = 1.25
    q = list(q)
    got = lib.percentiles(recs, q)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)               # (the all-NaN column)
        ref = np.nanpercentile(recs, q, axis=0)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-14)
    got1 = lib.percentiles(recs[:1], [50.0])
    np.testing.assert_allclose(got1[0], recs[0])


def check_em_block_missing(lib, path=1):
    """Missing data in BLOCKS (series that start late / end early / have a hole): the observation pattern is constant
    over long stretches, so the general path freezes its covariance recursion between pattern changes (src[t] logic of
    k_em_filter_smooth) -- results must still equal the oracle's period-by-period recursion."""
    X, _ = simulate_panel(20, 2, 260, rep=3)
    X[:60, 3] = np.nan; X[200:, 7] = np.nan; X[100:140, 11] = np.nan
    F0 = R.pca_score(np.nan_to_num(X), 2)
    Lam, Rv, A, Q = K.init_from_factors(X, F0, 2)
    ref = K.em_kalman(X, Lam, Rv, A, Q, p=2, max_iter=4)
    got = lib.em_kalman(X, Lam, Rv, A, Q, p=2, max_iter=4, path=path)
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=1e-11)
    np.testing.assert_allclose(got["F"], ref["F"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(got["Lam"], ref["Lam"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(got["A"], ref["A"], rtol=1e-8, atol=1e-10)


def check_instability(lib, panels, r=4, series=None, q=6, ccut=0.15, qlr0=False, data=None, factor=None, lastpre=104,
                      min_obs=80):
    """f4: Chow / QLR statistics (HAC) on the hom_fac_1 panel vs the oracle (pinned on the notebook's Table 4(a)).
    data / factor: another panel and its factors instead (no estimation); qlr0: also the q = 0 QLR, against the oracle's
    QLR with q = 0 over the same break rows."""
    import dynamic_factor_models_b200 as D
    if data is None:
        data, incl = panels["all_bpdata"], panels["all_inclcode"]
        mo = R.DFMModel(data, incl, 20, 40, 3, 224, 0, r, 1e-8, 4, 4)
        R.estimate_factor(mo, computeR2=False)
        factor = mo.factor
    cols = np.arange(data.shape[1]) if series is None else np.asarray(series)
    sub = type("M", (), {})(); sub.data = data[:, cols]; sub.factor = factor; sub.ns = len(cols)
    chow_o, qlr_o = R.instability_tests(sub, lastpre, q=q, ccut=ccut, min_obs=min_obs)
    mg = type("M", (), {})(); mg.data = data[:, cols]; mg.factor = factor   # same regressors: the test isolates the instability kernels
    got = D.instability_tests(mg, lastpre, q=q, ccut=ccut, min_obs=min_obs, lib=lib, want_q0=qlr0)
    chow_g, qlr_g = got[:2]
    assert np.array_equal(np.isnan(chow_o), np.isnan(chow_g)) and np.array_equal(np.isnan(qlr_o), np.isnan(qlr_g))
    ok = ~np.isnan(chow_o)
    assert ok.sum() >= 1
    np.testing.assert_allclose(chow_g[ok], chow_o[ok], rtol=1e-8)
    np.testing.assert_allclose(qlr_g[ok], qlr_o[ok], rtol=1e-8)
    if qlr0:
        _, qlr0_o = R.instability_tests(sub, lastpre, q=0, ccut=ccut, min_obs=min_obs)
        assert np.array_equal(np.isnan(qlr0_o), np.isnan(got[2]))
        np.testing.assert_allclose(got[2][ok], qlr0_o[ok], rtol=1e-8)


def check_fit_correlation(lib, panels, r=4, data=None, factors=None):
    """f4, lower half of Table 4(a): cor(yhat_full, yhat_pre/post) per series vs the oracle (same factors on both sides).
    data / factors: another panel and its (full, pre, post) factors instead (no estimation)."""
    if data is None:
        data, incl = panels["all_bpdata"], panels["all_inclcode"]
        ms = [R.DFMModel(data, incl, 20, 40, i0, i1, 0, r, 1e-8, 4, 4) for i0, i1 in ((3, 224), (3, 104), (105, 224))]
        for m in ms:
            R.estimate_factor(m, computeR2=False)
    else:
        ms = [type("M", (), dict(data=data, factor=f, ns=data.shape[1]))() for f in factors]
    for alt in ms[1:]:
        ref = R.fitted_value_correlations(ms[0], alt, 104)
        got = D.fitted_value_correlations(ms[0], alt, 104, lib=lib)
        assert np.array_equal(np.isnan(ref), np.isnan(got))
        ok = ~np.isnan(ref)
        np.testing.assert_allclose(got[ok], ref[ok], rtol=1e-9, atol=1e-11)


def check_cluster_sizes(lib, N=160, r=12, T=700):
    """General path, few panels: the thread-block cluster split of the frozen runs (8 / 2 CTAs per panel) gives the result of the
    single-CTA launch (different summation order of the tile partials only).  (The emulation build has no clusters.)"""
    import os
    X, _ = simulate_panel(N, r, T, rep=5)
    m = R.DFMModel(X, np.ones(N, int), 20, 40, 1, T, 0, r, 1e-8, 4, 1)
    R.estimate_factor(m, max_iter=2, computeR2=False)
    Lam, Rv, A, Q = K.init_from_factors(X, m.factor, 1)
    outs = {}
    for nc in ("1", "2", "8"):
        os.environ["DFM_CLUSTER"] = nc
        try:
            outs[nc] = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=4, path=1, want_PF=False)
        finally:
            del os.environ["DFM_CLUSTER"]
    for nc in ("2", "8"):
        np.testing.assert_allclose(outs[nc]["loglik"], outs["1"]["loglik"], rtol=1e-12)
        np.testing.assert_allclose(outs[nc]["F"], outs["1"]["F"], rtol=1e-9, atol=1e-11)
        np.testing.assert_allclose(outs[nc]["Lam"], outs["1"]["Lam"], rtol=1e-9, atol=1e-11)


def check_instability_edges(lib):
    """f4 edge cases: a series with too few observations on one side of the break -> NaN (as the notebook's rule), an
    all-missing series -> NaN, bad arguments -> status 1 (no exception from the kernel side, DFMError from the binding)."""
    rng = np.random.default_rng(3)
    T, r = 180, 3
    F = rng.standard_normal((T, r)); F[:4] = np.nan                         # factor rows outside the estimation window
    Y = F @ rng.standard_normal((r, 4)) + 0.5 * rng.standard_normal((T, 4))
    Y[np.isnan(Y)] = np.nan
    Y[:, 1] = np.nan                                                         # all missing
    Y[:70, 2] = np.nan                                                       # 20 observations before the break row 90: < 80
    out = lib.instability(Y, F, 90, q=4, ccut=0.15, min_obs=80)
    assert np.isfinite(out["chow"][0]) and np.isfinite(out["qlr"][0]) and out["qlr"][0] >= out["chow"][0] * (1 - 1e-12)
    assert np.isnan(out["chow"][1]) and np.isnan(out["qlr"][1]) and np.isnan(out["chow"][2])
    assert np.isfinite(out["chow"][3])
    m = type("M", (), {})(); m.data = Y; m.factor = F; m.ns = 4
    chow_o, qlr_o = R.instability_tests(m, 90, q=4)
    ok = ~np.isnan(chow_o)
    np.testing.assert_allclose(out["chow"][ok], chow_o[ok], rtol=1e-8); np.testing.assert_allclose(out["qlr"][ok], qlr_o[ok], rtol=1e-8)
    for bad in (dict(T_break=0), dict(T_break=T), dict(ccut=0.6), dict(q=9)):
        kw = dict(T_break=90, q=4, ccut=0.15); kw.update(bad)
        try:
            lib.instability(Y, F, kw["T_break"], q=kw["q"], ccut=kw["ccut"])
            raise AssertionError("bad argument accepted: %r" % (bad,))
        except D.DFMError as e:
            assert e.code == 1
