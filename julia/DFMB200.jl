# DFMB200.jl -- Julia-side binding a maintainer of QuantEcon/dynamic_factor_models would add to make
# the B200 library a drop-in for the hot path.  UNTESTED HERE (no Julia in the build image); it is
# deliberately thin: every function converts `Union{Missing,Float64}` <-> NaN, `ccall`s one entry
# point of include/dfm_b200.h and writes the results back into the reference's own structs
# (`DFMModel`, `VARModel`, `FactorEstimateStats` of dfm_functions.ipynb:43-111).
#
#   include("readin_functions.jl"); @nbinclude("dfm_functions.ipynb"); include("DFMB200.jl")
#   using .DFMB200
#   DFMB200.estimate_factor!(dfmm)                    # replaces estimate_factor!  (:328-382)
#   DFMB200.estimate!(dfmm, NonParametric())          # replaces estimate!         (:530-543)
#   DFMB200.estimate!(dfmm, Parametric())             # fills the empty slot of    :23
module DFMB200

const LIB = get(ENV, "DFM_B200_LIB", joinpath(@__DIR__, "..", "dynamic_factor_models_b200", "lib", "libdfm_b200.so"))
const MEM_HOST = Cint(0)
const LAST_ALS = Ref{Any}((iters = 0, status = 0, lambda = zeros(0, 0)))   # stats of the last estimate_factor! call

struct FactorOpts
    T::Cint; N::Cint; r::Cint; nt_min::Cint
    tol::Cdouble; max_iter::Clonglong
    compute_r2::Cint; n_constr::Cint
    constr_index::Ptr{Cint}; constr_R::Ptr{Cdouble}; constr_r::Ptr{Cdouble}
    batch::Cint; mem::Cint
end
struct FactorStats
    ssr::Cdouble; tss::Cdouble; nobs::Clonglong; iters::Cint; status::Cint
end
struct LoadingOpts
    T::Cint; ns::Cint; r::Cint; nt_min::Cint; n_uarlag::Cint
    n_constr::Cint; constr_index::Ptr{Cint}; constr_R::Ptr{Cdouble}; constr_r::Ptr{Cdouble}
    batch::Cint; mem::Cint
end
struct EmOpts
    T::Cint; N::Cint; r::Cint; p::Cint; max_iter::Cint; tol::Cdouble; batch::Cint; mem::Cint; path::Cint
end
struct EmInit; Lam::Ptr{Cdouble}; R::Ptr{Cdouble}; A::Ptr{Cdouble}; Q::Ptr{Cdouble}; P0::Ptr{Cdouble}; end
struct EmOut
    Lam::Ptr{Cdouble}; R::Ptr{Cdouble}; A::Ptr{Cdouble}; Q::Ptr{Cdouble}; P0::Ptr{Cdouble}
    F::Ptr{Cdouble}; PF::Ptr{Cdouble}; loglik::Ptr{Cdouble}; iters::Ptr{Cint}; status::Ptr{Cint}
end
struct LamConstr; n_constr::Cint; index::Ptr{Cint}; H::Ptr{Cdouble}; h::Ptr{Cdouble}; end

const handle = Ref{Ptr{Cvoid}}(C_NULL)
function gethandle(device::Integer = 0)
    if handle[] == C_NULL
        rc = ccall((:dfm_create, LIB), Cint, (Cint, Ref{Ptr{Cvoid}}), device, handle)
        rc == 0 || error("dfm_create failed with status $rc (a CUDA device is required; there is no CPU fallback)")
    end
    return handle[]
end
check(rc, what) = rc == 0 || error("$what: status $rc: " *
    unsafe_string(ccall((:dfm_last_error, LIB), Cstring, (Ptr{Cvoid},), handle[])))

tonan(A) = Float64[ismissing(x) ? NaN : Float64(x) for x in A]           # missing -> NaN, column-major kept
frommissing(A) = Union{Missing,Float64}[isnan(x) ? missing : x for x in A]

"""Replaces `estimate_factor!(m, max_iter, computeR2; lam_constr)` (dfm_functions.ipynb:328-382)."""
function estimate_factor!(m, max_iter::Integer = 100000000, computeR2::Bool = true; lam_constr = nothing)
    h = gethandle()
    X = tonan(m.data[m.initperiod:m.lastperiod, m.inclcode .== 1])
    T, N = size(X); r = m.nfac_u
    F = Matrix{Float64}(undef, T, r); Lam = Matrix{Float64}(undef, N, r); R2 = fill(NaN, N)
    stats = Ref(FactorStats(0, 0, 0, 0, 0))
    nc = lam_constr === nothing ? 0 : length(lam_constr.indices)
    idx = nc == 0 ? Cint[] : Cint.(lam_constr.indices .- 1)
    cR = nc == 0 ? Float64[] : Matrix{Float64}(lam_constr.R); cr = nc == 0 ? Float64[] : Vector{Float64}(lam_constr.r)
    GC.@preserve idx cR cr begin
        opts = Ref(FactorOpts(T, N, r, m.nt_min_factor_estimation, m.tol, max_iter, computeR2, nc,
                              pointer(idx), pointer(cR), pointer(cr), 1, MEM_HOST))
        check(ccall((:dfm_estimate_factor, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cdouble}, Ref{FactorOpts}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                     Ptr{Cdouble}, Ptr{Cdouble}, Ref{FactorStats}),
                    h, X, opts, C_NULL, F, Lam, R2, C_NULL, C_NULL, stats), "dfm_estimate_factor")
    end
    s = stats[]
    # status 2 / 3 = a period with fewer than r observations / a singular normal-equation system: the factors are NaN
    # (same rule as api.estimate_factor in the Python mirror); 4 = max_iter reached, which the reference accepts silently
    (s.status == 2 || s.status == 3) && error("dfm_estimate_factor: ALS failed (status $(s.status))")
    m.factor[m.initperiod:m.lastperiod, :] = F                              # :371
    m.fes.ssr, m.fes.tss, m.fes.nobs = s.ssr, s.tss, s.nobs                # :342-343, :366
    computeR2 && (m.fes.R2 .= frommissing(R2))
    LAST_ALS[] = (iters = Int(s.iters), status = Int(s.status), lambda = Lam)   # the reference discards these (:381)
    return nothing
end

"""Replaces `estimate_factor_loading!` (dfm_functions.ipynb:391-415)."""
function estimate_factor_loading!(m; lam_constr = nothing)
    h = gethandle()
    data = tonan(m.data[m.initperiod:m.lastperiod, :]); F = tonan(m.factor[m.initperiod:m.lastperiod, :])
    T, ns = size(data); r = m.nfac_t; L = m.n_uarlag
    lam = Matrix{Float64}(undef, ns, r); r2 = Vector{Float64}(undef, ns)
    uc = Matrix{Float64}(undef, ns, L); us = Vector{Float64}(undef, ns)
    nc = lam_constr === nothing ? 0 : length(lam_constr.indices)
    idx = nc == 0 ? Cint[] : Cint.(lam_constr.indices .- 1)
    cR = nc == 0 ? Float64[] : Matrix{Float64}(lam_constr.R); cr = nc == 0 ? Float64[] : Vector{Float64}(lam_constr.r)
    GC.@preserve idx cR cr begin
        opts = Ref(LoadingOpts(T, ns, r, m.nt_min_factorloading_estimation, L, nc, pointer(idx), pointer(cR), pointer(cr), 1, MEM_HOST))
        check(ccall((:dfm_estimate_loading, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Ref{LoadingOpts}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}),
                    h, data, F, opts, lam, r2, uc, us), "dfm_estimate_loading")
    end
    m.lambda .= lam; m.r2 .= frommissing(r2); m.uar_coef .= uc; m.uar_ser .= us
    return nothing
end

"""Replaces `estimate_var!` + `fill_matrices!` (dfm_functions.ipynb:444-492)."""
function estimate_var!(varm, compute_matrices::Bool = true)
    h = gethandle()
    F = tonan(varm.y[varm.initperiod:varm.lastperiod, :])
    T, r = size(F); p = varm.nlag; k = r * p; K = k + varm.withconst
    beta = Matrix{Float64}(undef, K, r); res = Matrix{Float64}(undef, T, r); seps = Matrix{Float64}(undef, r, r)
    M = Matrix{Float64}(undef, k, k); Q = Matrix{Float64}(undef, r, k); G = Matrix{Float64}(undef, k, r)
    check(ccall((:dfm_estimate_var, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                 Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}),
                h, F, T, r, p, varm.withconst, 1, MEM_HOST, beta, res, seps, M, Q, G), "dfm_estimate_var")
    varm.betahat .= beta; varm.seps .= seps
    varm.resid[varm.initperiod:varm.lastperiod, :] = frommissing(res)
    if compute_matrices; varm.M .= M; varm.Q .= Q; varm.G .= G; end
    return nothing
end

"""Replaces `impulse_response(varm, shock_ids, T)` (dfm_functions.ipynb:793-825)."""
function impulse_response(varm, shock_ids::AbstractVector, H::Integer)
    h = gethandle()
    k = size(varm.M, 1); r = size(varm.Q, 1); ids = Cint.(shock_ids .- 1)
    irf = Array{Float64,3}(undef, r, H, length(ids))
    check(ccall((:dfm_irf, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Ptr{Cint}, Cint, Cint, Ptr{Cdouble}),
                h, Float64.(varm.M), Float64.(varm.Q), Float64.(varm.G), k, r, H, length(ids), ids, 1, MEM_HOST, irf), "dfm_irf")
    return irf
end

"""Replaces the per-series loop of Table 4(a) (`compute_chow` / `compute_qlr` on `drop_missing_row([y X])`, Stock_Watson.ipynb):
Chow and QLR statistics (Bartlett HAC, `q` lags) of every series of `m.data` regressed on `m.factor`; `missing` where the
series has fewer than `min_obs` observations before or after row `lastpre`."""
function instability_tests(m, lastpre::Integer; q::Integer = 6, ccut::Real = 0.15, min_obs::Integer = 80)
    h = gethandle()
    data = tonan(m.data); F = tonan(m.factor)
    T, ns = size(data); r = size(F, 2)
    chow = Vector{Float64}(undef, ns); qlr = Vector{Float64}(undef, ns)
    check(ccall((:dfm_instability, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Cint, Cdouble, Cint, Cint,
                 Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cint}),
                h, data, F, T, ns, r, q, lastpre, Float64(ccut), min_obs, MEM_HOST, chow, qlr, C_NULL, C_NULL), "dfm_instability")
    return frommissing(chow), frommissing(qlr)
end

"""Second half of the Table 4(a) loop: `cor(yhat, yhat_alt)` per series, fitted values on `m.factor` and on `m_alt.factor`."""
function fitted_value_correlations(m, m_alt, lastpre::Integer; min_obs::Integer = 80)
    h = gethandle()
    data = tonan(m.data); F = tonan(m.factor); Fa = tonan(m_alt.factor)
    T, ns = size(data); r = size(F, 2)
    cor = Vector{Float64}(undef, ns)
    check(ccall((:dfm_fit_correlation, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Cdouble}, Ptr{Cint}),
                h, data, F, Fa, T, ns, r, lastpre, min_obs, MEM_HOST, cor, C_NULL), "dfm_fit_correlation")
    return frommissing(cor)
end

"""`estimate!(m, ::NonParametric)` (dfm_functions.ipynb:530-543) and the `Parametric` slot of :23.
`lam_constr_em` (Parametric only): a LambdaConstraint on the estimation series (as `lam_constr_f`) under which the state-space
EM runs (dfm_em_kalman_constrained); its `r` is divided by the block's standard deviations, as standardize_constraint! does."""
function estimate!(m, method = Main.NonParametric(); lam_constr_f = nothing, lam_constr_fl = nothing, lam_constr_em = nothing,
                   max_iter::Integer = 50, tol::Real = 1e-6)
    estimate_factor!(m, lam_constr = lam_constr_f)
    estimate_factor_loading!(m, lam_constr = lam_constr_fl)
    estimate_var!(m.factor_var_model)
    method isa Main.Parametric || return nothing
    # ---- state-space EM initialised by the non-parametric estimates
    h = gethandle()
    X = tonan(m.data[m.initperiod:m.lastperiod, m.inclcode .== 1]); T, N = size(X); r = m.nfac_t; p = m.n_factorlag; k = r * p
    Xs = similar(X); mu = Vector{Float64}(undef, N); sd = Vector{Float64}(undef, N)
    check(ccall((:dfm_standardize, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}),
                h, X, T, N, 1, MEM_HOST, Xs, mu, sd), "dfm_standardize")
    # series dropped by nt_min in the ALS step (NaN row of its Lambda) stay out of the state-space model as well --
    # the same masking as api._estimate_parametric, so that both host mirrors fit the same model
    lam_als = LAST_ALS[].lambda
    for i in 1:N
        isnan(lam_als[i, 1]) && (Xs[:, i] .= NaN)
    end
    F0 = tonan(m.factor[m.initperiod:m.lastperiod, :])
    Lam = Matrix{Float64}(undef, N, r); R = Vector{Float64}(undef, N); A = Matrix{Float64}(undef, r, k); Q = Matrix{Float64}(undef, r, r)
    check(ccall((:dfm_em_init_from_factors, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}),
                h, Xs, F0, T, N, r, p, 1, MEM_HOST, Lam, R, A, Q), "dfm_em_init_from_factors")
    F = Matrix{Float64}(undef, T, r); ll = fill(NaN, max_iter); it = Ref{Cint}(0); st = Ref{Cint}(0)
    nc = lam_constr_em === nothing ? 0 : length(lam_constr_em.indices)
    cidx = nc == 0 ? Cint[] : Cint.(lam_constr_em.indices .- 1)
    cH = nc == 0 ? Float64[] : Matrix{Float64}(lam_constr_em.R)
    ch = nc == 0 ? Float64[] : Vector{Float64}(lam_constr_em.r) ./ sd[lam_constr_em.indices]
    GC.@preserve Lam R A Q F ll cidx cH ch begin
        opts = Ref(EmOpts(T, N, r, p, max_iter, tol, 1, MEM_HOST, 0))
        init = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        out = Ref(EmOut(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL, pointer(F), C_NULL, pointer(ll),
                        Base.unsafe_convert(Ptr{Cint}, it), Base.unsafe_convert(Ptr{Cint}, st)))
        if nc == 0
            check(ccall((:dfm_em_kalman, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{EmOpts}, Ref{EmInit}, Ref{EmOut}), h, Xs, opts, init, out),
                  "dfm_em_kalman")
        else
            con = Ref(LamConstr(nc, pointer(cidx), pointer(cH), pointer(ch)))
            check(ccall((:dfm_em_kalman_constrained, LIB), Cint,
                        (Ptr{Cvoid}, Ptr{Cdouble}, Ref{EmOpts}, Ref{EmInit}, Ref{LamConstr}, Ref{EmOut}), h, Xs, opts, init, con, out),
                  "dfm_em_kalman_constrained")
        end
    end
    m.factor[m.initperiod:m.lastperiod, :] = F
    return (loglik = ll[1:it[]], iters = it[], Lam = Lam, R = R, A = A, Q = Q)
end

struct SsOpts; T::Cint; N::Cint; r::Cint; p::Cint; H::Cint; batch::Cint; mem::Cint; end
struct SsOut; F::Ptr{Cdouble}; PF::Ptr{Cdouble}; common::Ptr{Cdouble}; xhat::Ptr{Cdouble}; xvar::Ptr{Cdouble}
              loglik::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Smoothed factors, `H`-period forecasts and imputed values of the standardized panel `Xs` (NaN = missing) at the parameters
`em` returned by `estimate!(m, Parametric())` (dfm_kalman_smooth).  Rows 1..T+H; `xhat`/`xvar`/`common` in standardized units."""
function kalman_smooth(Xs::Matrix{Float64}, em, H::Integer)
    h = gethandle()
    T, N = size(Xs); r = size(em.Lam, 2); p = size(em.A, 2) ÷ r; Tp = T + H
    F = Matrix{Float64}(undef, Tp, r); PF = Array{Float64}(undef, r, r, Tp)
    common = Matrix{Float64}(undef, Tp, N); xhat = similar(common); xvar = similar(common)
    ll = Ref{Cdouble}(NaN); st = Ref{Cint}(0)
    GC.@preserve Xs em F PF common xhat xvar begin
        opts = Ref(SsOpts(T, N, r, p, H, 1, MEM_HOST))
        init = Ref(EmInit(pointer(em.Lam), pointer(em.R), pointer(em.A), pointer(em.Q), C_NULL))
        out = Ref(SsOut(pointer(F), pointer(PF), pointer(common), pointer(xhat), pointer(xvar),
                        Base.unsafe_convert(Ptr{Cdouble}, ll), Base.unsafe_convert(Ptr{Cint}, st)))
        check(ccall((:dfm_kalman_smooth, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{SsOpts}, Ref{EmInit}, Ref{SsOut}), h, Xs, opts, init, out),
              "dfm_kalman_smooth")
    end
    return (F = F, PF = PF, common = common, xhat = xhat, xvar = xvar, loglik = ll[], status = st[])
end

struct SimOpts; T::Cint; N::Cint; r::Cint; p::Cint; H::Cint; n_draw::Clonglong; draw0::Clonglong; seed::Culonglong; mem::Cint; end
struct SimOut; F::Ptr{Cdouble}; X::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Draws `draw0 .. draw0+n_draw-1` (stream `seed`) from the JOINT posterior of the factor path and the missing / forecast
cells of the standardized panel `Xs` at the parameters `em` of `estimate!(m, Parametric())` (dfm_simulation_smoother).
F: (T+H) x r x n_draw, X: (T+H) x N x n_draw (standardized units; the data where observed)."""
function simulation_smoother(Xs::Matrix{Float64}, em, H::Integer, n_draw::Integer, seed::Integer; draw0::Integer = 0)
    h = gethandle()
    T, N = size(Xs); r = size(em.Lam, 2); p = size(em.A, 2) ÷ r; Tp = T + H
    F = Array{Float64}(undef, Tp, r, n_draw); X = Array{Float64}(undef, Tp, N, n_draw); st = Ref{Cint}(0)
    GC.@preserve Xs em F X begin
        opts = Ref(SimOpts(T, N, r, p, H, n_draw, draw0, seed, MEM_HOST))
        init = Ref(EmInit(pointer(em.Lam), pointer(em.R), pointer(em.A), pointer(em.Q), C_NULL))
        out = Ref(SimOut(pointer(F), pointer(X), Base.unsafe_convert(Ptr{Cint}, st)))
        check(ccall((:dfm_simulation_smoother, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{SimOpts}, Ref{EmInit}, Ref{SimOut}),
                    h, Xs, opts, init, out), "dfm_simulation_smoother")
    end
    return (F = F, X = X, status = st[])
end

struct NewsOpts; T::Cint; N::Cint; r::Cint; p::Cint; H::Cint; news_rows::Cint; n_target::Cint
                 target_series::Ptr{Cint}; target_period::Ptr{Cint}; batch::Cint; mem::Cint; end
struct NewsOut; old_est::Ptr{Cdouble}; new_est::Ptr{Cdouble}; news::Ptr{Cdouble}; weight::Ptr{Cdouble}; contrib::Ptr{Cdouble}
                status::Ptr{Cint}; end

"""News decomposition (dfm_news) of the revision of each target between the standardized vintages `Xold` and `Xnew` (NaN =
missing; `Xnew` only adds cells, in its last `news_rows` rows) at the parameters `em` of `estimate!(m, Parametric())`.
`targets`: (series, period) pairs, 1-based, period <= T+H.  Returns old / new estimates, news (news_rows x N) and weights /
contributions (news_rows x N x n_target), all in standardized units."""
function news(Xold::Matrix{Float64}, Xnew::Matrix{Float64}, em, H::Integer, targets, news_rows::Integer)
    h = gethandle()
    T, N = size(Xold); r = size(em.Lam, 2); p = size(em.A, 2) ÷ r; nq = length(targets)
    ts = Cint[t[1] - 1 for t in targets]; tp = Cint[t[2] - 1 for t in targets]
    old = Vector{Float64}(undef, nq); new = similar(old); nw = Matrix{Float64}(undef, news_rows, N)
    w = Array{Float64}(undef, news_rows, N, nq); c = similar(w); st = Ref{Cint}(0)
    GC.@preserve Xold Xnew em ts tp old new nw w c begin
        opts = Ref(NewsOpts(T, N, r, p, H, news_rows, nq, pointer(ts), pointer(tp), 1, MEM_HOST))
        init = Ref(EmInit(pointer(em.Lam), pointer(em.R), pointer(em.A), pointer(em.Q), C_NULL))
        out = Ref(NewsOut(pointer(old), pointer(new), pointer(nw), pointer(w), pointer(c), Base.unsafe_convert(Ptr{Cint}, st)))
        check(ccall((:dfm_news, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cdouble}, Ref{NewsOpts}, Ref{EmInit}, Ref{NewsOut}),
                    h, Xold, Xnew, opts, init, out), "dfm_news")
    end
    return (old = old, new = new, news = nw, weights = w, contributions = c, status = st[])
end

struct SsbOpts; T::Cint; N::Cint; r::Cint; p::Cint; H_irf::Cint; H_fc::Cint; fc_rows::Cint; max_iter::Cint; tol::Cdouble
                n_rep::Clonglong; rep0::Clonglong; seed::Culonglong; mem::Cint; end
struct SsbOut; Lam::Ptr{Cdouble}; R::Ptr{Cdouble}; A::Ptr{Cdouble}; Q::Ptr{Cdouble}; irf::Ptr{Cdouble}; xhat::Ptr{Cdouble}
               xvar::Ptr{Cdouble}; loglik::Ptr{Cdouble}; iters::Ptr{Cint}; status::Ptr{Cint}; end

"""Parametric bootstrap (dfm_ss_bootstrap) of the state-space model `em` (the result of `estimate!(m, Parametric())`, P0
included) fitted to the standardized panel `Xs`: replicates `rep0 .. rep0+n_rep-1` (stream `seed`) are simulated, re-estimated
by EM from `em` and rotated back onto it.  Returns the aligned Lam (N x r x n_rep), R, A, Q, the impulse responses
irf (r x H_irf x r x n_rep, [shock, horizon, variable] as `dfm_irf`), xhat / xvar (fc_rows x N x n_rep: the last fc_rows of
the T+H_fc rows), loglik, iters, status (standardized units; status != 0: a failed replicate with NaN records)."""
function ss_bootstrap(Xs::Matrix{Float64}, em, n_rep::Integer, seed::Integer; H_irf::Integer = 24, H_fc::Integer = 0,
                      fc_rows::Integer = H_fc, max_iter::Integer = 50, tol::Real = 0.0, rep0::Integer = 0)
    h = gethandle()
    T, N = size(Xs); r = size(em.Lam, 2); k = size(em.A, 2); p = k ÷ r
    Lam = Array{Float64}(undef, N, r, n_rep); R = Matrix{Float64}(undef, N, n_rep); A = Array{Float64}(undef, r, k, n_rep)
    Q = Array{Float64}(undef, r, r, n_rep); irf = Array{Float64}(undef, r, H_irf, r, n_rep)
    xhat = Array{Float64}(undef, fc_rows, N, n_rep); xvar = similar(xhat)
    ll = Vector{Float64}(undef, n_rep); it = Vector{Cint}(undef, n_rep); st = Vector{Cint}(undef, n_rep)
    GC.@preserve Xs em Lam R A Q irf xhat xvar ll it st begin
        opts = Ref(SsbOpts(T, N, r, p, H_irf, H_fc, fc_rows, max_iter, tol, n_rep, rep0, seed, MEM_HOST))
        init = Ref(EmInit(pointer(em.Lam), pointer(em.R), pointer(em.A), pointer(em.Q), pointer(em.P0)))
        out = Ref(SsbOut(pointer(Lam), pointer(R), pointer(A), pointer(Q), pointer(irf), pointer(xhat), pointer(xvar), pointer(ll),
                         pointer(it), pointer(st)))
        check(ccall((:dfm_ss_bootstrap, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{SsbOpts}, Ref{EmInit}, Ref{SsbOut}), h, Xs, opts, init, out),
              "dfm_ss_bootstrap")
    end
    return (Lam = Lam, R = R, A = A, Q = Q, irf = irf, xhat = xhat, xvar = xvar, loglik = ll, iters = it, status = st)
end

struct GibbsPrior; kap_lam::Cdouble; a_R::Cdouble; b_R::Cdouble; kap_A::Cdouble; nu_Q::Cdouble; s_Q::Cdouble; end
struct GibbsOpts; T::Cint; N::Cint; r::Cint; p::Cint; H_irf::Cint; H_fc::Cint; fc_rows::Cint; n_chain::Cint; chain0::Clonglong
                  sweep0::Clonglong; n_burn::Cint; n_keep::Cint; thin::Cint; seed::Culonglong; mem::Cint; prior::GibbsPrior; end
struct GibbsOut; Lam::Ptr{Cdouble}; R::Ptr{Cdouble}; A::Ptr{Cdouble}; Q::Ptr{Cdouble}; irf::Ptr{Cdouble}; F::Ptr{Cdouble}
                 X::Ptr{Cdouble}; loglik::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Gibbs sampler (dfm_gibbs) of the state-space model on the standardized panel `Xs`: `n_chain` chains (ids chain0 ..), all
started at `em` (the result of `estimate!(m, Parametric())`, P0 included and held fixed), `n_burn` burn-in sweeps then `n_keep`
kept draws every `thin` sweeps, conjugate prior `prior` (standardized units; default kap_lam = kap_A = 0.01, a_R = 3, b_R = 1,
nu_Q = r + 2, s_Q = 1).  Returns the raw draws Lam (N x r x n_keep x n_chain), R, A, Q, the impulse responses of each draw
aligned onto `em` (irf: r x H_irf x r x n_keep x n_chain, [shock, horizon, variable] as `dfm_irf`), the factor paths
F ((T+H_fc) x r x ..), the predictive panel X (fc_rows x N x ..: the last fc_rows of the T+H_fc rows), loglik (n_sweep x
n_chain) and status (n_chain)."""
function gibbs(Xs::Matrix{Float64}, em, n_chain::Integer, seed::Integer; n_burn::Integer = 500, n_keep::Integer = 1000,
               thin::Integer = 1, H_irf::Integer = 24, H_fc::Integer = 0, fc_rows::Integer = H_fc, chain0::Integer = 0,
               sweep0::Integer = 0, prior = nothing)
    h = gethandle()
    T, N = size(Xs); r = size(em.Lam, 2); k = size(em.A, 2); p = k ÷ r; Tp = T + H_fc; ns = n_burn + n_keep * thin
    pr = prior === nothing ? GibbsPrior(0.01, 3.0, 1.0, 0.01, r + 2.0, 1.0) : prior
    rep(a) = repeat(vec(a), n_chain)
    iL = rep(em.Lam); iR = rep(em.R); iA = rep(em.A); iQ = rep(em.Q); iP = rep(em.P0)
    Lam = Array{Float64}(undef, N, r, n_keep, n_chain); R = Array{Float64}(undef, N, n_keep, n_chain)
    A = Array{Float64}(undef, r, k, n_keep, n_chain); Q = Array{Float64}(undef, r, r, n_keep, n_chain)
    irf = Array{Float64}(undef, r, max(H_irf, 0), r, n_keep, n_chain); F = Array{Float64}(undef, Tp, r, n_keep, n_chain)
    X = Array{Float64}(undef, fc_rows, N, n_keep, n_chain); ll = Matrix{Float64}(undef, ns, n_chain); st = Vector{Cint}(undef, n_chain)
    GC.@preserve Xs em iL iR iA iQ iP Lam R A Q irf F X ll st begin
        opts = Ref(GibbsOpts(T, N, r, p, H_irf, H_fc, fc_rows, n_chain, chain0, sweep0, n_burn, n_keep, thin, seed, MEM_HOST, pr))
        init = Ref(EmInit(pointer(iL), pointer(iR), pointer(iA), pointer(iQ), pointer(iP)))
        ref = Ref(EmInit(pointer(em.Lam), pointer(em.R), pointer(em.A), pointer(em.Q), C_NULL))
        out = Ref(GibbsOut(pointer(Lam), pointer(R), pointer(A), pointer(Q), H_irf > 0 ? pointer(irf) : C_NULL, pointer(F),
                           fc_rows > 0 ? pointer(X) : C_NULL, pointer(ll), pointer(st)))
        check(ccall((:dfm_gibbs, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{GibbsOpts}, Ref{EmInit}, Ref{EmInit}, Ref{GibbsOut}),
                    h, Xs, opts, init, ref, out), "dfm_gibbs")
    end
    return (Lam = Lam, R = R, A = A, Q = Q, irf = irf, F = F, X = X, loglik = ll, status = st)
end

"""Gibbs sampler under linear restrictions on the loadings (dfm_gibbs_constrained): as `gibbs` without impulse responses, with
`index` (0-based series), `Hc` (n_constr x r) and `hc` (n_constr) in STANDARDIZED units (em.lam_constr of a restricted fit)."""
function gibbs_constrained(Xs::Matrix{Float64}, em, index::Vector{Cint}, Hc::Matrix{Float64}, hc::Vector{Float64}, n_chain::Integer,
                           seed::Integer; n_burn::Integer = 500, n_keep::Integer = 1000, thin::Integer = 1, chain0::Integer = 0,
                           sweep0::Integer = 0, prior = nothing)
    h = gethandle()
    T, N = size(Xs); r = size(em.Lam, 2); k = size(em.A, 2); p = k ÷ r; ns = n_burn + n_keep * thin; nc = length(index)
    pr = prior === nothing ? GibbsPrior(0.01, 3.0, 1.0, 0.01, r + 2.0, 1.0) : prior
    rep(a) = repeat(vec(a), n_chain)
    iL = rep(em.Lam); iR = rep(em.R); iA = rep(em.A); iQ = rep(em.Q); iP = rep(em.P0)
    Lam = Array{Float64}(undef, N, r, n_keep, n_chain); R = Array{Float64}(undef, N, n_keep, n_chain)
    A = Array{Float64}(undef, r, k, n_keep, n_chain); Q = Array{Float64}(undef, r, r, n_keep, n_chain)
    ll = Matrix{Float64}(undef, ns, n_chain); st = Vector{Cint}(undef, n_chain)
    GC.@preserve Xs em iL iR iA iQ iP Lam R A Q ll st index Hc hc begin
        opts = Ref(GibbsOpts(T, N, r, p, 0, 0, 0, n_chain, chain0, sweep0, n_burn, n_keep, thin, seed, MEM_HOST, pr))
        init = Ref(EmInit(pointer(iL), pointer(iR), pointer(iA), pointer(iQ), pointer(iP)))
        con = Ref(LamConstr(nc, pointer(index), pointer(Hc), pointer(hc)))
        out = Ref(GibbsOut(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL, C_NULL, C_NULL, pointer(ll), pointer(st)))
        check(ccall((:dfm_gibbs_constrained, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cdouble}, Ref{GibbsOpts}, Ref{EmInit}, Ptr{Cvoid}, Ref{LamConstr}, Ref{GibbsOut}),
                    h, Xs, opts, init, C_NULL, con, out), "dfm_gibbs_constrained")
    end
    return (Lam = Lam, R = R, A = A, Q = Q, loglik = ll, status = st)
end

"""Series responses and forecast-error variance decompositions (dfm_series_responses) of B models Lam (N x r x B), R (N x B),
A (r x k x B), Q (r x r x B): resp, fevd (N x H x n_shock x B) and status (B); `scale` (N) multiplies resp (e.g. xstd)."""
function series_responses(Lam::Array{Float64,3}, R::Matrix{Float64}, A::Array{Float64,3}, Q::Array{Float64,3}, H::Integer;
                          n_shock::Integer = size(Lam, 2), scale = nothing)
    h = gethandle()
    N, r, B = size(Lam); p = size(A, 2) ÷ r
    resp = Array{Float64}(undef, N, H, n_shock, B); fevd = similar(resp); st = Vector{Cint}(undef, B)
    sc = scale === nothing ? Float64[] : Vector{Float64}(scale)
    GC.@preserve Lam R A Q resp fevd st sc begin
        models = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        check(ccall((:dfm_series_responses, LIB), Cint,
                    (Ptr{Cvoid}, Ref{EmInit}, Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Cdouble}, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cint}),
                    h, models, N, r, p, B, H, n_shock, scale === nothing ? C_NULL : pointer(sc), MEM_HOST, resp, fevd, st),
              "dfm_series_responses")
    end
    return (resp = resp, fevd = fevd, status = st)
end

struct HdOpts; N::Cint; r::Cint; p::Cint; Tp::Cint; t0::Cint; n_shock::Cint; n_model::Cint; mem::Cint; end
struct HdOut; shocks::Ptr{Cdouble}; contrib::Ptr{Cdouble}; rest::Ptr{Cdouble}; base::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Historical decompositions (dfm_historical_decomposition) of B models Lam (N x r x B), R (N x B), A (r x k x B), Q (r x r x B)
along their factor paths F (Tp x r x B) from the 0-based base row t0 (p - 1 <= t0 < Tp): shocks (Tp x r x B), contrib
(N x Tp x n_shock x B), rest and base (N x Tp x B), status (B); `scale` (N) multiplies the series' parts (e.g. xstd)."""
function historical_decomposition(Lam::Array{Float64,3}, R::Matrix{Float64}, A::Array{Float64,3}, Q::Array{Float64,3},
                                  F::Array{Float64,3}, t0::Integer; n_shock::Integer = size(Lam, 2), scale = nothing)
    h = gethandle()
    N, r, B = size(Lam); p = size(A, 2) ÷ r; Tp = size(F, 1)
    shocks = Array{Float64}(undef, Tp, r, B); contrib = Array{Float64}(undef, N, Tp, n_shock, B)
    rest = Array{Float64}(undef, N, Tp, B); base = similar(rest); st = Vector{Cint}(undef, B)
    sc = scale === nothing ? Float64[] : Vector{Float64}(scale)
    GC.@preserve Lam R A Q F shocks contrib rest base st sc begin
        models = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        opts = Ref(HdOpts(N, r, p, Tp, t0, n_shock, B, MEM_HOST))
        out = Ref(HdOut(pointer(shocks), pointer(contrib), pointer(rest), pointer(base), pointer(st)))
        check(ccall((:dfm_historical_decomposition, LIB), Cint,
                    (Ptr{Cvoid}, Ref{EmInit}, Ptr{Cdouble}, Ptr{Cdouble}, Ref{HdOpts}, Ref{HdOut}),
                    h, models, F, scale === nothing ? C_NULL : pointer(sc), opts, out), "dfm_historical_decomposition")
    end
    return (shocks = shocks, contrib = contrib, rest = rest, base = base, status = st)
end

struct SignOpts; N::Cint; r::Cint; p::Cint; n_model::Cint; H::Cint; n_shock::Cint; n_rot::Clonglong; n_keep::Cint; seed::Culonglong; mem::Cint; end
struct SignRestr; n::Cint; series::Ptr{Cint}; horizon::Ptr{Cint}; shock::Ptr{Cint}; sign::Ptr{Cint}; end
struct SignOut; n_accept::Ptr{Clonglong}; cand::Ptr{Clonglong}; rot::Ptr{Cdouble}; resp::Ptr{Cdouble}; fevd::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Shocks identified by sign restrictions (dfm_sign_restrictions) on B models Lam (N x r x B), R (N x B), A (r x k x B),
Q (r x r x B).  rows: (series, horizon, shock, sign) tuples, series and horizon 0-based, shock 1-based, sign +1 / -1.  Returns
n_accept (B), cand (n_keep x B, -1 for an empty slot), rot (r x r x n_keep x B), resp and fevd (N x H x n_shock x n_keep x B),
status (B); `scale` (N) multiplies resp (e.g. xstd); `ids` (B) the models' ids (default 0 .. B-1)."""
function sign_restrictions(Lam::Array{Float64,3}, R::Matrix{Float64}, A::Array{Float64,3}, Q::Array{Float64,3}, rows, H::Integer,
                           n_rot::Integer, n_keep::Integer; n_shock::Integer = maximum(r_[3] for r_ in rows), seed::Integer = 0,
                           ids = nothing, scale = nothing)
    h = gethandle()
    N, r, B = size(Lam); p = size(A, 2) ÷ r
    rs = Cint[r_[1] for r_ in rows]; rh = Cint[r_[2] for r_ in rows]; rj = Cint[r_[3] for r_ in rows]; rg = Cint[r_[4] for r_ in rows]
    na = Vector{Clonglong}(undef, B); cand = Array{Clonglong}(undef, n_keep, B); rot = Array{Float64}(undef, r, r, n_keep, B)
    resp = Array{Float64}(undef, N, H, n_shock, n_keep, B); fevd = similar(resp); st = Vector{Cint}(undef, B)
    sc = scale === nothing ? Float64[] : Vector{Float64}(scale)
    iv = ids === nothing ? Culonglong[] : Vector{Culonglong}(ids)
    GC.@preserve Lam R A Q rs rh rj rg na cand rot resp fevd st sc iv begin
        models = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        opts = Ref(SignOpts(N, r, p, B, H, n_shock, n_rot, n_keep, seed, MEM_HOST))
        rr = Ref(SignRestr(length(rows), pointer(rs), pointer(rh), pointer(rj), pointer(rg)))
        out = Ref(SignOut(pointer(na), pointer(cand), pointer(rot), pointer(resp), pointer(fevd), pointer(st)))
        check(ccall((:dfm_sign_restrictions, LIB), Cint,
                    (Ptr{Cvoid}, Ref{EmInit}, Ptr{Culonglong}, Ptr{Cdouble}, Ref{SignOpts}, Ref{SignRestr}, Ref{SignOut}),
                    h, models, ids === nothing ? C_NULL : pointer(iv), scale === nothing ? C_NULL : pointer(sc), opts, rr, out),
              "dfm_sign_restrictions")
    end
    return (n_accept = na, cand = cand, rot = rot, resp = resp, fevd = fevd, status = st)
end


struct NarrOpts; N::Cint; r::Cint; p::Cint; n_model::Cint; H::Cint; n_shock::Cint; n_rot::Clonglong; n_keep::Cint; seed::Culonglong; mem::Cint; Tp::Cint; n_sim::Cint; end
struct NarrRestr; n::Cint; kind::Ptr{Cint}; shock::Ptr{Cint}; series::Ptr{Cint}; row::Ptr{Cint}; h::Ptr{Cint}; sign::Ptr{Cint}; end
struct NarrOut; n_accept::Ptr{Clonglong}; cand::Ptr{Clonglong}; rot::Ptr{Cdouble}; resp::Ptr{Cdouble}; fevd::Ptr{Cdouble}; status::Ptr{Cint};
               n_ok::Ptr{Clonglong}; weight::Ptr{Cdouble}; eps::Ptr{Cdouble}; end

"""Narrative sign restrictions (dfm_narrative_sign_restrictions) on B models as `sign_restrictions`, along their factor paths F
(Tp x r x B).  narr: (kind, shock, series, row, h, sign) tuples, kind 0 shock sign / 1 most important / 2 overwhelming /
3 contribution sign, shock 1-based, series and row 0-based.  Returns sign_restrictions' fields and n_ok, weight (n_keep x B),
eps (Tp x n_shock x n_keep x B).  Not run in this repository's tests."""
function narrative_sign_restrictions(Lam::Array{Float64,3}, R::Matrix{Float64}, A::Array{Float64,3}, Q::Array{Float64,3},
                                     F::Array{Float64,3}, rows, narr, H::Integer, n_rot::Integer, n_keep::Integer;
                                     n_shock::Integer = maximum(vcat([1], [r_[3] for r_ in rows], [n_[2] for n_ in narr])),
                                     n_sim::Integer = 16384, seed::Integer = 0, ids = nothing, scale = nothing)
    h = gethandle()
    N, r, B = size(Lam); p = size(A, 2) ÷ r; Tp = size(F, 1)
    rs = Cint[r_[1] for r_ in rows]; rh = Cint[r_[2] for r_ in rows]; rj = Cint[r_[3] for r_ in rows]; rg = Cint[r_[4] for r_ in rows]
    nv = [Cint[n_[q] for n_ in narr] for q in 1:6]
    na = Vector{Clonglong}(undef, B); cand = Array{Clonglong}(undef, n_keep, B); rot = Array{Float64}(undef, r, r, n_keep, B)
    resp = Array{Float64}(undef, N, H, n_shock, n_keep, B); fevd = similar(resp); st = Vector{Cint}(undef, B)
    nok = Array{Clonglong}(undef, n_keep, B); w = Array{Float64}(undef, n_keep, B); eps = Array{Float64}(undef, Tp, n_shock, n_keep, B)
    sc = scale === nothing ? Float64[] : Vector{Float64}(scale)
    iv = ids === nothing ? Culonglong[] : Vector{Culonglong}(ids)
    GC.@preserve Lam R A Q F rs rh rj rg nv na cand rot resp fevd st nok w eps sc iv begin
        models = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        opts = Ref(NarrOpts(N, r, p, B, H, n_shock, n_rot, n_keep, seed, MEM_HOST, Tp, n_sim))
        rr = Ref(SignRestr(length(rows), pointer(rs), pointer(rh), pointer(rj), pointer(rg)))
        nr = Ref(NarrRestr(length(narr), pointer(nv[1]), pointer(nv[2]), pointer(nv[3]), pointer(nv[4]), pointer(nv[5]), pointer(nv[6])))
        out = Ref(NarrOut(pointer(na), pointer(cand), pointer(rot), pointer(resp), pointer(fevd), pointer(st), pointer(nok), pointer(w),
                          pointer(eps)))
        check(ccall((:dfm_narrative_sign_restrictions, LIB), Cint,
                    (Ptr{Cvoid}, Ref{EmInit}, Ptr{Cdouble}, Ptr{Culonglong}, Ptr{Cdouble}, Ref{NarrOpts}, Ref{SignRestr}, Ref{NarrRestr},
                     Ref{NarrOut}),
                    h, models, pointer(F), ids === nothing ? C_NULL : pointer(iv), scale === nothing ? C_NULL : pointer(sc), opts, rr, nr,
                    out), "dfm_narrative_sign_restrictions")
    end
    return (n_accept = na, cand = cand, rot = rot, resp = resp, fevd = fevd, status = st, n_ok = nok, weight = w, eps = eps)
end


struct ProxyOpts; N::Cint; r::Cint; p::Cint; n_model::Cint; Tp::Cint; H::Cint; n_inst::Cint; i0::Cint; q::Cint; block::Cint; n_boot::Cint;
                  seed::Culonglong; mem::Cint; end
struct ProxyOut; omega::Ptr{Cdouble}; resp::Ptr{Cdouble}; fevd::Ptr{Cdouble}; eps::Ptr{Cdouble}; n_obs::Ptr{Cint}; reliability::Ptr{Cdouble};
                 fs_pi::Ptr{Cdouble}; fs_F::Ptr{Cdouble}; status::Ptr{Cint}; end

"""Shocks identified by external instruments (dfm_proxy_identification) on B models as `sign_restrictions`, along their factor
paths F (Tp x r x B), with instruments Z (Tp x n_inst, NaN = unavailable) and the first stage's series i0 (0-based).  Returns omega
(r x (1 + n_boot) x n_inst x B), resp and fevd (N x H x (1 + n_boot) x n_inst x B), eps (Tp x n_inst x B), n_obs, reliability,
fs_pi, fs_F, status (n_inst x B); replicate 0 is the sample, 1 .. n_boot the moving-block bootstrap.  Not run in this
repository's tests."""
function proxy_identification(Lam::Array{Float64,3}, R::Matrix{Float64}, A::Array{Float64,3}, Q::Array{Float64,3},
                              F::Array{Float64,3}, Z::Matrix{Float64}, i0::Integer, H::Integer; n_boot::Integer = 0, block::Integer = 1,
                              q::Integer = 0, seed::Integer = 0, ids = nothing, scale = nothing)
    h = gethandle()
    N, r, B = size(Lam); p = size(A, 2) ÷ r; Tp = size(F, 1); ni = size(Z, 2); nr = 1 + n_boot
    om = Array{Float64}(undef, r, nr, ni, B); resp = Array{Float64}(undef, N, H, nr, ni, B); fevd = similar(resp)
    eps = Array{Float64}(undef, Tp, ni, B); nobs = Array{Cint}(undef, ni, B); rel = Array{Float64}(undef, ni, B)
    fpi = similar(rel); fF = similar(rel); st = Array{Cint}(undef, ni, B)
    sc = scale === nothing ? Float64[] : Vector{Float64}(scale)
    iv = ids === nothing ? Culonglong[] : Vector{Culonglong}(ids)
    GC.@preserve Lam R A Q F Z om resp fevd eps nobs rel fpi fF st sc iv begin
        models = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        opts = Ref(ProxyOpts(N, r, p, B, Tp, H, ni, i0, q, block, n_boot, seed, MEM_HOST))
        out = Ref(ProxyOut(pointer(om), pointer(resp), pointer(fevd), pointer(eps), pointer(nobs), pointer(rel), pointer(fpi), pointer(fF),
                           pointer(st)))
        check(ccall((:dfm_proxy_identification, LIB), Cint,
                    (Ptr{Cvoid}, Ref{EmInit}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Culonglong}, Ptr{Cdouble}, Ref{ProxyOpts}, Ref{ProxyOut}),
                    h, models, pointer(F), pointer(Z), ids === nothing ? C_NULL : pointer(iv), scale === nothing ? C_NULL : pointer(sc),
                    opts, out), "dfm_proxy_identification")
    end
    return (omega = om, resp = resp, fevd = fevd, eps = eps, n_obs = nobs, reliability = rel, fs_pi = fpi, fs_F = fF, status = st)
end

end # module
