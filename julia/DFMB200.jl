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

"""`estimate!(m, ::NonParametric)` (dfm_functions.ipynb:530-543) and the `Parametric` slot of :23."""
function estimate!(m, method = Main.NonParametric(); lam_constr_f = nothing, lam_constr_fl = nothing,
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
    GC.@preserve Lam R A Q F ll begin
        opts = Ref(EmOpts(T, N, r, p, max_iter, tol, 1, MEM_HOST, 0))
        init = Ref(EmInit(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL))
        out = Ref(EmOut(pointer(Lam), pointer(R), pointer(A), pointer(Q), C_NULL, pointer(F), C_NULL, pointer(ll),
                        Base.unsafe_convert(Ptr{Cint}, it), Base.unsafe_convert(Ptr{Cint}, st)))
        check(ccall((:dfm_em_kalman, LIB), Cint, (Ptr{Cvoid}, Ptr{Cdouble}, Ref{EmOpts}, Ref{EmInit}, Ref{EmOut}), h, Xs, opts, init, out),
              "dfm_em_kalman")
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

end # module
