"""Oracle checks on the dispatch branches of the non-parametric path: PCA (Gram mode, eigen-solver, finishing kernel), the
ALS sweep kernels, the loadings with their idiosyncratic AR step, the factor VAR and IRF, the instability tests and
fitted-value correlations, the percentile bands, and the batch limit of the launches that put the batch on gridDim.y.
CASES is the table; test_gpu_np_dispatch.py runs it on the H100 with the kernel-set assertion (dispatch_checks.KernelLog),
test_emu_np_dispatch.py on the host-emulation build.

Each case's comment gives the numbers that select its branch on the H100 (dfm_api.cu), with
em_lds(n) = n + (12 - n % 8) % 8:
  - run_pca: nmax = min(N, T) <= 64: k_jacobi; else the block size m = min(nmax, 64, max(2r, r + 16)) and
    subspace2_smem_doubles(nmax, m) = 2 em_lds(nmax) m + 3 m^2 + 4m + 196 doubles: k_subspace_eig2 when that is <= 110 KB
    and m <= 48, else k_subspace_eig;
  - k_pca_finish: mode 0 (balanced columns <= T) / mode 1 (more); the tensor-core product when N <= T, r <= 48, every
    column balanced and smFast = (r / 2 + 50) 8 + em_lds(nmax) r 8 + 64 <= 100 KB, else the scalar loop;
  - estimate_factor: k_als_fused2 (balanced, even T, r <= 8, fits 113 KB), k_als_masked (r <= 8, fits 100 KB), else the
    general loop k_als_lambda / k_gram_small / k_als_factor / k_als_check.  k_als_factor runs tpt_threads(np + r) threads
    (np = r (r + 1) / 2): 96 KB / (8 (np + r)) rounded down to a multiple of 32, clamped to [32, 128]; its systems take
    ((np + r) threads + 48) 8 bytes of shared memory while that is <= 220 KB (r <= 40), else a global scratch."""
import numpy as np

from oracle import dfm_ref as R
from oracle.dgp import simulate_panel
import dispatch_checks as DC
import parity_checks as P
from dynamic_factor_models_b200 import DFMError

METHODS = ("pca_score", "estimate_factor", "estimate_loading", "estimate_var", "irf", "instability", "fit_correlation",
           "percentiles", "em_kalman")
CASES = []


def case(id_, kernels):
    return DC.case(id_, kernels, table=CASES)


def raises(code, fn, *a, **kw):
    try:
        fn(*a, **kw)
    except DFMError as e:
        assert e.code == code, "status %d, expected %d: %s" % (e.code, code, e)
        return
    raise AssertionError("no error, expected status %d" % code)


SOLVERS = ("k_jacobi", "k_subspace_eig2", "k_subspace_eig")


def pca(solver):
    return {"pca_score": (("k_gram_tc", solver, "k_pca_finish"), tuple(s for s in SOLVERS if s != solver))}


# ---------------------------------------------------------------------------------------------------- PCA
# Raw scores against numpy's SVD with the documented sign rule (no sign alignment), on panels whose top singular values
# and largest singular-vector entries are apart (P.pca_sign_rule asserts it).
@case("pca_jacobi_nmax64_gram_mode1", pca("k_jacobi"))
def _(lib):
    # T = 64 < N = 90: Gram XX' (mode 1), nmax = 64 <= 64: k_jacobi; scalar finish (N > T)
    P.check_pca(lib, r=6, sizes=((64, 90),), sign_rule=True)


@case("pca_jacobi_nmax63_odd", pca("k_jacobi"))
def _(lib):
    # N = 63 < T = 120: mode 0, odd nmax = 63: k_jacobi; smFast = 424 + 64 * 6 * 8 + 64 = 3560 B: tensor-core finish
    P.check_pca(lib, r=6, sizes=((120, 63),), sign_rule=True)


@case("pca_eig2_nmax65", pca("k_subspace_eig2"))
def _(lib):
    # nmax = 65, r = 8: m = 24, (2 * 68 * 24 + 3 * 576 + 96 + 196) 8 = 41,760 B <= 110 KB: k_subspace_eig2
    P.check_pca(lib, r=8, sizes=((120, 65),), sign_rule=True)


@case("pca_eig_r25_m50", pca("k_subspace_eig"))
def _(lib):
    # nmax = 100, r = 25: m = 50 > 48: k_subspace_eig; smFast = 496 + 100 * 25 * 8 + 64 = 20,560 B: tensor-core finish
    P.check_pca(lib, r=25, sizes=((200, 100),), sign_rule=True)


@case("pca_eig_r48_m64", pca("k_subspace_eig"))
def _(lib):
    # nmax = 100, r = 48: m = 64 > 48: k_subspace_eig; smFast = 592 + 100 * 48 * 8 + 64 = 39,056 B: tensor-core finish
    P.check_pca(lib, r=48, sizes=((200, 100),), sign_rule=True)


@case("pca_eig_r24_plan_past_110KB", pca("k_subspace_eig"))
def _(lib):
    # nmax = 100, r = 24: m = 48, but (2 * 100 * 48 + 3 * 2304 + 192 + 196) 8 = 134,688 B > 110 KB: k_subspace_eig
    P.check_pca(lib, r=24, sizes=((200, 100),), sign_rule=True)


@case("pca_finish_scalar_mode0_T400_N300_r48", pca("k_subspace_eig"))
def _(lib):
    # N = 300 <= T = 400 but smFast = 592 + 300 * 48 * 8 + 64 = 115,856 B > 100 KB: scalar mode-0 finish; m = 64: k_subspace_eig
    P.check_pca(lib, r=48, sizes=((400, 300),), sign_rule=True)


@case("pca_finish_mode1_subspace", pca("k_subspace_eig2"))
def _(lib):
    # T = 100 < N = 150: Gram XX' (mode 1), nmax = 100, r = 8: m = 24, 47,264 B: k_subspace_eig2; scalar mode-1 finish
    P.check_pca(lib, r=8, sizes=((100, 150),), sign_rule=True)


@case("pca_batch3", pca("k_jacobi"))
def _(lib):
    # 3 panels in one call (grid.y / grid.x = batch) against one call per panel; nmax = 40: k_jacobi
    P.check_pca(lib, r=5, sizes=((120, 40),), sign_rule=True, batch=3)


# ---------------------------------------------------------------------------------------------------- ALS
ALS_GEN = {"estimate_factor": (("k_als_lambda", "k_gram_small", "k_als_factor", "k_als_check"), ("k_als_fused2<RT>", "k_als_masked<RT>"))}


@case("als_pca_start_missing_cols_r30", {"estimate_factor": (("k_subspace_eig", "k_pca_finish", "k_als_factor"),
                                                             ("k_jacobi", "k_subspace_eig2", "k_als_fused2<RT>", "k_als_masked<RT>"))})
def _(lib):
    # missing data in 40 of 80 columns: the PCA runs on the 40 balanced columns, but run_pca sizes its plan by
    # nmax = min(N, T) = 80 > 64, m = min(80, 60) = 60 > 48: k_subspace_eig; scalar mode-0 finish (not every column
    # balanced).  One sweep from the library's own PCA start against the oracle started from the sign rule, so a wrong
    # sign shows in F
    P.check_estimate_factor_same_init(lib, N=80, r=30, T=150, miss=0.03, iters=(1,), short_series=False, pca_start=True)


def _als_width(r):
    # k_als_factor threads: r = 12: np + r = 90 -> 136 -> 128; 13: 104 -> 118 -> 96; 15: 135 -> 91 -> 64; 18: 189 -> 65 -> 64;
    # 19: 209 -> 58 -> 32; 40: 860 -> 14 -> 32, ((860 * 32 + 48) 8 = 220,544 B <= 220 KB: systems in shared memory)
    @case("als_factor_r%d" % r, ALS_GEN)
    def _(lib):
        N, T = 2 * r + 12, 120 + 2 * r
        P.check_estimate_factor_same_init(lib, N=N, r=r, T=T, miss=0.04, iters=(1, 4))
        P.check_estimate_factor_same_init(lib, N=N, r=r, T=T, miss=0.0, iters=(3,), short_series=False)


for _r in (12, 13, 15, 18, 19, 40):
    _als_width(_r)


def _als_global(r):
    # (np + r) 32 + 48 doubles: r = 41: 231,296 B, 48: 315,008 B, 64: 549,248 B > 220 KB: systems in the global scratch
    # (48 is the largest r with the PCA start, 64 the largest with F_init)
    @case("als_factor_global_r%d" % r, ALS_GEN)
    def _(lib):
        P.check_estimate_factor_same_init(lib, N=r + 70, r=r, T=r + 100, miss=0.04, iters=(1, 3))


for _r in (41, 48, 64):
    _als_global(_r)


@case("als_factor_r8_too_big_for_fused", ALS_GEN)
def _(lib):
    # balanced, r = 8, N = 1200, T = 500: k_als_masked needs (8 * 501 + 8 * 1201 + 320 + 48) 8 = 111,872 B > 100 KB, and the
    # fused2 panel tiles exceed 113 KB: the general loop (k_als_factor at 128 threads)
    P.check_estimate_factor_same_init(lib, N=1200, r=8, T=500, miss=0.0, iters=(2,), short_series=False)


@case("als_masked_balanced_odd_T", {"estimate_factor": (("k_als_masked<RT>",), ("k_als_fused2<RT>", "k_als_factor"))})
def _(lib):
    # balanced but T = 151 odd: k_als_fused2 needs even T, so k_als_masked<4> runs
    P.check_estimate_factor_same_init(lib, N=30, r=4, T=151, miss=0.0, iters=(1, 5), short_series=False)


@case("als_batch_r12_different_sweeps", ALS_GEN)
def _(lib):
    # 3 balanced panels at r = 12 (general loop, 128 threads) that stop after different numbers of sweeps
    P.check_als_balanced(lib, N=40, r=12, T=150, B=3, per_panel=True)


@case("als_constraint_two_rows_one_series_r12", ALS_GEN)
def _(lib):
    # constraints always take the general loop; two rows on series 2
    Rm = np.zeros((2, 12)); Rm[0, 0] = 1.0; Rm[1, 1] = 1.0; Rm[1, 2] = -1.0
    P.check_estimate_factor_same_init(lib, N=36, r=12, T=140, miss=0.04, iters=(1, 4), constr=([2, 2], Rm, [0.5, -0.25]))


# ---------------------------------------------------------------------------------------------------- loadings
LOAD = {"estimate_loading": (("k_loading",), ())}


def _loading(id_, **kw):
    @case("loading_" + id_, LOAD)
    def _(lib):
        P.check_loading(lib, **kw)


_loading("r1", r=1)
_loading("r8", N=20, r=8)
_loading("r20", N=30, r=20, T=160)
_loading("lags1", n_uarlag=1)
_loading("lags4", n_uarlag=4, T=200)
_loading("lags16", n_uarlag=16, T=200)
_loading("nt_min_edge", edge_series=True, F_holes=(50, 51))
_loading("exact_combination", exact=True)
_loading("missing_factor_rows", F_holes=(30, 31, 77))
_loading("missing_factor_rows_lags16", F_holes=(0, 30, 31, 77, 199), n_uarlag=16, T=200)
_loading("batch3", F_holes=(30, 31, 77), batch=3, edge_series=True)


# ---------------------------------------------------------------------------------------------------- VAR and IRF
VAR_IRF = {"estimate_var": (("k_var",), ()), "irf": (("k_irf",), ())}


def var_smem(r, p, T, withconst=True):
    """k_var's shared memory (dfm_estimate_var): (K^2 + K r + r^2 + 16) 8 + T + 16 bytes, K = r p + withconst."""
    K = r * p + int(withconst)
    return (K * K + K * r + r * r + 16) * 8 + T + 16


@case("var_k64_r8_p8_tight", VAR_IRF)
def _(lib):
    # k = r p = 64, K = 65; T_used = T - p = K + r = 73 rows, the fewest that leave seps (r x r, from T_used - K residual
    # degrees of freedom) positive definite; IRF at H = 120 with shock ids out of order and repeated, and a batch of 3
    P.check_var_irf(lib, r=8, p=8, T=65 + 8 + 8, shocks=(5, 0, 5), H=120, batch=3, rtol=1e-7)


@case("var_r20_p4_tight", VAR_IRF)
def _(lib):
    # K = 81, T_used = K + r = 101; H = 1
    P.check_var_irf(lib, r=20, p=4, T=81 + 20 + 4, shocks=(19, 0), H=1, rtol=1e-7)


@case("var_noconst", VAR_IRF)
def _(lib):
    P.check_var_irf(lib, r=3, p=2, T=120, withconst=False)
    P.check_var_irf(lib, r=8, p=8, T=64 + 8 + 8, withconst=False, shocks=(7, 7, 1), H=30, rtol=1e-7)


@case("var_smem_edge", {"estimate_var": (("k_var",), ())})
def _(lib):
    # r = 20, p = 7: K = 141, 185,132 B <= 220 KB; p = 8: K = 161, 236,672 B > 220 KB: DFM_ERR_UNSUPPORTED
    assert var_smem(20, 7, 180) <= 220 * 1024 < var_smem(20, 8, 200)
    _, tr = simulate_panel(10, 20, 200, rep=6)
    out = lib.estimate_var(tr["F"][:180], 7, True)
    v = R.VARModel(tr["F"][:180].copy(), 7, True, 1, 180); R.estimate_var(v)
    np.testing.assert_allclose(out["betahat"], v.betahat, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(out["seps"], v.seps, rtol=1e-8)
    np.testing.assert_allclose(out["G"], v.G, rtol=1e-8, atol=1e-11)
    raises(6, lib.estimate_var, tr["F"], 8, True)


# ---------------------------------------------------------------------------------------------------- instability
INST = {"instability": (("k_instability",), ())}
FITC = {"fit_correlation": (("k_fit_corr",), ())}


def inst_smem(T, r):
    """k_instability's shared memory in doubles (inst_smem_doubles, dfm_kernels_inst.cuh)."""
    K = 2 * r
    ldg = K + (12 - K % 8) % 8
    return T * (r + 2) + (T + 8) * ldg + 6 * K * K + 2 * r * r + 6 * K + 64 + T // 2 + 8


def inst_panel(T, r, ns=3, rep=11):
    X, tr = simulate_panel(ns, r, T, rep=rep, standardize=False)
    F = tr["F"].copy()
    F[:2] = np.nan                                                   # factor rows outside the estimation window
    X[T // 3:T // 3 + 5, 0] = np.nan
    return X, F


def _instability(r, q):
    # r = 16: K = 2r = 32 regressors (the unrestricted Chow regression), the largest the kernel takes
    @case("instability_r%d_q%d" % (r, q), INST)
    def _(lib):
        X, F = inst_panel(220, r)
        P.check_instability(lib, None, q=q, qlr0=True, data=X, factor=F, lastpre=110, min_obs=60)


for _r in (1, 16):
    for _q in (0, 1, 7):
        _instability(_r, _q)


@case("instability_ccut_edges", INST)
def _(lib):
    # (r = 1: at ccut = 0.01 the first break leaves 2 rows before it)
    X, F = inst_panel(300, 1)
    for cc in (0.01, 0.49):
        P.check_instability(lib, None, q=2, ccut=cc, qlr0=True, data=X, factor=F, lastpre=100, min_obs=60)


@case("instability_largest_T_r16", INST)
def _(lib):
    # inst_smem_doubles(384, 16) * 8 = 225,216 B <= 220 KB < 225,440 B at T = 385: DFM_ERR_UNSUPPORTED
    assert inst_smem(384, 16) * 8 <= 220 * 1024 < inst_smem(385, 16) * 8
    X, F = inst_panel(385, 16, ns=2)
    P.check_instability(lib, None, q=3, qlr0=True, data=X[:384], factor=F[:384], lastpre=190, min_obs=80)
    raises(6, lib.instability, X, F, 190, q=3)


def _fitcorr(r):
    @case("fit_correlation_r%d" % r, FITC)
    def _(lib):
        X, tr = simulate_panel(5, r, 222, rep=13, standardize=False)
        F = tr["F"]
        pre = F.copy(); pre[104:] = np.nan
        post = F + 0.3 * np.random.default_rng(r).standard_normal(F.shape); post[:104] = np.nan
        X[:30, 1] = np.nan
        P.check_fit_correlation(lib, None, data=X, factors=(F, pre, post))


for _r in (20, 48):
    _fitcorr(_r)


# ---------------------------------------------------------------------------------------------------- percentiles
PCT = {"percentiles": (("k_percentiles",), ())}


@case("percentiles_sizes", PCT)
def _(lib):
    # n = 1024 and 1025 (the bitonic sort pads to 1024 / 2048), 16384 (pads to 16384: (16384 + 2) 8 = 131,088 B);
    # 16385 pads to 32768: 262,160 B > 220 KB: DFM_ERR_UNSUPPORTED
    for n in (1024, 1025, 16384):
        P.check_percentiles(lib, n=n, d=3)
    raises(6, lib.percentiles, np.zeros((16385, 2)), [50.0])


@case("percentiles_edges", PCT)
def _(lib):
    P.check_percentiles(lib, n=101, d=5, q=np.linspace(0.0, 100.0, 64), odd_columns=True)      # nq = 64, q = 0 and 100
    P.check_percentiles(lib, n=50, d=1, q=(0, 100, 37.5))


# ---------------------------------------------------------------------------------------------------- launch limits
@case("batch_65536_tiny_panels", {})
def _(lib):
    # 65,536 panels would put 65,536 blocks on gridDim.y (k_standardize, k_em_scan, ...): the call either fits them or
    # refuses with DFM_ERR_UNSUPPORTED; a launch failure (DFM_ERR_CUDA) fails the test
    from oracle import kalman_em as K
    B, T, N, r = 65536, 12, 3, 1
    rng = np.random.default_rng(5)
    f = rng.standard_normal((T, 1))
    X = f[None] * np.array([1.0, -0.5, 0.8]) + 0.3 * rng.standard_normal((B, T, N))
    picks = (0, B // 2, B - 1)
    try:
        out = lib.estimate_factor(X, r, nt_min=5, tol=1e-8, max_iter=3)
    except DFMError as e:
        assert e.code == 6, e
    else:
        for b in picks:
            m = R.DFMModel(X[b], np.ones(N, int), 5, 5, 1, T, 0, r, 1e-8, 4, 2); R.estimate_factor(m, max_iter=3)
            F, _ = P.sign_align(out["F"][b], m.factor)
            assert P.rmse(F, m.factor) < 1e-8
    Lam = np.tile(np.array([[1.0], [-0.5], [0.8]]), (B, 1, 1)); Rv = np.full((B, N), 0.1)
    A = np.full((B, 1, 1), 0.5); Q = np.ones((B, 1, 1))
    try:
        out = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=2, want_PF=False)
    except DFMError as e:
        assert e.code == 6, e
    else:
        for b in picks:
            ref = K.em_kalman(X[b], Lam[b], Rv[b], A[b], Q[b], p=1, max_iter=2)
            np.testing.assert_allclose(out["loglik"][b], ref["loglik"], rtol=1e-10)
            assert P.rmse(out["F"][b], ref["F"]) < 1e-8
