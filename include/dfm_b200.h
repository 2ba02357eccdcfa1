/* dfm_b200.h -- C ABI of the B200-native dynamic-factor-model hot path.
 *
 * The reference (QuantEcon/dynamic_factor_models) is pure Julia and has NO FFI / plugin
 * interface: its boundary is multiple dispatch on `EstimationMethod`
 * (dfm_functions.ipynb:21-23) with all state in the mutable fields of `DFMModel`
 * (dfm_functions.ipynb:89-111).  Each entry point below is what a Julia `ccall` (see
 * INTEGRATION.md and julia/DFMB200.jl) binds in place of one reference function; the
 * function it replaces is cited as dfm_functions.ipynb:<raw JSON line>.
 *
 * Conventions
 *  - all matrices are COLUMN-MAJOR Float64 (Julia layout); a panel is T x N, series i
 *    contiguous in t; missing observations are NaN (the Julia shim maps `missing` <-> NaN);
 *  - `batch` = B independent problems stored back to back (panel b at X + b*T*N, every
 *    output likewise); B = 1 is the reference's single-model call.  dfm_standardize, dfm_pca_score,
 *    dfm_estimate_factor, dfm_estimate_loading(_ex), dfm_irf, dfm_em_init_from_factors, dfm_em_kalman and
 *    dfm_kalman_smooth take B <= 65535 (their launches put the batch on the grid's y dimension); a larger
 *    batch returns DFM_ERR_UNSUPPORTED: split it into several calls;
 *  - `mem` says where the DATA pointers live: DFM_MEM_HOST (the library does the H2D/D2H
 *    copies on the handle's stream) or DFM_MEM_DEVICE (pointers are device pointers on the
 *    handle's device: nothing is copied).  Small option/constraint arrays are always host;
 *  - every entry point returns an int status (0 = ok) and never throws; work is issued on the
 *    handle's stream; host-memory outputs are complete when the call returns, device-memory
 *    outputs after dfm_sync();
 *  - there is NO CPU fallback: without a usable CUDA device dfm_create fails with
 *    DFM_ERR_CUDA and nothing else can be called.
 */
#ifndef DFM_B200_H
#define DFM_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define DFM_VERSION 100

enum {
  DFM_OK = 0,
  DFM_ERR_ARG = 1,          /* bad shape / null pointer / inconsistent options (reference: error(...) :124-126) */
  DFM_ERR_TOO_FEW_OBS = 2,  /* a regression has fewer observations than regressors */
  DFM_ERR_NOT_PD = 3,       /* a covariance / normal-equation matrix is not positive definite */
  DFM_ERR_NOT_CONVERGED = 4,/* informational, reported per problem in the stats structs only */
  DFM_ERR_CUDA = 5,         /* CUDA runtime error or no device */
  DFM_ERR_UNSUPPORTED = 6,  /* size outside what the kernels support (see DESIGN.md) */
  DFM_ERR_NCCL = 7
};

enum { DFM_MEM_HOST = 0, DFM_MEM_DEVICE = 1 };

typedef struct dfm_handle dfm_handle;

/* ---- handle ------------------------------------------------------------------------- */
int dfm_version(void);
const char* dfm_status_string(int status);
/* device = CUDA ordinal; the handle owns one stream and a growable device workspace. */
int dfm_create(int device, dfm_handle** out);
/* same, but work is issued on `cuda_stream` (a cudaStream_t, e.g. torch's current stream). */
int dfm_create_on_stream(int device, void* cuda_stream, dfm_handle** out);
int dfm_destroy(dfm_handle* h);
int dfm_sync(dfm_handle* h);
/* number of kernels this handle has launched since creation (bench.py's gpu_launches). */
long long dfm_launch_count(const dfm_handle* h);
const char* dfm_last_error(const dfm_handle* h);
/* Optional per-kernel device timing with CUDA events on the handle's stream (measurement aid for
 * bench.py's roofline leg; off by default, adds two event records per launch when on). */
int dfm_profile_enable(dfm_handle* h, int on);
int dfm_profile_query(dfm_handle* h, const char* kernel_name /*NULL = all*/, double* ms, long long* count);
int dfm_profile_reset(dfm_handle* h);
const char* dfm_profile_kernel_name(dfm_handle* h, int i);

/* ---- a2: standardize_data, dfm_functions.ipynb:501-509 ------------------------------- */
/* Xs = (X - mean)/std per column over non-missing entries, population std. */
int dfm_standardize(dfm_handle* h, const double* X, int T, int N, int batch, int mem,
                    double* Xs /*T x N*/, double* xmean /*N*/, double* xstd /*N*/);

/* ---- a4: pca_score, dfm_functions.ipynb:179-183 --------------------------------------- */
/* score = X V[:, 1:r] (principal-component scores of a balanced T x N block).  Column signs
 * are fixed by: the entry of largest magnitude of each right singular vector is positive
 * (LAPACK's signs, which the reference inherits, are arbitrary). */
int dfm_pca_score(dfm_handle* h, const double* X, int T, int N, int r, int batch, int mem,
                  double* score /*T x r*/);

/* ---- a7: estimate_factor!, dfm_functions.ipynb:328-382 -------------------------------- */
typedef struct {
  int T, N, r;              /* estimation block: rows initperiod..lastperiod, columns inclcode==1; r = nfac_u (nfac_o = 0) */
  int nt_min;               /* m.nt_min_factor_estimation  (:357, :375) */
  double tol;               /* m.tol; stop when |dSSR| < tol*T*N  (:368) */
  long long max_iter;       /* :328 default 100000000 */
  int compute_r2;           /* computeR2 (:329) */
  int n_constr;             /* rows of the stacked LambdaConstraint (:1063-1068); 0 = none */
  const int* constr_index;  /* [n_constr] 0-based series index of each row */
  const double* constr_R;   /* [n_constr x r] column-major */
  const double* constr_r;   /* [n_constr] UNstandardized r; divided by xstd internally (:1182-1186) */
  int batch;
  int mem;
} dfm_factor_opts;

typedef struct {
  double ssr, tss;          /* m.fes.ssr, m.fes.tss */
  long long nobs;           /* m.fes.nobs */
  int iters;                /* ALS sweeps executed (the reference is silent about this) */
  int status;               /* DFM_OK, DFM_ERR_NOT_PD, DFM_ERR_NOT_CONVERGED (hit max_iter), DFM_ERR_TOO_FEW_OBS */
} dfm_factor_stats;

/* X: T x N raw (unstandardized) estimation block with NaN.  F_init: optional T x r starting
 * factors (NULL = PCA of the balanced sub-panel as the reference does, :345-348).  r <= 64 with
 * F_init, r <= 48 with the PCA start (DFM_ERR_UNSUPPORTED past that).
 * Outputs (any may be NULL): F T x r (= m.factor[initperiod:lastperiod,:]); Lambda N x r in
 * standardized units (the loop-local `lambda` of :351, NaN rows for series with < nt_min obs);
 * R2 N (m.fes.R2, NaN = missing); xmean, xstd N; stats [batch]. */
int dfm_estimate_factor(dfm_handle* h, const double* X, const dfm_factor_opts* opts,
                        const double* F_init, double* F, double* Lambda, double* R2,
                        double* xmean, double* xstd, dfm_factor_stats* stats);

/* ---- a9: estimate_factor_loading! (+ uar, lagmat, compute_r2), :391-415, :295-311, :565-569 */
typedef struct {
  int T, ns, r;             /* rows initperiod..lastperiod of ALL ns series */
  int nt_min;               /* m.nt_min_factorloading_estimation */
  int n_uarlag;             /* m.n_uarlag */
  int n_constr; const int* constr_index; const double* constr_R; const double* constr_r; /* :loading constraints */
  int batch;
  int mem;
} dfm_loading_opts;
/* data T x ns (raw units, NaN), F T x r (NaN = missing).  Each series is fitted on the rows where it and
 * every factor are observed (drop_missing_row, :396).  Outputs: lambda ns x r, r2 ns, uar_coef ns x n_uarlag,
 * uar_ser ns.  Series with < nt_min usable rows get NaN (the reference leaves them undefined). */
int dfm_estimate_loading(dfm_handle* h, const double* data, const double* F, const dfm_loading_opts* opts,
                         double* lambda, double* r2, double* uar_coef, double* uar_ser);
/* Same regression, plus what the reference keeps in locals: `constant` ns (the intercept b[end] of :399-401) and
 * `resid` T x ns (the residuals `ehat` of :400, NaN where the observation is missing or the series was not fitted) --
 * amengual_watson_test (:741-752) residualises the panel with exactly this regression.  `status` (HOST int[batch], may
 * be NULL): 0, or DFM_ERR_NOT_PD if some series' regression / constraint / AR step was singular (those series are NaN).
 * constant / resid / status may be NULL. */
int dfm_estimate_loading_ex(dfm_handle* h, const double* data, const double* F, const dfm_loading_opts* opts,
                            double* lambda, double* r2, double* uar_coef, double* uar_ser, double* constant,
                            double* resid, int* status);

/* ---- a10: estimate_var! + fill_matrices!, :444-492 ------------------------------------ */
/* F: T x r (rows initperiod..lastperiod; NaN = missing).  K = r*p + withconst.  As estimate_var! does through
 * ols_skipmissing(..., Balanced()) (:242-252, :452), every row t whose y_t or one of its p lags is missing is dropped;
 * T_used = number of rows kept.
 * betahat K x r; resid T x r (NaN on dropped rows, incl. the first p); seps r x r (= e'e/(T_used-K)); M k x k, Q r x k,
 * G k x r with chol(seps) lower in its top block (k = r*p).  Any output may be NULL.
 * A panel that cannot be fitted (T_used <= K, singular regression, seps not PD) has NaN in all of its outputs; the call
 * returns that panel's error code when batch == 1 or when NO panel of the batch could be fitted, DFM_OK otherwise. */
int dfm_estimate_var(dfm_handle* h, const double* F, int T, int r, int p, int withconst, int batch, int mem,
                     double* betahat, double* resid, double* seps, double* M, double* Q, double* G);

/* ---- f4: instability tests of the loadings: compute_chow / compute_qlr / regress_hac / hac / form_hscrc (dfm_functions.ipynb)
 * and the per-series loop of Stock_Watson.ipynb Table 4(a) ------------------------------------------------------------- */
/* For every series i of data (T x ns column-major, NaN = missing): rows with a missing y or factor are dropped
 * (drop_missing_row([y X])); chow[i] = Wald statistic of the break-dummy interactions in the regression of y on
 * [F, F .* D] with Bartlett HAC(q) covariance, D = 1 after the first T_break kept rows (the notebook applies the row number
 * of the break date to the rows that survive the drop); qlr[i] = max of that statistic over the break rows
 * floor(ccut Td) .. Td - floor(ccut Td); qlr0 (may be NULL) the same with q = 0.  NaN where y has fewer than min_obs
 * observations before or after row T_break.  status (may be NULL): 3 where a covariance was not positive definite. */
int dfm_instability(dfm_handle* h, const double* data, const double* F, int T, int ns, int r, int q, int T_break, double ccut,
                    int min_obs, int mem, double* chow /*ns*/, double* qlr /*ns*/, double* qlr0 /*ns or NULL*/, int* status /*ns or NULL*/);

/* Second half of the Table 4(a) loop: cor[i] = correlation between the fitted values of series i on F (full-sample factors)
 * and on F_alt (factors of another sample; NaN rows outside it), each from ols_skipmissing(y, X, Balanced()) without
 * intercept, over the rows where both fitted values exist.  Same min_obs rule (NaN otherwise). */
int dfm_fit_correlation(dfm_handle* h, const double* data, const double* F, const double* F_alt, int T, int ns, int r, int T_break,
                        int min_obs, int mem, double* cor /*ns*/, int* status /*ns or NULL*/);

/* ---- a11: impulse_response / compute_irf_single_shock!, :793-825 ----------------------- */
/* irf[:, h, j] = Q M^h G[:, shock_ids[j]],  h = 0..H-1;  irf is r x H x n_shock column-major. */
int dfm_irf(dfm_handle* h, const double* M, const double* Q, const double* G, int k, int r, int H,
            int n_shock, const int* shock_ids /*host, 0-based*/, int batch, int mem, double* irf);

/* ---- a': estimate!(m, ::Parametric) -- the slot declared at dfm_functions.ipynb:23 ----- */
/* Gaussian state-space EM; NO reference implementation exists (spec = oracle/kalman_em.py).
 *   z_t = M z_{t-1} + [eta_t;0], eta~N(0,Q), z_t = [f_t..f_{t-p+1}], M = companion(A) (the
 *   reference's own companion form :477-492);  x_t = Lam f_t + e_t, e~N(0,diag R);  z_1~N(0,P0).
 * One EM iteration = E-step (Kalman filter + RTS smoother incl. lag-one covariances, update in
 * information form) + M-step (Lam, R, A, Q; P0 held fixed). */
typedef struct {
  int T, N, r, p;
  int max_iter;             /* iterations are E+M; */
  double tol;               /* stop after iteration j>=2 when |ll_j-ll_{j-1}| <= tol*(|ll_j|+|ll_{j-1}|)/2 ; 0 = run max_iter */
  int batch;
  int mem;
  int path;                 /* 0 = auto, 1 = general multi-kernel path, 2 = fused per-panel kernel (LDG->DMMA), 3 = fused per-panel kernel with TMA bulk-copy ring (needs even T) */
} dfm_em_opts;

typedef struct {            /* initial parameters; all column-major, per panel back to back */
  const double* Lam;        /* N x r (NaN row = series excluded) */
  const double* R;          /* N */
  const double* A;          /* r x k, k = r*p  ([A_1 ... A_p]) */
  const double* Q;          /* r x r */
  const double* P0;         /* k x k or NULL => stationary covariance of the initial (A,Q) by Lyapunov doubling */
} dfm_em_init;

typedef struct {            /* outputs; any pointer may be NULL */
  double* Lam; double* R; double* A; double* Q; double* P0;   /* parameters after the last M-step (P0 as used) */
  double* F;                /* T x r   smoothed factors E[f_t | x_1..T] of the last E-step */
  double* PF;               /* r x r x T  smoothed covariances Var[f_t | x_1..T] */
  double* loglik;           /* max_iter per panel: loglik[j] = log-likelihood of the parameters entering iteration j (NaN beyond iters) */
  int* iters;               /* [batch] */
  int* status;              /* [batch] */
} dfm_em_out;

/* X: T x N STANDARDIZED panel (NaN = missing), e.g. dfm_standardize output; batch panels back to back.
 * Synchronous: results are in `out` on return.  With DFM_MEM_HOST and a batch larger than the number of panels the
 * fused kernel keeps resident (296 on a B200 for C2-shaped panels) the upload, the EM iterations and the download
 * overlap inside the call (one kernel launch that starts before the data has arrived; see DESIGN.md 4.4) -- pinned
 * host buffers make the copies truly asynchronous, pageable ones work but are staged by the CUDA runtime. */
int dfm_em_kalman(dfm_handle* h, const double* X, const dfm_em_opts* opts, const dfm_em_init* init,
                  const dfm_em_out* out);

/* ---- a'': smoothing, nowcasting and forecasting with a fitted state-space model --------- */
/* The model of dfm_em_kalman at GIVEN parameters (no M-step): one Kalman filter + RTS smoother pass over the panel and H
 * periods after it.  A forecast period is one in which no series is observed, so the same pass gives the smoothed
 * factors of t <= T (the ragged edge included), the forecasts of t > T, and E[x_it | data] for every missing cell. */
typedef struct {
  int T, N, r, p;             /* in-sample panel T x N, STANDARDIZED, NaN = missing (as dfm_em_kalman) */
  int H;                      /* periods T+1 .. T+H to forecast; 0 = smoothing only */
  int batch, mem;
} dfm_ss_opts;

typedef struct {              /* any pointer may be NULL (not computed); per panel back to back; all column-major */
  double* F;                  /* (T+H) x r        E[f_t | observed x]  (forecasts for t > T) */
  double* PF;                 /* r x r x (T+H)    Var[f_t | observed x] */
  double* common;             /* (T+H) x N        lambda_i' E[f_t | x]  (compute_series, dfm_functions.ipynb:552) */
  double* xhat;               /* (T+H) x N        E[x_it | x]: x_it where observed, common_it otherwise */
  double* xvar;               /* (T+H) x N        Var[x_it | x]: 0 where observed, lambda_i' PF_t lambda_i + R_i otherwise */
  double* loglik;             /* [batch]          log-likelihood of the observed cells */
  int* status;                /* [batch]          0, or DFM_ERR_NOT_PD (a covariance not positive definite or R_i <= 0: that
                                                   panel's outputs are NaN) */
} dfm_ss_out;

/* X: T x N standardized panels back to back; params: (Lam, R, A, Q) per panel as dfm_em_kalman's initial parameters,
 * P0 == NULL => the same stationary prior by Lyapunov doubling.  A series whose Lambda row or R_i is NaN is out of the
 * model: its columns of common / xhat / xvar are NaN.  Size limits and error codes as dfm_em_kalman's general path
 * (k = r*p <= 48); H < 0 is DFM_ERR_ARG.  The parameter arrays are only read.  Synchronous for host memory. */
int dfm_kalman_smooth(dfm_handle* h, const double* X, const dfm_ss_opts* opts, const dfm_em_init* params, const dfm_ss_out* out);

/* ---- simulation smoother: draws from the JOINT posterior of the factor path and the missing cells ---------------------
 * dfm_kalman_smooth gives marginals (one period, one cell at a time).  This call draws (f_1 .. f_{T+H}, x_missing) given the
 * observed cells at fixed parameters, so that any function of a path -- a 4-quarter growth rate, an annual average, the
 * probability of staying below a threshold, a ratio of imputed cells -- gets its posterior distribution from the draws; one
 * draw per sweep is also the factor step of a Gibbs sampler.  Mean-corrected simulation smoother (Durbin & Koopman 2002) on
 * the E-step of dfm_kalman_smooth; a draw costs O((T+H) k^2) whatever N (the spec is tests/simsmooth_oracle.py).
 * Random numbers: the Philox4x32-10 stream of the replication generators (below) with replication id = draw id and four
 * streams (element indices; Tp = T + H, k = r p):
 *    7  z+_0 = L_P0 nu                                  element a        (a < k)
 *    8  state shocks eta_t of periods t >= 1            element t r + a  (a < r)
 *    9  xi_t, the N(0, C_t) term of the observations    element t r + a  (a < r)
 *   10  eps_it, the idiosyncratic draw of a missing cell element i Tp + t (drawn for missing cells only)
 * Draw j of a call is draw id draw0 + j, a pure function of (seed, draw id): any split of a draw range over calls or GPUs
 * (dfm_shard_range) gives bit-identical draws.  oracle/dgp.py restates the stream; tests/simsmooth_oracle.py the four tags. */
typedef struct {
  int T, N, r, p;             /* in-sample panel T x N, STANDARDIZED, NaN = missing (as dfm_kalman_smooth); ONE model per call */
  int H;                      /* periods T+1 .. T+H after the panel */
  long long n_draw;           /* >= 1 */
  long long draw0;            /* draw id of the first draw, >= 0 */
  unsigned long long seed;
  int mem;
} dfm_sim_opts;

typedef struct {              /* any of F / X may be NULL (not computed); all column-major, draw after draw */
  double* F;                  /* n_draw x ((T+H) x r)   factor path draws f~_t */
  double* X;                  /* n_draw x ((T+H) x N)   panel draws: x_it where observed, lambda_i' f~_t + sqrt(R_i) eps_it where
                                                        missing (the H periods after the panel included), NaN columns for series
                                                        out of the model */
  int* status;                /* [1]  0, or DFM_ERR_NOT_PD (a covariance not positive definite or R_i <= 0: the draws are NaN) */
} dfm_sim_out;

/* X: T x N standardized panel; params: (Lam, R, A, Q[, P0]) of one model as dfm_kalman_smooth's.  Size limits and error codes
 * as dfm_kalman_smooth; n_draw < 1 or draw0 < 0 is DFM_ERR_ARG.  The device workspace does not grow with n_draw (the draws
 * are made in chunks).  Synchronous for host memory. */
int dfm_simulation_smoother(dfm_handle* h, const double* X, const dfm_sim_opts* opts, const dfm_em_init* params, const dfm_sim_out* out);

/* ---- news decomposition: why the nowcast moved between two data vintages -------------------------------------------------
 * At fixed parameters, the revision of a target y = x_{i*, t*} between an old vintage and a new one that only ADDS cells is
 * a sum over the released cells j (Banbura & Modugno 2014; Banbura, Giannone, Modugno & Reichlin 2013):
 *     E[y | new] - E[y | old] = sum_j w_j I_j,   I_j = x_j - E[x_j | old] (the news),   w = Cov(y, I | old) Var(I | old)^-1.
 * The weights come from the joint covariance of the factors of the periods that hold a news cell or a target (W of them)
 * given the old vintage, through a Woodbury solve of size W r (no n_news x n_news matrix); the spec is tests/news_oracle.py.
 * A target observed in the old vintage has revision 0 and weights 0; a released target has weight 1 on its own cell; a
 * target in a series out of the model (NaN loading or R) is NaN.  A new cell of a series out of the model is not news. */
typedef struct {
  int T, N, r, p, H;          /* as dfm_ss_opts; both panels STANDARDIZED with the same means / stds, NaN = missing */
  int news_rows;              /* news cells may lie only in rows T - news_rows .. T - 1 (the release window); 1 <= news_rows <= T */
  int n_target;               /* 1 .. 64 */
  const int* target_series;   /* HOST [n_target], 0-based column */
  const int* target_period;   /* HOST [n_target], 0-based row in 0 .. T+H-1 (rows >= T: forecasts) */
  int batch, mem;             /* batch = vintage pairs, each with its own parameters (as dfm_kalman_smooth) */
} dfm_news_opts;

typedef struct {              /* any pointer may be NULL (not computed); per pair back to back; column-major */
  double* old_est;            /* [n_target]                    E[y_q | old] (the data where y_q is observed in the old vintage) */
  double* new_est;            /* [n_target]                    old_est + the sum of the contributions (fixed summation order) */
  double* news;               /* news_rows x N                 I_j at the news cells, NaN elsewhere */
  double* weight;             /* news_rows x N x n_target      w_qj at the news cells, 0 elsewhere */
  double* contrib;            /* news_rows x N x n_target      w_qj I_j at the news cells, 0 elsewhere */
  int* status;                /* [batch]  0; DFM_ERR_NOT_PD (the E-step failed: a covariance not positive definite or
                                 R_i <= 0); DFM_ERR_ARG (this pair's vintages are inconsistent: an old cell missing or changed
                                 in the new one, or a new cell above the window).  A failed pair's outputs are NaN; the other
                                 pairs are unaffected. */
} dfm_news_out;

/* X_old, X_new: T x N standardized panels, pairs back to back; params: (Lam, R, A, Q[, P0]) per pair as dfm_kalman_smooth's.
 * Size limits as dfm_kalman_smooth.  W r <= 128, with W bounded by the number of distinct rows of the window and the target
 * periods (checked here, before any data is read; DFM_ERR_UNSUPPORTED past it).  Bad targets or options: DFM_ERR_ARG.
 * Synchronous for host memory. */
int dfm_news(dfm_handle* h, const double* X_old, const double* X_new, const dfm_news_opts* opts, const dfm_em_init* params,
             const dfm_news_out* out);

/* Initial (Lam, R, A, Q) for dfm_em_kalman from a standardized panel and factor estimates
 * (per-series OLS on F without constant, residual variance, VAR(p) without constant) --
 * the role uar_ser / fill_matrices! outputs would play (:405-412, :477-492). */
int dfm_em_init_from_factors(dfm_handle* h, const double* Xs, const double* F, int T, int N, int r, int p,
                             int batch, int mem, double* Lam, double* R, double* A, double* Q);

/* ---- K9 (SURVEY.md 2.3 / 8d): replication generators.  The reference has no Monte-Carlo / bootstrap / RNG code (its
 * notebook never draws a random number); SURVEY.md 8d freezes the definitions these entry points implement.  Draws come
 * from a counter-based Philox4x32-10 stream that is a pure function of (seed, replication id, stream, element): panel
 * `rep0 + b` is bit-identical whatever the batch split or the number of GPUs.  oracle/dgp.py restates the stream. */
/* Synthetic DGP (C2 / C3 / C5): Lam ~ N(0,1); f_t = diag(a) f_{t-1} + eta_t, a ~ U(.2,.8), burn-in 100; e_it ~ N(0, s2_i),
 * s2_i ~ U(.5,1.5); x = Lam f + e, column-standardised as standardize_data (:501-509).
 * X: batch panels T x N column-major; F_true (may be NULL): the simulated factors, T x r column-major per panel. */
int dfm_simulate_panels(dfm_handle* h, unsigned long long seed, long long rep0, int batch, int T, int N, int r, int mem,
                        double* X, double* F_true);

/* Residual bootstrap of a fitted non-parametric model (C4): resample the factor-VAR residuals (`varm.resid`, :464) with
 * replacement, rebuild f* through `betahat` (:463; the first p rows of the fitted factors start the recursion), draw the
 * idiosyncratic AR(n_uarlag) processes from (uar_coef, uar_ser) (:405-412) after `burn` periods, x* = Lam f* + u*, and
 * re-impose the NaN pattern of `data`.  Series whose lam row / uar_ser is NaN come back as NaN columns. */
typedef struct {
  int T, ns, r, p;          /* window length (rows initperiod..lastperiod), series, factors, VAR lags */
  int n_uarlag;             /* <= 16 */
  int n_resid;              /* rows of `resid` */
  int burn;                 /* burn-in periods of the idiosyncratic processes */
  int batch; int mem;
  unsigned long long seed; long long rep0;     /* replication ids rep0 .. rep0 + batch - 1 */
} dfm_boot_opts;
/* F0 T x r; resid n_resid x r; beta (1 + r p) x r = [const; lag 1; ...; lag p]; lam ns x r; uar_coef ns x n_uarlag;
 * uar_ser ns; data T x ns (only its NaN pattern is read); all column-major.  X: batch panels T x ns column-major. */
int dfm_bootstrap_panels(dfm_handle* h, const dfm_boot_opts* opts, const double* F0, const double* resid, const double* beta,
                         const double* lam, const double* uar_coef, const double* uar_ser, const double* data, double* X);

/* The whole C4 replication step in one call ("one panel + B bootstrap seeds", SURVEY.md 8b): dfm_bootstrap_panels ->
 * dfm_estimate_factor (standardise, PCA start, ALS with nt_min / tol as estimate_factor!) -> factor signs aligned with F0 ->
 * dfm_estimate_var (VAR(p) with constant) -> dfm_irf for all r shocks, device resident between the stages.  Inputs as
 * dfm_bootstrap_panels (pass the ESTIMATION series only: lam, uar_*, data restricted to inclcode == 1).
 * irf: batch records [shock j][horizon h][variable i] = r*H*r doubles each (NaN record = failed replication);
 * als_iters / als_status: HOST int[batch] or NULL.  Synchronous. */
int dfm_bootstrap_irf(dfm_handle* h, const dfm_boot_opts* opts, const double* F0, const double* resid, const double* beta,
                      const double* lam, const double* uar_coef, const double* uar_ser, const double* data, int nt_min,
                      double tol, int H, double* irf, int* als_iters, int* als_status);

/* ---- (f)3: percentile bands over the replication axis (the post-processing step behind impulse_response, :793-825).
 * recs: n x d ROW-major (one record of d statistics per replication, as gathered by dfm_allgather_results); q: nq
 * percentiles in [0, 100] (HOST array); out: nq x d row-major.  numpy.percentile's default (linear) interpolation; NaN
 * records (failed replications) are ignored.  n <= 16384. */
int dfm_percentiles(dfm_handle* h, const double* recs, long long n, int d, const double* q, int nq, int mem, double* out);

/* ---- (e): the single collective of the multi-GPU path ---------------------------------- */
/* AllGather `count` doubles per rank of per-replication result records (device pointers on the
 * handle's device) with ncclAllGather on the handle's stream.  `nccl_comm` is an ncclComm_t
 * created by the caller (NCCL.jl / torch).  libnccl is resolved with dlopen at first use. */
int dfm_allgather_results(dfm_handle* h, void* nccl_comm, const double* send, double* recv, long long count);

/* contiguous shard [begin,end) of `n_rep` replications for rank `rank` of `world` (host helper). */
int dfm_shard_range(long long n_rep, int rank, int world, long long* begin, long long* end);

#ifdef __cplusplus
}
#endif
#endif /* DFM_B200_H */
