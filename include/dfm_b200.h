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
/* irf[:, h, j] = Q M^h G[:, shock_ids[j]],  h = 0..H-1;  irf is r x H x n_shock column-major.
 * k <= 14076 (the two k-vectors of a shock live in shared memory); larger k: DFM_ERR_UNSUPPORTED. */
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

/* The same EM under linear restrictions on the loadings (the reference's LambdaConstraint, :1063-1186, e.g. the named-factor
 * normalisation of Stock & Watson's Figure 7): row q says  H[q,:] lam_{index[q]} = h[q].  Host arrays, STANDARDIZED units
 * (divide the reference's r by the series' xstd, as standardize_constraint! does); H is n_constr x r column-major.  The same
 * restriction applies to every panel of the batch.  The measurement M-step of a restricted series i (rows H_i, values h_i) is
 * the exact constrained maximiser
 *     lu = S_i^-1 s_i,  Y = S_i^-1 H_i',  G = H_i Y,  lam_i = lu - Y G^-1 (H_i lu - h_i),  R_i as the unrestricted formula
 * (S_i = sum_{t obs} E[f f'], s_i = sum_{t obs} x_it E[f]), so the log-likelihood stays monotone.  loglik[0] belongs to the
 * initial parameters as given (they may violate the restriction); from iteration 1 on the parameters satisfy it.
 *   constr == NULL or n_constr == 0: exactly dfm_em_kalman (same dispatch, same bits).
 *   With rows, the call always runs the general multi-kernel path (never the fused kernels or the streaming host path);
 *   opts->path 2 or 3 -> DFM_ERR_UNSUPPORTED.
 *   DFM_ERR_ARG: an index outside [0, N), more than r rows on one series, a non-finite H or h entry, a NULL array with
 *   n_constr > 0, n_constr < 0.
 *   Dependent rows on a series (singular G, relative Cholesky pivot <= 1e-12) -> that panel's status is DFM_ERR_NOT_PD, as a
 *   failed unrestricted solve.  Rows on a series out of the model (NaN Lam row or R) are ignored. */
typedef struct {
  int n_constr;             /* rows; 0 = none */
  const int* index;         /* [n_constr] 0-based series of each row */
  const double* H;          /* [n_constr x r] column-major */
  const double* h;          /* [n_constr] */
} dfm_lam_constr;

int dfm_em_kalman_constrained(dfm_handle* h, const double* X, const dfm_em_opts* opts, const dfm_em_init* init,
                              const dfm_lam_constr* constr, const dfm_em_out* out);

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

/* ---- parametric bootstrap of a fitted state-space model: bands with parameter uncertainty ------------------------------
 * Forecasts, posterior draws and news condition on the EM estimates theta^ = (Lam, R, A, Q).  This call draws B panels from
 * the model at theta^, re-runs the EM on all of them from theta^, brings every replicate back into the rotation of theta^
 * and returns its parameters, impulse responses and (optionally) forecasts, so that bands over the replicates carry the
 * estimation uncertainty of theta (the spec is tests/ss_bootstrap_oracle.py).
 * Panels (standardized model units, not re-standardized):  z_1 = L_P0 nu,  z_t = M z_{t-1} + [L_Q eta_t; 0],
 * x_it = lam_i' f_t + sqrt(R_i) eps_it where the template panel is observed, NaN where it is missing (the original missing
 * pattern and ragged edge) and in the columns of series out of the model (NaN Lam row or R_i).  L_P0, L_Q: lower Cholesky
 * factors, a pivot <= 1e-12 max diag counting as a zero column (the simulation smoother's rule).
 * Random numbers: the Philox4x32-10 stream of the replication generators with replication id = rep0 + b and three streams
 * (element indices; k = r p), after the simulation smoother's 7-10:
 *   11  nu, z_1 = L_P0 nu                              element a        (a < k)
 *   12  state shocks eta_t of periods t >= 1           element t r + a  (a < r)
 *   13  eps_it, the idiosyncratic draw of a cell        element i T + t  (drawn for cells the template observes)
 * so replicate b is a pure function of (seed, rep0 + b): any split of a replication range (dfm_shard_range) gives
 * bit-identical panels, and dfm_ss_bootstrap's replicate b re-estimates exactly dfm_ss_simulate_panels' panel b. */
/* X: T x N template (standardized; only its NaN pattern is read); params: (Lam, R, A, Q, P0) of ONE model, P0 required
 * (e.g. the EM's P0 output).  Xout: batch panels T x N column-major, replication ids rep0 .. rep0 + batch - 1.
 * k = r p > 48: DFM_ERR_UNSUPPORTED.  Synchronous for host memory. */
int dfm_ss_simulate_panels(dfm_handle* h, const double* X, int T, int N, int r, int p, const dfm_em_init* params, unsigned long long seed,
                           long long rep0, int batch, int mem, double* Xout);

typedef struct {
  int T, N, r, p;             /* the fitted model's panel T x N (STANDARDIZED, NaN = missing) and state shape */
  int H_irf;                  /* > 0: impulse-response horizons 0 .. H_irf - 1 */
  int H_fc;                   /* >= 0: periods after the panel for the forecasts */
  int fc_rows;                /* 0 .. T + H_fc: trailing rows of the padded (T + H_fc) x N forecast panel returned per replicate
                                 (so that the ragged edge can be included); 0 = no forecasts */
  int max_iter; double tol;   /* EM of every replicate, as dfm_em_opts (tol = 0: run max_iter iterations) */
  long long n_rep;            /* >= 1 replicates */
  long long rep0;             /* replication id of the first replicate, >= 0 */
  unsigned long long seed;
  int mem;
} dfm_ssb_opts;

typedef struct {              /* any pointer may be NULL (not computed / not returned); per replicate back to back; column-major */
  double* Lam;                /* N x r     aligned loadings (NaN rows for series out of the model) */
  double* R;                  /* N         idiosyncratic variances */
  double* A;                  /* r x k     aligned [A_1 .. A_p] */
  double* Q;                  /* r x r     aligned state-shock covariance */
  double* irf;                /* r x H_irf x r records [shock j][horizon h][variable i] as dfm_bootstrap_irf's: Q M^h G e_j with
                                 G = [chol(Q~); 0] (orthogonalized shocks of the aligned model) */
  double* xhat;               /* fc_rows x N   E[x_it | data] at the replicate's parameters (last fc_rows rows of T + H_fc) */
  double* xvar;               /* fc_rows x N   Var[x_it | data] at the replicate's parameters */
  double* loglik;             /* [n_rep]   log-likelihood of the parameters entering the replicate's last EM iteration */
  int* iters;                 /* [n_rep]   EM iterations */
  int* status;                /* [n_rep]   0; the EM status when not 0; DFM_ERR_NOT_PD when the alignment fails (Lam*' W Lam* or
                                 X singular, or Q~ not positive definite; see DESIGN.md 4.9).  A failed replicate has NaN
                                 parameters, impulse responses and forecasts; loglik / iters stay the EM's. */
} dfm_ssb_out;

/* Alignment (rotation f -> K f of the EM estimates Lam*, R*, A*, Q* onto theta^), W = diag(1 / R^_i) over the series in the model:
 *   X = (Lam*' W Lam*)^-1 Lam*' W Lam^,  K = X^-1,  Lam~ = Lam* X,  A~_l = K A*_l X,  Q~ = K Q* K',  R~ = R*.
 * X: T x N standardized panel of the fitted model; params: theta^ (Lam, R, A, Q, P0), P0 required (the EM holds it fixed; every
 * replicate's EM starts from theta^ with it).  Balanced panels with p = 1, r <= 8 and even T re-estimate on dfm_em_kalman's
 * fused path, everything else on its general path.  Bad shapes / options (H_irf <= 0, n_rep < 1, fc_rows > T + H_fc, ...):
 * DFM_ERR_ARG; k = r p > 48: DFM_ERR_UNSUPPORTED; per-replicate failures go to status only.  The replicates run in
 * sub-batches whose size depends only on (T, N, r, p) and the device (the last one filled up with the following replication
 * ids, whose results are discarded), so the device memory of a call does not grow with n_rep and replicate rep0 + b has the
 * same bits whatever n_rep, the shard split or the number of calls.  Synchronous. */
int dfm_ss_bootstrap(dfm_handle* h, const double* X, const dfm_ssb_opts* opts, const dfm_em_init* params, const dfm_ssb_out* out);

/* ---- Bayesian estimation of the state-space model: batched Gibbs chains ----------------------------------------------
 * The model of dfm_em_kalman (standardized panel, NaN = missing, P0 HELD FIXED) with a conjugate proper prior, standardized units:
 *   lam_i | R_i ~ N(0, (R_i / kap_lam) I_r),  R_i ~ IG(a_R, b_R);   A' | Q ~ MN(0, I_k / kap_A, Q),  Q ~ IW(nu_Q, s_Q I_r).
 * Sweep s of chain c at theta = (Lam, R, A, Q), id = gibbs_id(c, s) = c 2^24 + s, Tp = T + H_fc (the spec is tests/gibbs_oracle.py):
 *   1. factor step: (z~_0 .. z~_{Tp-1}, x~_missing) exactly as dfm_simulation_smoother's draw `id` at theta;
 *   2. per series in the model, over its observed in-sample periods: L_i = chol(kap_lam I + S_i), m_i = L_i^-T L_i^-1 s_i,
 *      R_i = (b_R + (q_i - s_i' m_i) / 2) / Gamma(a_R + n_i / 2),  lam_i = m_i + sqrt(R_i) L_i^-T nu_i
 *      (S_i = sum f~ f~', s_i = sum x f~, q_i = sum x^2);  series out of the model (NaN Lam row or R_i) stay NaN;
 *   3. regression of f~_t on z~_{t-1}, t = 1 .. T-1 (the lag block of z~_0 gives the pre-sample lags):
 *      Q ~ IW(nu_Q + T - 1, s_Q I + Y'Y - B^' Z'Y) by Bartlett,  A' = B^ + L_Z^-T Xi L_Q',  B^ = (kap_A I + Z'Z)^-1 Z'Y;
 *   4. the forecast periods t >= T are drawn in step 1 for the predictive output only.
 * Draws of A are kept as drawn (no stationarity restriction).
 * Random numbers: the Philox4x32-10 stream with replication id gibbs_id(c, s); the factor step uses the simulation smoother's
 * tags 7-10 unchanged, the parameter step (element indices; Gamma number e = i for R_i, N + j for the Bartlett diagonal B_jj):
 *   14  nu_i                                       element i r + a          (a < r)
 *   15  Bartlett B_ij (i > j), then Xi (k x r)     element i + r j;  r^2 + a + k b
 *   16  normals of the Gamma sampler               element 64 e + j         (attempt j < 64 of Gamma number e)
 *   17  uniforms of the Gamma sampler              element 64 e + j
 * Gamma(alpha >= 1) is Marsaglia & Tsang; if all 64 attempts of a number are rejected (probability < 1e-80) it is d = alpha - 1/3.
 * Chain c is a pure function of (seed, c, its initial theta, sweep0). */
typedef struct {
  double kap_lam, a_R, b_R;   /* loadings / idiosyncratic variances: kap_lam > 0, a_R >= 1, b_R > 0 */
  double kap_A, nu_Q, s_Q;    /* transition: kap_A > 0, s_Q > 0, nu_Q + T - r >= 2 */
} dfm_gibbs_prior;

typedef struct {
  int T, N, r, p;             /* panel T x N (STANDARDIZED, NaN = missing) and state shape, k = r p <= 48 */
  int H_irf;                  /* >= 0: impulse-response horizons 0 .. H_irf - 1 (0 = none) */
  int H_fc;                   /* >= 0: periods after the panel drawn for the predictive panel */
  int fc_rows;                /* 0 .. T + H_fc: trailing rows of the (T + H_fc) x N predictive panel returned per kept draw */
  int n_chain;                /* >= 1 */
  long long chain0;           /* chain id of the first chain; chain ids < 2^16 */
  long long sweep0;           /* index of the first sweep; sweep indices < 2^24 */
  int n_burn, n_keep, thin;   /* >= 0, >= 1, >= 1: n_sweep = n_burn + n_keep thin per chain */
  unsigned long long seed;
  int mem;
  dfm_gibbs_prior prior;
} dfm_gibbs_opts;

typedef struct {              /* any pointer may be NULL; per chain back to back (chain-major, then kept draw); column-major */
  double* Lam;                /* n_keep x (N x r)      kept draws (NaN rows for series out of the model) */
  double* R;                  /* n_keep x N */
  double* A;                  /* n_keep x (r x k) */
  double* Q;                  /* n_keep x (r x r) */
  double* irf;                /* n_keep x (r x H_irf x r)  records [shock][horizon][variable] of dfm_irf at the draw aligned onto ref
                                 (dfm_ss_bootstrap's rotation and G = [chol(Q~); 0]); NaN where the alignment fails */
  double* F;                  /* n_keep x (Tp x r)     factor path of the kept sweep */
  double* X;                  /* n_keep x (fc_rows x N) predictive panel of the kept sweep (last fc_rows rows of Tp): the data where
                                 observed, lam_i' f~_t + sqrt(R_i) eps_it where missing or after the panel (at the theta entering
                                 the sweep, as the factor draw), NaN for series out of the model */
  double* loglik;             /* n_sweep               log-likelihood of the parameters entering each sweep */
  int* status;                /* [n_chain] 0, or 3: an E-step failed or a P_{t+1|t} or Cholesky factor was not positive definite
                                 (the chain's records from that sweep on are NaN) */
} dfm_gibbs_out;

/* X: T x N standardized panel; init: (Lam, R, A, Q, P0) of every chain, back to back (P0 required, e.g. the EM's); ref: theta^
 * (Lam, R, A, Q) that the impulse responses are aligned onto (may be NULL when H_irf = 0).  Kept draw j of a chain is the state
 * after sweep sweep0 + n_burn + (j + 1) thin - 1, so a call with init = the last kept draw and sweep0 advanced by n_sweep
 * continues the chains.  The chains run in sub-batches whose size depends only on (T, N, r, p) and the device (the last one
 * filled with the chain ids that follow, started from copies of the last chain's init, their results discarded): chain c has
 * the same bits whatever n_chain, chain0 or the shard split, and the device memory does not grow with n_chain, n_keep or the
 * number of sweeps.  Bad options: DFM_ERR_ARG; k > 48: DFM_ERR_UNSUPPORTED.  Synchronous. */
int dfm_gibbs(dfm_handle* h, const double* X, const dfm_gibbs_opts* opts, const dfm_em_init* init, const dfm_em_init* ref,
              const dfm_gibbs_out* out);

/* The same sampler under linear restrictions on the loadings (dfm_lam_constr, STANDARDIZED units, as dfm_em_kalman_constrained),
 * e.g. the named-factor normalisation of Stock & Watson's Figure 7.  For a restricted series i (rows H_i, values h_i, m_i <= r)
 * the prior on lam_i is N(0, R_i / kap_lam I) CONDITIONED on H_i lam_i = h_i, so its conditional posterior is exact: with
 * S~ = kap_lam I + S_i (L_i = chol(S~)), Y = S~^-1 H_i', G = H_i Y, m_i = S~^-1 s_i,
 *     lam*_i = m_i - Y G^-1 (H_i m_i - h_i)                      (the EM's correction, S~ in place of S)
 *     R_i    = (b_R + (q_i - 2 s_i' lam*_i + lam*_i' S~ lam*_i - kap_lam h_i' (H_i H_i')^-1 h_i) / 2) / Gamma(a_R + n_i / 2)
 *     lam_i  = the same correction applied to the unrestricted draw m_i + sqrt(R_i) L_i^-T nu_i
 * (the r - m_i free dimensions cancel from the shape).  A restricted series uses the unrestricted series' random numbers (tag
 * 14 elements i r + a, Gamma number i); unrestricted series, the factor step and the transition step are unchanged.
 *   constr == NULL or n_constr == 0: exactly dfm_gibbs (same bits).
 *   DFM_ERR_ARG: the restriction errors of dfm_em_kalman_constrained, and out->irf != NULL with rows (the rotation onto ref
 *   would rotate the draws off the restriction).  Rows on a series out of the model are ignored.  Dependent rows on a series
 *   (relative pivot of G <= 1e-12) give that chain status 3. */
int dfm_gibbs_constrained(dfm_handle* h, const double* X, const dfm_gibbs_opts* opts, const dfm_em_init* init, const dfm_em_init* ref,
                          const dfm_lam_constr* constr, const dfm_gibbs_out* out);

/* ---- series responses and forecast-error variance decompositions of many models --------------------------------------
 * models: n_model models (Lam N x r, R N, A r x k, Q r x r; P0 unused) back to back as dfm_em_init's batch layout, k = r p.
 * Per model, L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L (h = 0 .. H-1, M the companion matrix of A), c_{i,h} = lam_i' Psi_h (1 x r):
 *   resp[i,h,j] = scale_i c_{i,h,j}                                           (n_shock = r: api.series_irf)
 *   fevd[i,h,j] = sum_{l<=h} c_{i,l,j}^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i)    (share of the (h+1)-step forecast-error variance of
 *                                                                             x_i due to shock j, idiosyncratic part included)
 * for the leading n_shock shocks (1 <= n_shock <= r); outputs N x H x n_shock per model, column-major, either may be NULL.
 * scale: N (e.g. xstd; NULL = 1).  Series out of the model (NaN Lam row or R_i) get NaN columns.  status [n_model] (may be
 * NULL): 0, or DFM_ERR_NOT_PD when Q is not positive definite or A / Q hold a NaN (a failed chain): that model's outputs are
 * NaN.  All arrays in `mem`.  r <= 64; bad arguments: DFM_ERR_ARG; r p > 14076 (dfm_irf's bound): DFM_ERR_UNSUPPORTED.
 * Synchronous for host memory. */
int dfm_series_responses(dfm_handle* h, const dfm_em_init* models, int N, int r, int p, int n_model, int H, int n_shock,
                         const double* scale, int mem, double* resp, double* fevd, int* status);

/* ---- historical decompositions of many models -------------------------------------------------------------------------
 * models: n_model models (Lam N x r, R N, A = [A_1 .. A_p] r x k, Q r x r; P0 unused) back to back as dfm_em_init's batch
 * layout, k = r p; F: n_model factor paths f_0 .. f_{Tp-1} (Tp x r each), path b belonging to model b.  Per model, L = chol(Q)
 * (lower), M the companion matrix of A, Psi_h = [M^h]_{1:r,1:r} L (as dfm_series_responses):
 *   structural shocks   eps_t = L^-1 (f_t - sum_{l=1..p} A_l f_{t-l})  for t >= p, NaN for t < p;
 *   base row t0 (p - 1 <= t0 < Tp): z_t0 = [f_t0; ..; f_{t0-p+1}] lies inside the path (no pre-sample lags);
 *   for t > t0:  contrib[i,t,j] = scale_i lam_i' sum_{s=t0+1..t} Psi_{t-s} e_j eps_{j,s}   (the leading n_shock shocks j)
 *                rest[i,t]      = the same sum over the shocks j >= n_shock
 *                base[i,t]      = scale_i lam_i' [M^{t-t0} z_t0]_{1:r}
 *   for t <= t0: contrib = rest = 0, base = scale_i lam_i' f_t;
 * so base + sum_j contrib + rest = scale_i lam_i' f_t (the common component) at every row.  Series out of the model (NaN Lam
 * row or R_i; R is read for that test only) get NaN columns.  status [n_model]: 0, or DFM_ERR_NOT_PD when A or Q holds a NaN,
 * Q is not positive definite or the path holds a NaN (a failed chain): that model's outputs are NaN, the others unaffected.
 * Identification: under f -> K f with K's first row e_1' (the rotations a restriction naming factor 1 leaves free), eps_1,
 * contrib[..., 0], rest (n_shock = 1) and base do not change; the other shocks' columns do, their sum does not.
 * Everything column-major, models back to back, in `mem`; the models run in chunks of a size fixed by the shapes (device
 * memory does not grow with n_model; model b has the same bits whatever n_model).  Bad arguments (a NULL required pointer,
 * t0 outside [p - 1, Tp), n_shock outside [1, r], a bad mem): DFM_ERR_ARG; k > 48: DFM_ERR_UNSUPPORTED.  Synchronous for host
 * memory. */
typedef struct { int N, r, p, Tp, t0, n_shock, n_model, mem; } dfm_hd_opts;
typedef struct {
  double* shocks;             /* n_model x (Tp x r)              eps */
  double* contrib;            /* n_model x (N x Tp x n_shock) */
  double* rest;               /* n_model x (N x Tp) */
  double* base;               /* n_model x (N x Tp) */
  int* status;                /* [n_model] */
} dfm_hd_out;                 /* any may be NULL */
int dfm_historical_decomposition(dfm_handle* h, const dfm_em_init* models, const double* F, const double* scale,
                                 const dfm_hd_opts* opts, const dfm_hd_out* out);

/* ---- shocks identified by sign restrictions on series responses ------------------------------------------------------
 * models: n_model models (Lam N x r, R N, A r x k, Q r x r; P0 unused) as dfm_series_responses, k = r p; ids: HOST array of
 * n_model model ids < 2^40 (NULL = 0 .. n_model-1; the Gibbs path passes gibbs_id(chain, sweep)); scale: N in `mem` (NULL = 1).
 * Per model b, L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L and c_{i,h} = lam_i' Psi_h (1 x r), as dfm_series_responses.
 *   Rows rho = (series i, horizon h, shock j, sign s): 0 <= i < N, 0 <= h < H, 1 <= j <= n_shock, s = +1 or -1 (a horizon
 *   range is several rows).
 *   Candidate c (0 <= c < n_rot): Z r x r, Z[a, j] = normal number c r^2 + a + r j of the Philox stream of id_b, tag 18;
 *   Omega = Q_Z diag(sign(diag R_Z)) from the QR of Z (Haar distributed; column j depends on Z's columns 0..j only).
 *   Acceptance: for each shock j with rows, v_rho = s_rho c_{i_rho,h_rho} omega_j over its rows; all v > 0: kept; all v < 0:
 *   omega_j -> -omega_j and kept; otherwise the candidate is rejected (strict inequalities).  Shocks without rows are kept as
 *   drawn.
 * Outputs per model (any pointer may be NULL; in `mem`, models back to back, column-major):
 *   n_accept [n_model]                  accepted candidates among the n_rot;
 *   cand     [n_model x n_keep]         the first n_keep accepted candidates in candidate order, -1 for an empty slot;
 *   rot      n_keep x (r x r)           their Omega (flips applied);
 *   resp     n_keep x (N x H x n_shock) scale_i c_{i,h} Omega e_j;
 *   fevd     n_keep x (N x H x n_shock) sum_{l<=h} (c_{i,l} Omega e_j)^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i) (dfm_series_responses on
 *                                       the records Psi_h Omega; the denominator does not depend on Omega);
 *   status   [n_model]                  0; DFM_ERR_NOT_PD when A or Q holds a NaN or Q is not positive definite; DFM_ERR_ARG when a
 *                                       restricted series is out of the model (NaN loading row or R_i).  Such a model accepts
 *                                       nothing; its neighbours are unaffected.
 * Empty slots have NaN rot, resp and fevd; series out of the model NaN resp and fevd columns.  Under f -> K f the accepted set
 * of series responses does not change (DESIGN.md 4.14).  The models run in chunks and the candidates in batches whose sizes
 * depend only on the shapes: device memory grows with neither n_model nor n_rot, and model b has the same bits whatever
 * n_model.  Bounds: r <= 16 (the candidates' columns live in shared memory), n <= 256 rows, k <= 48, n_keep <= 65535:
 * DFM_ERR_UNSUPPORTED past them.  Bad arguments (a NULL required pointer, a row outside its range, n_shock outside [1, r],
 * n_rot < 1, n_keep < 1, an id >= 2^40, a bad mem): DFM_ERR_ARG.  Synchronous for host memory. */
typedef struct {
  int N, r, p, n_model, H, n_shock;
  long long n_rot;            /* candidates per model, >= 1 */
  int n_keep;                 /* kept slots per model, >= 1 */
  unsigned long long seed;
  int mem;
} dfm_sign_opts;
typedef struct {
  int n;                      /* rows, 0 .. 256; HOST arrays of n (NULL when n = 0) */
  const int* series;          /* 0-based series i */
  const int* horizon;         /* 0 .. H-1 */
  const int* shock;           /* 1 .. n_shock */
  const int* sign;            /* +1 or -1 */
} dfm_sign_restr;
typedef struct {
  long long* n_accept;
  long long* cand;
  double* rot;
  double* resp;
  double* fevd;
  int* status;
} dfm_sign_out;
int dfm_sign_restrictions(dfm_handle* h, const dfm_em_init* models, const unsigned long long* ids, const double* scale,
                          const dfm_sign_opts* opts, const dfm_sign_restr* restr, const dfm_sign_out* out);

/* ---- narrative sign restrictions (Antolin-Diaz & Rubio-Ramirez 2018) --------------------------------------------------
 * dfm_sign_restrictions with statements about dated episodes added, and the importance weight of every kept draw.  models, ids,
 * scale, restr and the candidates (tag 18, the same ids and Omega) as dfm_sign_restrictions; F: n_model factor paths f_0 ..
 * f_{Tp-1} (Tp x r each, column-major, in `mem`).  Per model, with L = chol(Q), Psi_h and c_{i,h} = lam_i' Psi_h as there:
 *   u_t = L^-1 (f_t - sum_{l=1..p} A_l f_{t-l}) (t >= p); the structural shocks eps~_t = Omega' u_t;
 *   H_{i,k}(t, h) = sum_{l=0..h} (c_{i,l} omega_k)(omega_k' u_{t+h-l}) = omega_k' G_{i,t,h} omega_k, G = sum_l c_{i,l}' u_{t+h-l}':
 *   the contribution of shock k to series i over rows t .. t+h, i.e. dfm_historical_decomposition's contrib[i, t+h, k] from
 *   base row t - 1 on the model rotated by Omega' L^-1.
 *   Narrative rows (kind, shock j, series i, row t, window h, sign s), t a 0-based row of the path, p <= t, t + h < Tp, h < H:
 *     kind 0  shock sign          s eps~_{j,t} > 0                          (series and h unused)
 *     kind 1  most important      |H_{i,j}(t,h)| > max_{k != j} |H_{i,k}(t,h)|   (sign unused)
 *     kind 2  overwhelming        |H_{i,j}(t,h)| > sum_{k != j} |H_{i,k}(t,h)|   (sign unused)
 *     kind 3  contribution sign   s H_{i,j}(t,h) > 0
 *   Acceptance: shock by shock, as dfm_sign_restrictions: a shock's sign rows fix omega_j's orientation (4.14's flip rule) and
 *   its kind-0 rows are tested at it; a shock with no sign rows takes its orientation from its kind-0 rows (all > 0 keep, all
 *   < 0 flip, otherwise rejected).  H is quadratic in omega_k, so kinds 1-3 do not depend on the orientation: kind-3 rows are
 *   tested with their shock, kinds 1 and 2 once every column of Omega is drawn (the same columns as the kept Omega).
 *   Importance weight: the narrative event has probability w(theta, Omega) under structural shocks drawn N(0, I); conditioning
 *   on it divides the likelihood by w, so the kept draw's weight is 1 / w.  w is estimated from n_sim simulations:
 *   e_{k,tau} ~ N(0, 1) for every shock k and every period tau of the sorted union of the rows' periods (t for kind 0, t .. t+h
 *   otherwise; nP of them), the rows evaluated with H^sim_{i,k} = sum_l (c_{i,l} omega_k) e_{k,t+h-l} and eps~ = e; n_ok
 *   counts the simulations that satisfy every row and weight = n_sim / n_ok (+Inf when n_ok = 0).  e_{k,tau} of simulation s
 *   is normal number (s nP + p) r + k of the Philox stream of the model id, tag 19 (p the position of tau; < 2^34 within the
 *   bounds), common to every candidate of the model: the weights are a pure function of (seed, id, Omega).  With kind-0 rows
 *   only, on K distinct (shock, period) pairs, w = 2^-K exactly.
 *   With no narrative rows the call gives dfm_sign_restrictions' n_accept, cand, rot, resp and fevd bits, and weight 1.
 * Outputs: those of dfm_sign_restrictions, and per kept slot (any may be NULL; in `mem`):
 *   n_ok     [n_model x n_keep]                 the simulations that satisfy every row (0 for an empty slot);
 *   weight   [n_model x n_keep]                 n_sim / n_ok; +Inf when n_ok = 0; NaN for an empty slot or a failed model;
 *   eps      n_keep x (Tp x n_shock)            eps~_t of the leading n_shock shocks (NaN for t < p), column-major.
 * status: dfm_sign_restrictions' codes, also 3 when the path holds a NaN and DFM_ERR_ARG when a narrative series (kinds 1-3) is
 * out of the model; a model with several failures reports the first of: A or Q with a NaN or Q not positive definite (3), a sign
 * row's series out of the model (DFM_ERR_ARG), a NaN path row (3), a narrative series out of the model (DFM_ERR_ARG).  Bounds: dfm_sign_restrictions', at most 64 narrative rows, nP r <= 2^14, n_sim <= 2^20, and the shared
 * memory of the candidate kernel within 220 KB: (c + 1) r 64 + n r + r nK0 + r^2 nK123 doubles (c the columns drawn, r when
 * rows of kinds 1 / 2 exist; n the sign rows; nK0, nK123 the narrative rows of kind 0 and of kinds 1-3), e.g. at r = 16 with
 * every column drawn and 256 sign rows, 25 narrative rows of kinds 1-3; and the simulation kernel's, sum over the rows of
 * kinds 1-3 of (h + 1) r doubles: DFM_ERR_UNSUPPORTED past them.
 * Bad arguments (those of dfm_sign_restrictions, F NULL, Tp < 1, n_sim < 1, a kind outside 0..3, a sign other than +-1 on
 * kinds 0 / 3, a shock outside [1, n_shock], a series outside [0, N) on kinds 1-3, t < p, h < 0, h >= H, t + h >= Tp):
 * DFM_ERR_ARG.  Models in chunks and candidates in batches as dfm_sign_restrictions: model b has the same bits whatever n_model.
 * Synchronous for host memory. */
typedef struct {
  int N, r, p, n_model, H, n_shock;
  long long n_rot;
  int n_keep;
  unsigned long long seed;
  int mem;
  int Tp;                     /* rows of each factor path */
  int n_sim;                  /* simulations of the weight, 1 .. 2^20 */
} dfm_narr_opts;
typedef struct {
  int n;                      /* rows, 0 .. 64; HOST arrays of n (NULL when n = 0) */
  const int* kind;            /* 0 .. 3 */
  const int* shock;           /* 1 .. n_shock */
  const int* series;          /* 0-based series i (kinds 1-3) */
  const int* row;             /* 0-based row t of the path */
  const int* h;               /* window 0 .. H-1 (kinds 1-3) */
  const int* sign;            /* +1 or -1 (kinds 0, 3) */
} dfm_narr_restr;
typedef struct {
  long long* n_accept;
  long long* cand;
  double* rot;
  double* resp;
  double* fevd;
  int* status;
  long long* n_ok;
  double* weight;
  double* eps;
} dfm_narr_out;
int dfm_narrative_sign_restrictions(dfm_handle* h, const dfm_em_init* models, const double* F, const unsigned long long* ids,
                                    const double* scale, const dfm_narr_opts* opts, const dfm_sign_restr* restr,
                                    const dfm_narr_restr* narr, const dfm_narr_out* out);

/* ---- shocks identified by external instruments (proxy SVAR / SVAR-IV; Stock & Watson 2018) ------------------------------
 * models: n_model models (Lam N x r, R N, A = [A_1 .. A_p] r x k, Q r x r; P0 unused) as dfm_series_responses, k = r p; F: n_model
 * factor paths f_0 .. f_{Tp-1} (Tp x r each, column-major); Z: Tp x n_inst instruments (column-major, NaN = unavailable), the same
 * for every model; ids: HOST array of n_model model ids < 2^40 (NULL = 0 .. n_model-1); scale: N (NULL = 1).  All but ids in `mem`.
 * Per model, L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L and c_{i,h} = lam_i' Psi_h (as dfm_series_responses), and for t >= p
 * eta_t = f_t - sum_{l=1..p} A_l f_{t-l}, u_t = L^-1 eta_t.  Instrument k:
 *   T_k = {t >= p : z_{k,t} finite, f_t .. f_{t-p} finite} (n_k periods; see status for a NaN path row), zbar,
 *   s^2 = (1/n_k) sum (z - zbar)^2 and Gamma_k = (1/n_k) sum eta_t (z_t - zbar) over T_k; omega_k = L^-1 Gamma_k / |L^-1 Gamma_k|
 *   (the shock covaries positively with its instrument; b_k = L omega_k has b_k' Q^-1 b_k = 1: a one-standard-deviation shock);
 *   eps_{k,t} = omega_k' u_t (t >= p);
 *   resp[i,h] = scale_i c_{i,h} omega_k;  fevd[i,h] = sum_{l<=h} (c_{i,l} omega_k)^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i);
 *   reliability rho^2_k = |L^-1 Gamma_k|^2 / s^2 (not clamped: along a smoothed path it can exceed 1);
 *   first stage: y_t = lam_i0' eta_t on [1, z_{k,t}] over T_k, fs_pi the slope, fs_F = fs_pi^2 / V[1,1] with V the HAC(q) covariance
 *   of the OLS coefficients (Bartlett weights 1 - j/(q+1); q = 0: White's), the periods of T_k taken as consecutive.
 *   Moving-block bootstrap, replicate rho = 1 .. n_boot: T_k's periods indexed 0 .. n_k-1, l = min(block, n_k), ceil(n_k / l) block
 *   starts s_j = floor(u_j (n_k - l + 1)), u_j the uniform number (rho n_inst + k) Tp + j of the Philox stream of the model id,
 *   tag 20 (distinct for every (rho, k, j) since j < Tp); the blocks of (u_t, z_t) concatenated and cut at n_k give omega*, resp*
 *   and fevd* as above (a gap in the instrument is treated as adjacent periods).  Replicate 0 is the sample itself.  Record rho
 *   of model b is a function of (seed, id_b, k, rho, block) and the data alone: it does not depend on n_boot, n_model or chunking.
 * Outputs (any may be NULL; models back to back, column-major):
 *   omega        n_model x n_inst x (1 + n_boot) x r;
 *   resp, fevd   n_model x n_inst x (1 + n_boot) x (N x H);
 *   eps          n_model x n_inst x Tp            (NaN for t < p and rows with a NaN in f_t .. f_{t-p});
 *   n_obs (int), reliability, fs_pi, fs_F, status (int)   n_model x n_inst.
 * status per (model, instrument), the first of: 3 (DFM_ERR_NOT_PD) when A or Q holds a NaN or Q is not positive definite; DFM_ERR_ARG
 * when series i0 is out of the model (NaN loading row or R_i0); 3 when a NaN in the path touches a period of T_k (f_t .. f_{t-p}),
 * n_k < 3, or Gamma_k = 0.  Such a pair has NaN outputs (n_obs still counted); a bootstrap replicate with Gamma* = 0 has a NaN
 * record.  Neighbours are unaffected.  Bounds: k <= 48, n_inst <= 8, n_boot <= 65535, Tp (r + 1) + 64 r <= 28160 (the
 * bootstrap kernel's shared memory, e.g. Tp <= 3072 at r = 8): DFM_ERR_UNSUPPORTED past them.  Bad arguments (a NULL required
 * pointer, Tp < 1, H < 1, n_inst < 1, i0 outside [0, N), q < 0, block < 1, n_boot < 0, an id >= 2^40, a bad mem): DFM_ERR_ARG.
 * Synchronous for host memory. */
typedef struct {
  int N, r, p, n_model, Tp, H;
  int n_inst;                 /* instruments, 1 .. 8 */
  int i0;                     /* the first stage's series, 0 .. N-1 */
  int q;                      /* HAC lags of the first stage, >= 0 */
  int block;                  /* bootstrap block length, >= 1 */
  int n_boot;                 /* bootstrap replicates, 0 .. 65535 */
  unsigned long long seed;
  int mem;
} dfm_proxy_opts;
typedef struct {
  double* omega;
  double* resp;
  double* fevd;
  double* eps;
  int* n_obs;
  double* reliability;
  double* fs_pi;
  double* fs_F;
  int* status;
} dfm_proxy_out;
int dfm_proxy_identification(dfm_handle* h, const dfm_em_init* models, const double* F, const double* Z, const unsigned long long* ids,
                             const double* scale, const dfm_proxy_opts* opts, const dfm_proxy_out* out);

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

/* Weighted percentile bands per statistic, over the records ok that are not NaN and whose weight is > 0 and finite (NaN where
 * none is): in sorted order, the first record i with 100 sum_{j <= i} w_j >= q sum_j w_j, decided in exact arithmetic.  This is
 * numpy.percentile(recs[ok], q, axis=0, weights=w[ok], method="inverted_cdf") without numpy's rounding of the cumulative sums
 * and of q / 100; with equal weights it is numpy's unweighted inverted_cdf.  The sums are exact while they fit in 106 bits of the smallest weight's grid (always for
 * max w / min w <= 2^36, so every narrative weight n_sim / n_ok); beyond that a quantile within about 2^-100 of the total
 * from a cumulative weight may pick the neighbouring record.  recs as dfm_percentiles, w: n weights (both in `mem`).
 * n <= 16384 (as dfm_percentiles). */
int dfm_percentiles_weighted(dfm_handle* h, const double* recs, const double* w, long long n, int d, const double* q, int nq, int mem,
                             double* out);

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
