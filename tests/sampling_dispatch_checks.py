"""Oracle checks of the sampling entry points at the state sizes and edges they accept: dfm_simulation_smoother, dfm_news,
dfm_ss_bootstrap and dfm_gibbs at k = r p up to 48 and r up to 36 (the general path's shared-memory plan, ss_check), the
refusal at r = 37, partial tiles, a call whose draws span two chunks and a Gibbs sub-batch capped by memory.  CASES is the
table; test_gpu_sampling_dispatch.py runs it on the H100 with the kernel-set assertion of dispatch_checks.KernelLog,
test_emu_sampling_dispatch.py on the host-emulation build (no launch profiler there).  Each case runs as case.run(lib, nsm),
nsm = the device's SM count (132 on an H100; the emulation build fixes it at 132).

Branches inside a kernel cannot be seen from the launch profiler; each case's comment gives the predicate and the numbers
that decide them:
  - k_gibbs_paths: one warp per chain, lane owns rows lane and lane + 32 of its mat-vecs; the second row exists for k > 32;
  - wt_gemm tiles of k_sim_paths (the k x (k + 2 r) and k x 2k gain products) and k_news_cov (k x k) with m = k > 32;
  - k_news_cov's W r-sized part in shared memory iff (news_cov_small + news_cov_big) * 8 <= 220 KiB (news_big_in_smem);
  - dfm_simulation_smoother's chunk of draws (sim_chunk) and the sub-batch of dfm_ss_bootstrap / dfm_gibbs (ssb_batch),
    restated below;
  - ss_check: k <= 48 and em_fs_smem_doubles(r, p, staging tile) * 8 <= 220 KiB; at p = 1 that holds up to r = 36 for one
    panel and for 264 panels (tile 8 either way: 224 096 B) and fails at r = 37 (tile 8 for one panel: 236 824 B; tile 4
    for 264 panels: 232 824 B).

dfm_gibbs' own refusal `gibbs_draw_smem_doubles(r, p) * 8 > 220 KiB` cannot fire: enumerating every (r, p) with r p <= 48 it
holds only for p = 1, r = 45 .. 48 (227 584 B at r = 45), and ss_check refuses every r > 36 at p = 1 first
(test_gibbs_draw_guard_unreachable in the emulation file checks the enumeration)."""
import numpy as np

from dynamic_factor_models_b200 import DFMError, Library
from dispatch_checks import KernelLog, case  # noqa: F401  (KernelLog: used by the GPU file)
import em_constr_checks as ECC
import gibbs_checks as GC
import news_checks as NC
import parity_checks as P
import simsmooth_checks as SC
import ss_bootstrap_checks as BC

METHODS = ("simulation_smoother", "news", "ss_bootstrap", "gibbs", "em_kalman")
CASES = []

KMAX_SMEM = 220 * 1024                 # kMaxSmem of dfm_api.cu
CHUNK_BYTES = 512 << 20                # kSimChunkBytes
SIM_ND, SIM_PD, SS_NS = 16, 8, 64
NEWS_MAXQ, NEWS_TP, NEWS_QC = 64, 8, 8
GB_NC, GB_NT, GB_NS = 32, 128, 32


# ---------------------------------------------------------------------------------------- the host's size rules, restated
def sim_chunk(n_draw, Tp, N, r, k, stageF, stageX):
    """Draws per chunk of dfm_simulation_smoother (sim_chunk in dfm_api.cu)."""
    per = Tp * (k + r + (r if stageF else 0) + (N if stageX else 0)) * 8
    c = max(SIM_ND, CHUNK_BYTES // per)
    c = min(c, (65535 // ((N + SS_NS - 1) // SS_NS)) * SIM_PD)
    return min(c, n_draw)


def ssb_batch(nsm, T, N, r, p):
    """Replicates / chains per sub-batch of dfm_ss_bootstrap and dfm_gibbs (ssb_batch in dfm_api.cu)."""
    k = r * p; kk = k * k; rk = r * k; np_ = r * (r + 1) // 2
    par = N * r + N + rk + r * r
    per = 8 * (T * N + T * r + 8 * par + 3 * kk + T * (2 * kk + 2 * k + 2 * np_ + 4 * r + 4) + 64 * k + 16 * (kk + rk))
    return min(max(1, CHUNK_BYTES // per), min(2 * nsm, 65535))


def news_big_in_smem(r, p, W, nq):
    """Is the W r-sized part of k_news_cov in shared memory (news_cov_small_doubles + news_cov_big_doubles <= kMaxSmem)?"""
    k, n = r * p, W * r
    small = 7 * k * k + 8 + NEWS_MAXQ
    big = 2 * k * n + 2 * n * n + n * nq + r * n
    return (small + big) * 8 <= KMAX_SMEM


def gibbs_draw_smem(r, p):
    k = r * p
    return (3 * k * k + 4 * k * r + 7 * r * r + 2 * k + 8) * 8


def _lds(k):
    return k + ((12 - k % 8) % 8)


def em_fs_smem(r, p, stg):
    k = r * p; kk = k * k; rr = r * r; rk = r * k
    return 8 * (9 * kk + 7 * rr + 3 * rk + 6 * k + 2 * r + 128 + 3 * k * 16 + r * (stg + 4) + (2 * stg + 1) * _lds(k) + 8 + 192)


def ss_accepts(nsm, batch, r, p):
    """ss_check's size rule (fs_stage_periods, then the smem bound)."""
    stg = 256 if batch <= nsm else 16
    if batch <= nsm:
        while stg > 8 and em_fs_smem(r, p, stg) > KMAX_SMEM:
            stg //= 2
    elif em_fs_smem(r, p, 4) <= 112 * 1024:
        while stg > 4 and em_fs_smem(r, p, stg) > 112 * 1024:
            stg //= 2
    else:
        while stg > 4 and em_fs_smem(r, p, stg) > KMAX_SMEM:
            stg //= 2
    return r * p <= 48 and em_fs_smem(r, p, stg) <= KMAX_SMEM


# ---------------------------------------------------------------------------------------------------- kernel sets
FS = "k_em_filter_smooth"
FUSED = ("k_em_fused<RT>", "k_em_fused2<RT>")
SIM = {"simulation_smoother": (("k_sim_gains", "k_sim_paths", "k_sim_project", FS), FUSED + ("k_gibbs_paths", "k_ss_project"))}
SIM_F = {"simulation_smoother": (("k_sim_gains", "k_sim_paths", FS), FUSED + ("k_sim_project", "k_gibbs_paths", "k_ss_project"))}
NEWS = {"news": (("k_news_window", "k_news_cov", "k_news_project", "k_news_finish", FS), FUSED + ("k_sim_paths", "k_ss_project"))}
SSB = {"ss_bootstrap": (("k_ss_sim_chol", "k_ss_simulate", "k_ss_sim_project", FS, "k_ss_align", "k_irf", "k_ss_project", "k_ss_fc_rows"),
                        FUSED)}
GIBBS = {"gibbs": ((FS, "k_sim_gains", "k_gibbs_paths", "k_gibbs_stats", "k_gibbs_draw", "k_sim_project", "k_ss_fc_rows", "k_ss_align",
                    "k_irf"), FUSED + ("k_sim_paths",))}
GIBBS_NOIRF = {"gibbs": ((FS, "k_sim_gains", "k_gibbs_paths", "k_gibbs_stats", "k_gibbs_draw", "k_sim_project"),
                         FUSED + ("k_sim_paths", "k_ss_align", "k_irf"))}
HOLES = ((0, 40, 3), (120, 170, 7), (60, 90, 11), (170, 200, 2))


def sampling_case(id_, kernels):
    return case(id_, kernels, table=CASES)


def _code(fn):
    try:
        fn()
    except DFMError as e:
        return e.code
    return 0


def _same_as_fresh_handle(lib, call):
    """call(lib) on the handle after a refusal gives the bits of call() on a fresh handle."""
    got = call(lib)
    fresh = Library(lib.path)
    try:
        ref = call(fresh)
    finally:
        fresh.close()
    for n in ref:
        np.testing.assert_array_equal(got[n], ref[n], err_msg=n)


def _big_model(N, r, p, T, seed=3):
    """Shapes of a model of r factors, p lags (values only have to pass the argument checks)."""
    rng = np.random.default_rng(seed)
    k = r * p
    return dict(X=rng.standard_normal((T, N)), Lam=0.1 * rng.standard_normal((N, r)), R=np.ones(N), A=np.zeros((r, k)), Q=np.eye(r),
                P0=np.eye(k))


# ---------------------------------------------------------------------------------------------------- 1. simulation smoother
@sampling_case("sim_k48_r12_p4_holes", SIM)
def _(lib, nsm):
    # k = 48 > 32: k_sim_paths' wt_gemm tiles with m = 48 (k x (k + 2r) = 48 x 72 forward, 48 x 96 backward); the E-step is one
    # panel: 512 threads, an 8-CTA cluster (8 <= nsm), staging tile 8 (em_fs_smem = 219 552 B), two-row scan; missing cells,
    # four blocks of missing data and H = 8 forecast periods
    assert ss_accepts(nsm, 1, 12, 4) and not ss_accepts(nsm, 1, 13, 4)
    SC.check_sim(lib, N=40, r=12, T=200, p=4, miss=0.05, H=8, holes=HOLES, n_draw=3, draw0=5)


@sampling_case("sim_r36_p1", SIM)
def _(lib, nsm):
    # r = 36, p = 1: the largest r ss_check takes at p = 1 (tile 8: 224 096 <= 225 280 B); k = 36 > 32
    assert ss_accepts(nsm, 1, 36, 1)
    SC.check_sim(lib, N=120, r=36, T=150, p=1, miss=0.05, H=4, n_draw=2)


@sampling_case("sim_r37_refused", SIM)
def _(lib, nsm):
    # r = 37, p = 1: em_fs_smem at tile 8 = 236 824 B > 225 280: status 6 (DFM_ERR_UNSUPPORTED) before any launch
    assert not ss_accepts(nsm, 1, 37, 1)
    m = _big_model(120, 37, 1, 60)
    assert _code(lambda: lib.simulation_smoother(m["X"], m["Lam"], m["R"], m["A"], m["Q"], p=1, H=2, n_draw=2)) == 6
    X, Lam, Rv, A, Q = SC.problem(N=20, r=3, T=50, p=2, miss=0.1)
    _same_as_fresh_handle(lib, lambda L: L.simulation_smoother(X, Lam, Rv, A, Q, p=2, H=3, n_draw=5, seed=SC.SEED, draw0=2))


@sampling_case("sim_N130_partial_tiles", SIM)
def _(lib, nsm):
    # N = 130: three SS_NS = 64 series tiles of k_sim_project, the last with 2 series; 21 draws: two k_sim_paths CTAs of
    # SIM_ND = 16 (the second with 5) and three k_sim_project draw tiles of SIM_PD = 8 (the last with 5)
    assert 21 % SIM_ND and 21 % SIM_PD and 130 % SS_NS
    SC.check_sim(lib, N=130, r=3, T=60, p=2, miss=0.1, H=3, n_draw=21, draw0=7)


@sampling_case("sim_chunk_boundary", SIM_F)
def _(lib, nsm):
    # F-only host output: sim_chunk = 512 MiB / (Tp (k + 2 r) 8) = 2^29 / (8192 * 16 * 8) = 512 draws (the grid.y bound,
    # 65535 * 8, does not bind at N = 12); 515 draws are two chunks, [0, 512) and [512, 515), the second from id draw0 + 512
    N, r, p, T, H, n, d0 = 12, 4, 2, 8188, 4, 515, 3
    ch = sim_chunk(n, T + H, N, r, r * p, True, False)
    assert ch == 512 < n
    X, Lam, Rv, A, Q = SC.problem(N=N, r=r, T=T, p=p, miss=0.05)
    got = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=n, seed=SC.SEED, draw0=d0, outputs=("F",))
    assert got["status"] == 0 and got["F"].shape == (n, T + H, r)
    for j in (0, ch - 1, ch, n - 1):
        one = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=1, seed=SC.SEED, draw0=d0 + j, outputs=("F",))
        np.testing.assert_array_equal(got["F"][j], one["F"][0], err_msg="draw %d" % j)
    refF, _ = SC.simulation_smoother(X, Lam, Rv, A, Q, None, p, H, SC.SEED, [d0 + ch - 1, d0 + ch])
    SC.compare(dict(F=got["F"][[ch - 1, ch]]), refF, None)


# ---------------------------------------------------------------------------------------------------- 2. news
def _news(lib, N, r, p, T, H, news_rows, targets, miss=0.05):
    Xo, Xn, Lam, Rv, A, Q = NC.vintages(N, r, T, p, miss, news_rows=news_rows)
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=p, H=H, targets=targets, news_rows=news_rows)
    assert got["status"] == 0
    NC.compare(got, NC.news_spec(Xo, Xn, Lam, Rv, A, Q, None, p, H, targets, news_rows))


@sampling_case("news_k48_cov_in_smem", NEWS)
def _(lib, nsm):
    # k = 48, W = 3 rows, 3 targets inside the window: W r = 36; small part 7 * 48^2 + 72 = 16 200, big part
    # 2 * 48 * 36 + 2 * 36^2 + 36 * 3 + 12 * 36 = 6 588 doubles: 182 304 <= 225 280 B, the W r part in shared memory
    assert news_big_in_smem(12, 4, 3, 3)
    T = 200
    _news(lib, N=40, r=12, p=4, T=T, H=0, news_rows=3, targets=[(0, T - 1), (39, T - 2), (5, T - 3)])


@sampling_case("news_k48_cov_global", NEWS)
def _(lib, nsm):
    # k = 48, W = 3 rows + 2 target periods outside the window (T - 8 and the forecast T) = 5: W r = 60; big part
    # 2 * 48 * 60 + 2 * 60^2 + 60 * 5 + 12 * 60 = 13 980 doubles: 241 440 > 225 280 B, the W r part in global scratch
    assert not news_big_in_smem(12, 4, 5, 5)
    T = 200
    _news(lib, N=40, r=12, p=4, T=T, H=1, news_rows=3, targets=[(0, T - 1), (39, T - 2), (5, T - 3), (1, T - 8), (2, T)])


@sampling_case("news_r36_p1", NEWS)
def _(lib, nsm):
    # r = 36, p = 1, W = 3: W r = 108 <= NEWS_MAXN = 128; big part 2 * 36 * 108 + 2 * 108^2 + 108 * 3 + 36 * 108 = 35 316
    # doubles: global scratch (355 680 > 225 280 B); k = 36 > 32
    assert 3 * 36 <= 128 and not news_big_in_smem(36, 1, 3, 3)
    T = 150
    _news(lib, N=120, r=36, p=1, T=T, H=0, news_rows=3, targets=[(0, T - 1), (119, T - 2), (7, T - 3)])


@sampling_case("news_N130_partial_tiles", NEWS)
def _(lib, nsm):
    # N = 130: three NEWS_NS = 64 series tiles (the last with 2); news_rows = 11: two NEWS_TP = 8 row tiles (the last with 3);
    # 10 targets: two NEWS_QC = 8 target passes of k_news_project (the last with 2); W = 11 + 4 = 15, W r = 45
    T, nr = 80, 11
    tg = [(0, T - 1), (129, T - 2), (64, T - 3), (65, T - 11), (127, T - 6), (3, T - 7), (1, T - 20), (2, T - 30), (5, T), (128, T + 1)]
    assert nr % NEWS_TP and len(tg) > NEWS_QC and 130 % 64
    assert news_big_in_smem(3, 2, 15, len(tg))
    _news(lib, N=130, r=3, p=2, T=T, H=2, news_rows=nr, targets=tg, miss=0.1)


# ---------------------------------------------------------------------------------------------------- 3. parametric bootstrap
@sampling_case("ssb_k48_r12_p4", SSB)
def _(lib, nsm):
    # k = 48: a sub-batch of ssb_batch = 63 replicates (memory cap: 2^29 / 8.5 MB per replicate < 2 nsm); the EM on it runs
    # the general path at k = 48 (many panels: tile 8), then k_ss_align and dfm_irf (k_irf) at k = 48, and the forecast
    # E-step (dfm_kalman_smooth) at the aligned parameters
    T, N, r, p = 200, 40, 12, 4
    assert ssb_batch(nsm, T, N, r, p) < 2 * nsm
    X, th = BC.fitted(N=N, r=r, T=T, p=p, miss=0.05, exclude=(6,), ragged=2)
    BC.check_bootstrap(lib, X, th, p, n_rep=2, rep0=1, max_iter=2, H_irf=4, H_fc=2, fc_rows=3)


@sampling_case("ssb_r36_p1", SSB)
def _(lib, nsm):
    # r = 36, p = 1 (k = 36 > 32): the EM without the multi-CTA contraction (r > 32), k_ss_align's r x r solves at r = 36
    T, N, r, p = 150, 120, 36, 1
    X, th = BC.fitted(N=N, r=r, T=T, p=p, miss=0.05)
    BC.check_bootstrap(lib, X, th, p, n_rep=2, rep0=0, max_iter=2, H_irf=3, H_fc=1, fc_rows=2)


@sampling_case("em_r20_after_restricted_em", {"em_kalman": (("k_em_mstep_series", "k_em_contract", FS), FUSED)})
def _(lib, nsm):
    # The EM inside dfm_ss_bootstrap after a restricted EM in the same process: k_em_mstep_series needs
    # (2 np + r + 8) * 8 B of shared memory, 3 584 B at r = 20, and the restricted call at r = 3 set the kernel's attribute
    # to (2 * 6 + 3 + 8 + 18) * 8 = 328 B; the unrestricted call must set it again (it once did not, and its launches at
    # r = 36 failed after any restricted call: status 5)
    ECC.check_vs_spec(lib, N=20, r=3, T=60, p=1, miss=0.1, iters=2)
    P.check_em(lib, N=60, r=20, T=150, p=1, miss=0.1, iters=2, path=1, ll_cell_tol=1e-12)


# ---------------------------------------------------------------------------------------------------- 4. Gibbs
def _chains(lib, N, r, p, T, miss=0.05, **kw):
    X, th = GC.model(N=N, r=r, T=T, p=p, miss=miss, exclude=(4,), ragged=3)
    args = dict(n_chain=2, n_burn=1, n_keep=2, H_fc=2, fc_rows=3, H_irf=4, chain0=1, sweep0=2)
    args.update(kw)
    GC.check_chains(lib, X, th, p, **args)


@sampling_case("gibbs_k48_r12_p4", GIBBS)
def _(lib, nsm):
    # k = 48 > 32: k_gibbs_paths' second row per lane (rows 32 .. 47), k_gibbs_draw's 48 x 48 transition solve and r = 12
    # per-series packed solves and Bartlett draw, k_ss_align / k_irf at k = 48; ssb_batch = 63 chains per sweep
    _chains(lib, N=40, r=12, p=4, T=200)


@sampling_case("gibbs_k36_r12_p3", GIBBS)
def _(lib, nsm):
    # k = 36: rows 32 .. 35 on lanes 0 .. 3
    _chains(lib, N=40, r=12, p=3, T=200)


@sampling_case("gibbs_r36_p1", GIBBS)
def _(lib, nsm):
    # r = 36, p = 1: the largest r at p = 1 (ss_check at batch ssb_batch); 36 x 36 per-series solves and NIW draw
    assert ss_accepts(nsm, ssb_batch(nsm, 150, 120, 36, 1), 36, 1)
    _chains(lib, N=120, r=36, p=1, T=150, H_irf=3)


@sampling_case("gibbs_N200_missing", GIBBS)
def _(lib, nsm):
    # N = 200 > GB_NT = 128: k_gibbs_draw's series loop runs series 128 .. 199 on a second round of threads, with their
    # missing-cell downdates; k_gibbs_stats: series tiles of GB_NS = 32 (the last with 8) and C r = 264 * 5 = 1 320 factor
    # columns, 41 full GB_NC = 32 tiles and one of 8
    T, N, r, p = 60, 200, 5, 1
    C = ssb_batch(nsm, T, N, r, p)
    assert N > GB_NT and N % GB_NS and (C * r) % GB_NC, (C, r)
    _chains(lib, N=N, r=r, p=p, T=T, miss=0.1)


@sampling_case("gibbs_r37_refused", GIBBS_NOIRF)
def _(lib, nsm):
    # r = 37, p = 1: ss_check refuses at the sub-batch size (status 6); the next call on the handle is a fresh handle's
    T, N = 60, 120
    assert not ss_accepts(nsm, ssb_batch(nsm, T, N, 37, 1), 37, 1)
    m = _big_model(N, 37, 1, T)
    init = {n: m[n] for n in ("Lam", "R", "A", "Q", "P0")}
    assert _code(lambda: lib.gibbs(m["X"], init, p=1, n_chain=1, n_keep=1, prior=GC.PRIOR, seed=GC.SEED)) == 6
    X, th = GC.model(N=14, r=3, T=40, p=1)
    ini = GC._inits(th, 3)
    _same_as_fresh_handle(lib, lambda L: L.gibbs(X, ini, p=1, n_chain=3, n_burn=1, n_keep=2, seed=GC.SEED, H_fc=1, fc_rows=2,
                                                 prior=GC.PRIOR, outputs=("Lam", "R", "A", "Q", "F", "X")))


@sampling_case("gibbs_chain_split_capped_batch", GIBBS_NOIRF)
def _(lib, nsm):
    # N = 1 300, T = 200, r = 2: ssb_batch = 2^29 / 2 383 456 B per chain = 225 < 2 nsm = 264, so a sub-batch is capped by
    # memory, not by the SM count; a call on chains [0, C + 10) runs two sub-batches, and calls on [0, 20) and on
    # [C - 8, C + 8), which straddles the big call's boundary, give the same bits
    T, N, r, p = 200, 1300, 2, 1
    C = ssb_batch(nsm, T, N, r, p)
    assert C < 2 * nsm, C
    X, th = GC.model(N=N, r=r, T=T, p=p, miss=0.05, exclude=(4,), ragged=2)
    base = GC._inits(th, C + 10)
    kw = dict(p=p, sweep0=2, n_burn=1, n_keep=1, seed=GC.SEED, H_fc=1, fc_rows=2, prior=GC.PRIOR, outputs=("Lam", "R", "F", "X"))
    sub = lambda c0, n: {m: base[m][c0:c0 + n] for m in base}
    big = lib.gibbs(X, sub(0, C + 10), n_chain=C + 10, chain0=0, **kw)
    assert (big["status"] == 0).all()
    for c0, n in ((0, 20), (C - 8, 16)):
        got = lib.gibbs(X, sub(c0, n), n_chain=n, chain0=c0, **kw)
        for m in got:
            np.testing.assert_array_equal(got[m], big[m][c0:c0 + n], err_msg="%s [%d, %d)" % (m, c0, c0 + n))
