"""Oracle checks on the dispatch branches of the library: the kernel family dfm_api.cu picks from r, p, T, N, the batch
size, the SM count and whether a panel has NaNs, and the branches inside k_em_filter_smooth that depend on k = r p, the
thread count and the staging tile.  CASES is the table; test_gpu_dispatch.py runs it on the H100 with the kernel-set
assertion, test_emu_dispatch.py on the host-emulation build (profiling is compiled out there).

Host-level choices are asserted from the launch profiler (KernelLog).  Branches inside a kernel cannot be seen that way;
each case's comment gives the predicate and the numbers that decide them, for the H100 (132 SMs):
  - em_run_scan: k <= 32 one row per lane, k > 32 two rows per lane (k_em_filter_smooth, dfm_kernels_em.cuh);
  - backward Gram sums of the frozen runs: DMMA tiles in registers if nt00 + nt11 <= 6 * warps, else plain sums, with
    nt00 = ceil(k / 8)^2, nt11 = ceil(r / 8) ceil(k / 8);
  - threads of k_em_filter_smooth: 512 for batch <= 2 * 132, else 256; a thread-block cluster of 8 / 4 / 2 CTAs per panel
    while batch * 8 / 4 / 2 <= 132;
  - staging tile: up to 256 periods for batch <= 132, else 16 (or less to fit the shared-memory plan)."""
import collections

import numpy as np

from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel
import forecast_checks as FC
import parity_checks as P

FS = "k_em_filter_smooth"
EMB = ("k_emb_contract<NCB>", "k_emb_mstep<NCB>", "k_emb_close")
FUSED = ("k_em_fused<RT>", "k_em_fused2<RT>")


class KernelLog:
    """A Library whose calls of the named methods run with the launch profiler on; seen[method] collects the kernel names
    those calls launched (the launch-site strings of dfm_api.cu, e.g. "k_emb_contract<NCB>").  Other attributes pass
    through, so the parity checks take a KernelLog in place of a Library."""

    def __init__(self, lib, methods=("em_kalman", "em_init_from_factors", "kalman_smooth", "estimate_factor")):
        self._lib = lib
        self.seen = {m: set() for m in methods}

    def __getattr__(self, name):
        attr = getattr(self._lib, name)
        if name not in self.seen:
            return attr

        def call(*a, **kw):
            self._lib.profile(True)
            try:
                return attr(*a, **kw)
            finally:
                self.seen[name] |= set(self._lib.profile_report())
                self._lib.profile(False)
        return call

    def check(self, kernels):
        """kernels: {method: (launched, not_launched)}; each name of `launched` was launched by some call of the method,
        no name of `not_launched` by any."""
        for m, (yes, no) in kernels.items():
            seen = self.seen[m]
            assert seen, "%s was not called" % m
            missing = set(yes) - seen
            assert not missing, "%s did not launch %s (launched: %s)" % (m, sorted(missing), sorted(seen))
            extra = set(no) & seen
            assert not extra, "%s launched %s (launched: %s)" % (m, sorted(extra), sorted(seen))


# ---------------------------------------------------------------------------------------------------- the new checks
def _panels(B, N, r, T, p, miss=0.0, holes=(), every=3, rep0=800):
    """B panels; those with b % every == 0 get missing_frac = miss and the (t0, t1, i) holes, the others are balanced.
    Starting parameters from each panel's own PCA factors."""
    Xb = []
    for b in range(B):
        hit = every > 0 and b % every == 0
        X, _ = simulate_panel(N, r, T, rep=rep0 + b, missing_frac=miss if hit else 0.0)
        if hit:
            for t0, t1, i in holes:
                X[t0:t1, i] = np.nan
        Xb.append(X)
    Xb = np.stack(Xb)
    inits = [K.init_from_factors(Xb[b], R.pca_score(np.nan_to_num(Xb[b]), r), p) for b in range(B)]
    return (Xb,) + tuple(np.stack([i[j] for i in inits]) for j in range(4))


def check_em_many_panels(lib, B, N, r, T, p=1, iters=2, miss=0.0, holes=(), every=3, ll_cell_tol=1e-12):
    """General path on B panels (the many-panel plan of k_em_filter_smooth once B > the SM count); the first, second,
    middle and last panels against the oracle and against a one-panel call, which runs the few-panel plan (512 threads,
    staging tile up to 256, a cluster of CTAs): two GPU plans with different summation orders, compared to 1e-9."""
    Xb, Lam, Rv, A, Q = _panels(B, N, r, T, p, miss, holes, every)
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=p, max_iter=iters, path=1)
    assert (got["status"] == 0).all() and (got["iters"] == iters).all()
    for b in sorted({0, 1, B // 2, B - 1}):
        mine = {n: got[n][b] for n in ("F", "PF", "Lam", "R", "A", "Q", "P0", "loglik")}
        ref = K.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=p, max_iter=iters)
        P.compare_em(mine, ref, P.ll_atol(Xb[b], ll_cell_tol))
        one = lib.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=p, max_iter=iters, path=1)
        np.testing.assert_allclose(mine["loglik"], one["loglik"], rtol=1e-9, atol=P.ll_atol(Xb[b], 1e-13))
        assert P.rmse(mine["F"], one["F"]) < 1e-9
        for n in ("PF", "Lam", "R", "A", "Q"):
            np.testing.assert_allclose(mine[n], one[n], rtol=1e-9, atol=1e-11, err_msg=n)


def check_em_init_batch(lib, B, N, r, T, p=1, miss=0.1, every=2):
    """em_init_from_factors on a batch mixing balanced panels (every `every`-th has missing data, one of its series with
    fewer than r + 1 observations) vs oracle.kalman_em.init_from_factors panel by panel."""
    Xb = np.stack([simulate_panel(N, r, T, rep=900 + b, missing_frac=miss if b % every == 0 else 0.0)[0] for b in range(B)])
    Xb[0, r:, 1] = np.nan                                   # r observations: no regression, NaN loading and R
    F = np.stack([R.pca_score(np.nan_to_num(Xb[b]), r) for b in range(B)])
    got = lib.em_init_from_factors(Xb, F, p)
    for b in range(B):
        ref = K.init_from_factors(Xb[b], F[b], p)
        P.compare_em_init(tuple(g[b] for g in got), ref)
    assert np.isnan(got[0][0, 1]).all() and np.isnan(got[1][0, 1])


# ---------------------------------------------------------------------------------------------------- the case table
Case = collections.namedtuple("Case", "id run kernels")
CASES = []


def case(id_, kernels, table=CASES):
    def reg(fn):
        table.append(Case(id_, fn, kernels))
        return fn
    return reg


def em(yes, no):
    return {"em_kalman": (yes, no)}


# (without the multi-CTA contraction the host does not count the panels with missing data, so k_em_contract is launched
#  as well and returns at once for balanced panels)
GEN_BAL = em(("k_em_contract_bal", "k_em_mstep_series", "k_em_prep", FS), EMB + ("k_emb_cinit",) + FUSED)
EMB_BAL = em(EMB + ("k_em_prep", FS), ("k_em_contract", "k_em_contract_bal", "k_em_mstep_series") + FUSED)
GEN_MISS = em(("k_em_contract", "k_em_mstep_series", "k_em_prep", FS), ("k_emb_contract<NCB>", "k_emb_mstep<NCB>", "k_em_contract_bal") + FUSED)
MIXED = em(("k_em_contract", "k_em_mstep_series", "k_em_prep", FS) + EMB, ("k_em_contract_bal",) + FUSED)
INIT_PLAIN = {"em_init_from_factors": (("k_als_lambda", "k_var"), ("k_emb_init_flags", "k_emb_mstep<NCB>", "k_gram_small"))}
INIT_EMB = {"em_init_from_factors": (("k_emb_init_flags", "k_gram_small", "k_emb_mstep<NCB>", "k_als_lambda", "k_var"), ())}
SMOOTH = {"kalman_smooth": (("k_em_contract", "k_em_contract_bal", FS, "k_ss_project"), EMB + ("k_em_mstep_series",) + FUSED)}
HOLES = ((0, 60, 3), (230, 300, 7), (100, 140, 11), (250, 300, 2))


# 1, 3: r > 32 turns the multi-CTA contraction off (emb_plan: r <= 32): k_em_contract_bal, k_em_mstep_series and the
# closing k_em_prep run on balanced panels, and em_init_from_factors takes its plain per-series regressions.
@case("r34_p1_one_panel", GEN_BAL | INIT_PLAIN)
def _(lib):
    # k = 34 > 32: two-row scan; 1 panel: 512 threads, 8-CTA cluster, nt00 + nt11 = 25 + 25 = 50 <= 96: register Gram sums
    P.check_em(lib, N=120, r=34, T=300, p=1, iters=2, path=1, ll_cell_tol=1e-12)


@case("r34_p1_270_panels", GEN_BAL)
def _(lib):
    # 270 > 264 panels: 256 threads, nt00 + nt11 = 50 > 48: plain-sum Gram; staging tile 16; k = 34: two-row scan
    check_em_many_panels(lib, B=270, N=120, r=34, T=300)


@case("r34_init_mixed_batch", INIT_PLAIN)
def _(lib):
    check_em_init_batch(lib, B=3, N=120, r=34, T=150)


# 2: k > 32 states (two-row scan) up to the general path's k = 48, balanced (frozen runs of >= 256 periods) and with blocks
# of missing data (the frozen runs end at each block edge)
@case("k36_r12_p3_one_panel", EMB_BAL)
def _(lib):
    # k = 36 > 32: two-row scan; 512 threads, nt00 + nt11 = 25 + 10 = 35 <= 96: register Gram sums; cluster of 8
    P.check_em(lib, N=40, r=12, T=320, p=3, iters=2, path=1, ll_cell_tol=1e-12)


@case("k48_r12_p4_holes_one_panel", GEN_MISS)
def _(lib):
    # k = 48: two-row scan; nt00 + nt11 = 36 + 12 = 48 <= 96; missing data: k_em_contract (np = 78)
    P.check_em(lib, N=40, r=12, T=300, p=4, iters=2, path=1, holes=HOLES, ll_cell_tol=1e-12)


@case("k48_r8_p6_one_panel", EMB_BAL)
def _(lib):
    # k = 48, r = 8: one DMMA column block in the contraction, six lags in the companion shift
    P.check_em(lib, N=30, r=8, T=300, p=6, iters=2, path=1, ll_cell_tol=1e-12)


@case("k36_r12_p3_160_panels", EMB_BAL)
def _(lib):
    # 132 < 160 <= 264: 512 threads, staging tile 16; k = 36: two-row scan; nt00 + nt11 = 35 <= 96: register Gram sums
    check_em_many_panels(lib, B=160, N=40, r=12, T=300, p=3)


@case("k48_r8_p6_150_panels_holes", MIXED)
def _(lib):
    # 150 panels, every third with blocks of missing data: both contraction families; k = 48: two-row scan; 512 threads,
    # nt00 + nt11 = 36 + 6 = 42 <= 96
    check_em_many_panels(lib, B=150, N=30, r=8, T=300, p=6, holes=HOLES)


@case("kalman_smooth_k48_r12_p4", SMOOTH)
def _(lib):
    FC.check_kalman_smooth(lib, N=40, r=12, T=300, p=4, H=8, ll_cell_tol=1e-12)


@case("kalman_smooth_k48_r8_p6_holes", SMOOTH)
def _(lib):
    FC.check_kalman_smooth(lib, N=30, r=8, T=300, p=6, H=8, holes=HOLES, ll_cell_tol=1e-12)


@case("kalman_smooth_r34_p1", SMOOTH)
def _(lib):
    FC.check_kalman_smooth(lib, N=120, r=34, T=150, p=1, H=8, ll_cell_tol=1e-12)


# 4: the many-panel plan of the general path
@case("r8_p1_300_panels_missing", MIXED)
def _(lib):
    # 300 > 264: 256 threads, staging tile 16, nt00 + nt11 = 2 <= 48; k = 8: one-row scan; every third panel 10 % missing
    check_em_many_panels(lib, B=300, N=24, r=8, T=120, miss=0.1)


@case("r4_p2_140_panels", EMB_BAL)
def _(lib):
    # 132 < 140 <= 264: 512 threads, staging tile 16, no cluster; k = 8
    check_em_many_panels(lib, B=140, N=16, r=4, T=150, p=2, every=0)


# 5: missing data at r > 8 (k_em_contract: thread per period, np = 78 / 210 packed information-matrix entries) and
# batches mixing balanced and missing panels (both contraction families, k_em_prep with skip_bal, k_emb_close)
@case("r12_missing", GEN_MISS)
def _(lib):
    P.check_em(lib, N=40, r=12, T=150, p=1, miss=0.1, iters=3, path=1, ll_cell_tol=1e-12)


@case("r20_missing", GEN_MISS)
def _(lib):
    P.check_em(lib, N=60, r=20, T=150, p=1, miss=0.1, iters=2, path=1, ll_cell_tol=1e-12)


@case("r12_mixed_batch", MIXED)
def _(lib):
    P.check_em_batch(lib, B=3, N=40, r=12, T=150, p=1, path=1)


@case("r20_p2_mixed_batch", MIXED)
def _(lib):
    # (k = 40; r = 28 with p = 2 would be k = 56, past the general path's shared-memory plan)
    P.check_em_batch(lib, B=3, N=60, r=20, T=150, p=2, path=1)


@case("r28_mixed_batch", MIXED)
def _(lib):
    P.check_em_batch(lib, B=3, N=90, r=28, T=150, p=1, path=1)


@case("r12_init_mixed_batch", INIT_EMB)
def _(lib):
    check_em_init_batch(lib, B=4, N=40, r=12, T=150)


# 6: column blocks of 8 in k_emb_contract<NCB> / k_emb_mstep<NCB>: one live column in the last block (9, 17, 25) and full
# blocks (16, 24, 32)
def _balanced(r):
    @case("balanced_r%d" % r, EMB_BAL)
    def _(lib):
        P.check_em(lib, N=3 * r + 4, r=r, T=150, p=1, iters=2, path=1, ll_cell_tol=1e-12)
        P.check_em_batch_balanced(lib, B=3, N=3 * r + 4, r=r, T=150, path=1, ll_cell_tol=1e-12)


for _r in (9, 16, 17, 24, 25, 32):
    _balanced(_r)


# 7: template instantiations of the fused kernels (the dispatch over r = 1..8)
def _fused(r, N, T):
    @case("fused_r%d" % r, em(("k_em_fused<RT>",), ("k_em_fused2<RT>", FS)))
    def _(lib):
        P.check_em(lib, N=N, r=r, T=T, p=1, iters=4, path=2)


def _fused2(r, N, T):
    @case("fused2_r%d_N%d_T%d" % (r, N, T), em(("k_em_fused2<RT>",), ("k_em_fused<RT>", FS)))
    def _(lib):
        P.check_em(lib, N=N, r=r, T=T, p=1, iters=4, path=3)


def _als_fused(r):
    @case("als_fused_r%d" % r, {"estimate_factor": (("k_als_fused2<RT>",), ("k_als_masked<RT>", "k_als_factor"))})
    def _(lib):
        P.check_als_balanced(lib, N=3 * r + 8, r=r, T=150, B=2)


def _als_masked(r):
    @case("als_masked_r%d" % r, {"estimate_factor": (("k_als_masked<RT>",), ("k_als_fused2<RT>", "k_als_factor"))})
    def _(lib):
        P.check_als_batch(lib, B=3, N=3 * r + 6, r=r, T=150)


for _r, _N, _T in ((2, 16, 150), (4, 21, 150), (6, 31, 151), (7, 40, 150)):
    _fused(_r, _N, _T)
for _r, _N, _T in ((2, 16, 264), (6, 27, 150), (7, 40, 302)):            # N % 8 = 3 and one short chunk (150 < 172) at r = 6
    _fused2(_r, _N, _T)
for _r in (1, 2, 4, 5, 6, 7):
    _als_fused(_r)
for _r in (4, 5, 6, 7):
    _als_masked(_r)
