"""Oracle checks of dfm_em_kalman_constrained (the state-space EM under linear restrictions on the loadings) at the sizes and
edges it accepts: k_emb_mstep_constr<NCB> at every column-block count NCB = 1 .. 4, restricted series in every series tile,
at the tile edges and in a ragged last tile, time splits with a ragged last split, the shared memory of r = 27 .. 32 (above
the 48 KiB default only because of the restriction's scratch), r = 36 and k = 48 on the general path, missing data,
mixed batches, the stopping rule, the order of the rows, nearly dependent rows and caller device memory.  CASES is the
table; test_gpu_em_constr_dispatch.py runs it on the H100 with the kernel-set assertion of dispatch_checks.KernelLog,
test_emu_em_constr_dispatch.py on the host-emulation build (no launch profiler there).  Each case runs as
case.run(lib, nsm, alloc): nsm = the device's SM count (132 on an H100 and in the emulation build), alloc(a) = (address,
fetch) of a copy of the array a in device memory.

Branches inside a kernel cannot be seen from the launch profiler; each case asserts the predicate it exists for, with the
host's rules restated below (the constants are read from the kernel sources, so a change of the plan fails here instead of
moving a case quietly into another branch):
  - emb_plan (r <= 32, balanced panels): the M contraction k_emb_mstep_constr<NCB> runs one CTA per EMB_TILE = 64 series
    (ntM tiles) and time split (tsM splits of tper periods, the last CTA to arrive sums the splits); NCB = ceil(r / 8);
    thread 0 of each tile corrects the tile's restricted series one at a time after the thread-per-series solve;
  - its shared memory is mstep_smem(r) + em_constr_scratch(r) 8 B (mstep_constr_smem), raised past the 48 KiB default
    per call;
  - r > 32 or missing data: k_em_mstep_series, one CTA per series, S_ff downdated by the series' missing periods;
  - ss_check (sampling_dispatch_checks.ss_accepts): r = 37 at p = 1 is refused with status 6."""
import collections
import os
import re

import numpy as np

from dynamic_factor_models_b200._lib import MEM_DEVICE, from_cm, to_cm
from dispatch_checks import KernelLog, case  # noqa: F401  (KernelLog: used by the GPU file)
from identified_dispatch_checks import DEFAULT_SMEM, constr
from sampling_dispatch_checks import _big_model, _code, ss_accepts
import em_constr_checks as CC
import em_constr_oracle as O
from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel

METHODS = ("em_kalman",)
CASES = []
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynamic_factor_models_b200", "csrc")


def _grab(name, pattern, what):
    with open(os.path.join(CSRC, name)) as f:
        m = re.search(pattern, f.read(), re.M)
    assert m, "kernel source changed (%s): update tests/em_constr_dispatch_checks.py" % what
    return m.groups()


# ---------------------------------------------------------------------------------------- the host's size rules, restated
EMB_TILE = int(_grab("dfm_kernels_emb.cuh", r"^#define EMB_TILE (\d+)\b", "EMB_TILE")[0])
EMB_MAXSPLIT = int(_grab("dfm_kernels_emb.cuh", r"^#define EMB_MAXSPLIT (\d+)\b", "EMB_MAXSPLIT")[0])
EMB_RMAX = int(_grab("dfm_api.cu", r"^\s*e\.on = r <= (\d+);", "emb_plan: e.on")[0])
SMM_PAD = int(_grab("dfm_api.cu", r"e\.smM = \(\(size_t\)2 \* r \* r \+ \(size_t\)2 \* EMB_TILE \* \(r \+ 1\) \+ (\d+)\) \* 8;",
                    "emb_plan: e.smM")[0])
_grab("dfm_kernels_em.cuh", r"int em_constr_scratch\(int r\) \{ return (r \* r \+ r \* \(r \+ 1\) / 2 \+ r); \}", "em_constr_scratch")

EmbPlan = collections.namedtuple("EmbPlan", "on ncb ntM tsM tper")


def _cdiv(a, b):
    return -(-a // b)


def emb_plan(T, N, r, B, nsm):
    """The M-contraction plan of emb_plan in dfm_api.cu: (on, NCB, series tiles ntM, time splits tsM, periods per split)."""
    if r > EMB_RMAX:
        return EmbPlan(False, 0, 0, 0, 0)
    target = 2 * nsm
    ntE = _cdiv(T, EMB_TILE)
    ns = max(_cdiv(N, EMB_MAXSPLIT), min(_cdiv(target, ntE * B), _cdiv(N, 32)))
    nper = (_cdiv(N, ns) + 3) & ~3
    nsE = _cdiv(N, nper)
    ntM = _cdiv(N, EMB_TILE)
    ts = max(1, min(_cdiv(target, ntM * B), _cdiv(T, 32)))
    tper = (_cdiv(T, ts) + 3) & ~3
    tsM = _cdiv(T, tper)
    if nsE * B > 65535 or tsM * B > 65535:
        return EmbPlan(False, 0, 0, 0, 0)
    return EmbPlan(True, _cdiv(r, 8), ntM, tsM, tper)


def em_constr_scratch(r):
    return r * r + r * (r + 1) // 2 + r


def mstep_smem(r):
    """Shared memory of k_emb_mstep<NCB> (EmbPlan::smM)."""
    return (2 * r * r + 2 * EMB_TILE * (r + 1) + SMM_PAD) * 8


def mstep_constr_smem(r):
    """Shared memory of k_emb_mstep_constr<NCB>: smM and lam_constr_correct's scratch."""
    return mstep_smem(r) + em_constr_scratch(r) * 8


def cluster(B, nsm):
    """CTAs per panel of k_em_filter_smooth (fs_cluster_size)."""
    return next((c for c in (8, 4, 2) if B * c <= nsm), 1)


assert emb_plan(150, 200, 32, 1, 132)[2:] == (4, 5, 32) and emb_plan(150, 200, 32, 300, 132).tsM == 1
assert emb_plan(200, 70, 12, 1, 132)[2:4] == (2, 7)
assert mstep_constr_smem(26) == 47656 and (mstep_constr_smem(27), mstep_smem(27)) == (50176, 41104)
assert (mstep_constr_smem(32), mstep_smem(32)) == (63616, 50944)


# ---------------------------------------------------------------------------------------------------- kernel sets
FS = "k_em_filter_smooth"
FUSED = ("k_em_fused<RT>", "k_em_fused2<RT>")
EMB_K = ("k_emb_contract<NCB>", "k_emb_mstep_constr<NCB>", "k_emb_mstep<NCB>", "k_emb_close", "k_emb_cinit")
EMB_C = {"em_kalman": (("k_emb_contract<NCB>", "k_emb_mstep_constr<NCB>", "k_emb_close", "k_em_prep", FS),
                       ("k_emb_mstep<NCB>", "k_em_mstep_series", "k_em_contract", "k_em_contract_bal") + FUSED)}
# (without the multi-CTA contraction the host does not count the panels with missing data, so k_em_contract is launched
#  as well and returns at once for balanced panels: dispatch_checks.GEN_BAL)
GEN_C = {"em_kalman": (("k_em_contract_bal", "k_em_mstep_series", "k_em_prep", FS), EMB_K + FUSED)}
MISS_C = {"em_kalman": (("k_em_contract", "k_em_mstep_series", "k_em_prep", FS),
                        ("k_emb_contract<NCB>", "k_emb_mstep_constr<NCB>", "k_emb_mstep<NCB>", "k_em_contract_bal") + FUSED)}
# a mixed batch, or a balanced and a missing-data call in one case
MIXED_C = {"em_kalman": (tuple(sorted(set(EMB_C["em_kalman"][0]) | set(MISS_C["em_kalman"][0]))),
                         ("k_emb_mstep<NCB>", "k_em_contract_bal") + FUSED)}
EMB_AND_PLAIN = {"em_kalman": (EMB_C["em_kalman"][0] + ("k_emb_mstep<NCB>",),
                               tuple(k for k in EMB_C["em_kalman"][1] if k != "k_emb_mstep<NCB>"))}


def em_constr_case(id_, kernels):
    return case(id_, kernels, table=CASES)


# ---------------------------------------------------------------------------------------------------- the comparison
PAR_TOL = 1e-8


def compare_full(got, ref, cons, par_tol=PAR_TOL, ll_rtol=1e-10):
    """One panel's results against em_constr_oracle.em_kalman from the same start: em_constr_checks.compare (log-likelihood
    rtol ll_rtol and monotone from iteration 1, Lam / R / A / Q / F within par_tol of max |ref|, each series' restriction to
    1e-12) on the iterations the spec ran (NaN log-likelihood beyond them), PF and P0 at the bars of
    parity_checks.compare_em, status 0 and the spec's iteration count; series out of the model keep NaN loadings, and a
    pinned series (m = r rows) has Lam_i = H_i^-1 h_i to 1e-12."""
    n = ref["iters"]
    assert got["status"] == 0 and got["iters"] == n, (got["status"], got["iters"], n)
    assert np.isnan(got["loglik"][n:]).all(), got["loglik"][n:]
    CC.compare(dict(got, loglik=got["loglik"][:n]), ref, cons, par_tol, ll_rtol)
    np.testing.assert_allclose(got["PF"], ref["PsF"], rtol=1e-7, atol=1e-10, err_msg="PF")
    np.testing.assert_allclose(got["P0"], ref["P0"], rtol=1e-9, atol=1e-11, err_msg="P0")
    out = np.isnan(ref["R"])
    assert np.isnan(got["Lam"][out]).all()
    N, r = got["Lam"].shape
    for i, (Hi, hi) in O.by_series(cons, N).items():
        if len(hi) == r and not out[i]:
            lam = np.linalg.solve(Hi, hi)
            np.testing.assert_allclose(got["Lam"][i], lam, rtol=0, atol=1e-12 * max(1.0, np.abs(lam).max()), err_msg="pinned %d" % i)


def model(N, r, T, p, miss=0.0, ragged=0, exclude=(), rep=5):
    """A simulated standardized panel (missing_frac miss; the last `ragged` periods of the first half of the series missing)
    and its start from PCA factors (oracle init_from_factors); the series in `exclude` out of the model (NaN loadings)."""
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    if ragged:
        X[T - ragged:, :N // 2] = np.nan
    Lam, Rv, A, Q = K.init_from_factors(X, R.pca_score(np.nan_to_num(X), r), p)
    Lam[list(exclude)] = np.nan
    return X, (Lam, Rv, A, Q)


def check(lib, X, th, p, cons, iters=3, tol=0.0):
    """The device call against the spec from the same start (compare_full); returns (device, spec)."""
    ref = O.em_kalman(X, *th, p=p, max_iter=iters, tol=tol, constr=cons)
    got = lib.em_kalman(X, *th, p=p, max_iter=iters, tol=tol, constr=cons)
    compare_full(got, ref, cons)
    return got, ref


def _restricted(cons, N):
    return sorted(O.by_series(cons, N))


def _close(a, b, rtol, what):
    """max |a - b| <= rtol * max(1, max |b|) (NaN where b is NaN)."""
    assert (np.isnan(a) == np.isnan(b)).all(), what
    if not np.isnan(b).all():
        err = np.nanmax(np.abs(a - b))
        assert err <= rtol * max(1.0, np.nanmax(np.abs(b))), (what, err)


OUTS = ("Lam", "R", "A", "Q", "P0", "F", "PF", "loglik")

# rows of the k = 48 cases: series 0 pinned (m = r = 12), 63 with m = 11 (the last series of tile 0), three Gaussian rows on
# 64 (the first series of tile 1), one row on the last series 69 and one on the excluded series 5 (ignored)
ROWS70 = ((0, 12, True), (63, 11, True), (64, 3, False), (69, 1, True), (5, 1, True))


# ---------------------------------------------------------------------------------------------------- 1. k_emb_mstep_constr
@em_constr_case("emb_k48_r12_p4", EMB_C)
def _(lib, nsm, alloc):
    # (N, r, p, T) = (70, 12, 4, 200): NCB = 2, two series tiles (64 + 6), tsM = 7 splits of 32 periods, the last with 8;
    # restricted series in both tiles and at both edges of tile 0
    T, N, r, p = 200, 70, 12, 4
    e = emb_plan(T, N, r, 1, nsm)
    assert e.on and (e.ncb, e.ntM, e.tsM, e.tper) == (2, 2, 7, 32) and T - (e.tsM - 1) * e.tper == 8 and N % EMB_TILE == 6
    X, th = model(N, r, T, p, exclude=(5,))
    cons = constr(r, ROWS70)
    assert [i // EMB_TILE for i in _restricted(cons, N)] == [0, 0, 0, 1, 1]
    check(lib, X, th, p, cons)


@em_constr_case("emb_r24_p1_N200", EMB_C)
def _(lib, nsm, alloc):
    # (200, 24, 1, 150): NCB = 3, four series tiles, the last with 8 series; 5 splits of 32 periods (the last 22); rows on
    # series 0 (pinned, m = 24), 63 (m = 23), 64, 127, 128 and 199 (the last series of the ragged tile), and on the excluded
    # 100.  (p = 1: at p = 2, k = 48, the filter's shared-memory plan refuses r = 24 -- ss_check.)
    T, N, r, p = 150, 200, 24, 1
    e = emb_plan(T, N, r, 1, nsm)
    assert e.on and (e.ncb, e.ntM, e.tsM) == (3, 4, 5) and N % EMB_TILE == 8
    assert ss_accepts(nsm, 1, r, p) and not ss_accepts(nsm, 1, r, 2)
    X, th = model(N, r, T, p, exclude=(100,), rep=6)
    cons = constr(r, ((0, 24, True), (63, 23, True), (64, 2, False), (127, 5, True), (128, 1, True), (199, 3, False), (100, 1, True)))
    assert {i // EMB_TILE for i in _restricted(cons, N)} == {0, 1, 2, 3}
    check(lib, X, th, p, cons, iters=3)


@em_constr_case("emb_r27_attr", EMB_AND_PLAIN)
def _(lib, nsm, alloc):
    # k_emb_mstep_constr<4>'s attribute is the kernel's for the whole process and is set per call: restricted r = 27
    # (50 176 B > 48 KiB; without the restriction 41 104 B would fit the default), unrestricted r = 27 (k_emb_mstep<4>),
    # restricted r = 26 (47 656 B, under the default), restricted r = 27 again -- each against the spec
    T, N = 120, 90
    assert mstep_constr_smem(27) == 50176 > DEFAULT_SMEM >= mstep_smem(27) == 41104
    assert mstep_constr_smem(26) == 47656 <= DEFAULT_SMEM
    for r in (26, 27):
        e = emb_plan(T, N, r, 1, nsm)
        assert e.on and e.ncb == 4 and e.ntM == 2
    X27, th27 = model(N, 27, T, 1, rep=7)
    X26, th26 = model(N, 26, T, 1, rep=8)
    c27 = constr(27, ((0, 27, True), (64, 3, False), (89, 1, True)))
    c26 = constr(26, ((0, 26, True), (70, 2, False)))
    first, _ = check(lib, X27, th27, 1, c27, iters=2)
    check(lib, X27, th27, 1, None, iters=2)
    check(lib, X26, th26, 1, c26, iters=2)
    again, _ = check(lib, X27, th27, 1, c27, iters=2)
    for n in OUTS:
        np.testing.assert_array_equal(again[n], first[n], err_msg=n)


@em_constr_case("emb_r32_p1", EMB_C)
def _(lib, nsm, alloc):
    # (200, 32, 1, 150): NCB = 4, the largest r of the multi-CTA path, 63 616 B of shared memory; series 0 pinned by an
    # invertible 32 x 32 H (lam_constr_correct's packed G is 32 x 32), series 1 with m = 31, two Gaussian rows on series 199
    T, N, r = 150, 200, 32
    e = emb_plan(T, N, r, 1, nsm)
    assert e.on and (e.ncb, e.ntM, e.tsM) == (4, 4, 5) and mstep_constr_smem(r) == 63616
    X, th = model(N, r, T, 1, rep=9)
    check(lib, X, th, 1, constr(r, ((0, 32, True), (1, 31, True), (199, 2, False))), iters=2)


@em_constr_case("emb_every_series", EMB_C)
def _(lib, nsm, alloc):
    # (70, 3, 1, 120): every series restricted, m cycling 1, 2, 3 (m = 3 pins the series): the thread-per-series loop
    # finishes no series, thread 0 corrects all 64 of tile 0 and the 6 of tile 1
    T, N, r = 120, 70, 3
    e = emb_plan(T, N, r, 1, nsm)
    assert e.on and (e.ncb, e.ntM) == (1, 2) and N - EMB_TILE == 6
    X, th = model(N, r, T, 1, rep=10)
    cons = constr(r, tuple((i, i % 3 + 1, i % 3 == 2 or i % 2 == 0) for i in range(N)))
    assert _restricted(cons, N) == list(range(N))
    check(lib, X, th, 1, cons, iters=4)


# ---------------------------------------------------------------------------------------------------- 2. k_em_mstep_series
@em_constr_case("general_r36_balanced", GEN_C)
def _(lib, nsm, alloc):
    # r = 36 > 32: no multi-CTA contraction, the balanced panel takes k_em_contract_bal and k_em_mstep_series; r = 36 is the
    # largest r ss_check accepts at p = 1, r = 37 is refused (status 6) before any launch.  Series 0 pinned (a 36 x 36 G),
    # series 3 with m = 35, one Gaussian row on the last series
    T, N, r = 150, 120, 36
    assert not emb_plan(T, N, r, 1, nsm).on and ss_accepts(nsm, 1, r, 1) and not ss_accepts(nsm, 1, 37, 1)
    m = _big_model(N, 37, 1, 60)
    c37 = constr(37, ((0, 1, True),))
    assert _code(lambda: lib.em_kalman(m["X"], m["Lam"], m["R"], m["A"], m["Q"], p=1, max_iter=2, constr=c37)) == 6
    X, th = model(N, r, T, 1, rep=11)
    check(lib, X, th, 1, constr(r, ((0, 36, True), (3, 35, True), (119, 1, False))), iters=2)


@em_constr_case("missing_k48_r12_p4", MISS_C)
def _(lib, nsm, alloc):
    # ROWS70 on a panel with 5 % missing cells and a ragged edge of 3 periods; series 64 (three Gaussian rows) keeps 8 < r
    # observations, thinned after the start was computed (init_from_factors drops a series with <= r observations): its S_ff
    # is k_em_mstep_series' downdate of S_ff by 192 missing periods
    T, N, r, p = 200, 70, 12, 4
    X, th = model(N, r, T, p, miss=0.05, ragged=3, exclude=(5,), rep=12)
    keep = np.flatnonzero(~np.isnan(X[:, 64]))[::20][:8]
    thin = np.full(T, np.nan); thin[keep] = X[keep, 64]
    X[:, 64] = thin
    assert np.count_nonzero(~np.isnan(X[:, 64])) == 8 < r and not np.isnan(th[0][64]).any()
    check(lib, X, th, p, constr(r, ROWS70))


@em_constr_case("mixed_batch_r12_p2", MIXED_C)
def _(lib, nsm, alloc):
    # (70, 12, 2, 80), 4 panels, balanced and 5 %-missing alternating: every iteration runs k_emb_mstep_constr on panels 0, 2
    # and k_em_mstep_series on 1, 3 (skip_bal); tsM = 3 for the batch as for one panel.  Each panel against the spec and its
    # one-panel call (1e-10)
    T, N, r, p, B = 80, 70, 12, 2, 4
    assert emb_plan(T, N, r, B, nsm).tsM == emb_plan(T, N, r, 1, nsm).tsM == 3
    pans = [model(N, r, T, p, miss=0.05 * (b % 2), exclude=(5,), rep=20 + b) for b in range(B)]
    cons = constr(r, ROWS70)
    Xb = np.stack([x for x, _ in pans])
    thb = [np.stack([t[j] for _, t in pans]) for j in range(4)]
    got = lib.em_kalman(Xb, *thb, p=p, max_iter=3, constr=cons)
    for b, (X, th) in enumerate(pans):
        mine = {n: got[n][b] for n in OUTS + ("iters", "status")}
        one = lib.em_kalman(X, *th, p=p, max_iter=3, constr=cons)
        for n in OUTS:
            _close(mine[n], one[n], 1e-10, (n, b))
        compare_full(mine, O.em_kalman(X, *th, p=p, max_iter=3, constr=cons), cons)


@em_constr_case("few_vs_many_r12", EMB_C)
def _(lib, nsm, alloc):
    # (70, 12, 1, 60): one panel (an 8-CTA cluster filter, tsM = 2) against the same panel at positions 0 and 132 of a
    # 133-panel call (133 > nsm: no cluster, tsM = 1); 1e-10, and each against the spec
    T, N, r, B = 60, 70, 12, 133
    assert emb_plan(T, N, r, 1, nsm).tsM == 2 and emb_plan(T, N, r, B, nsm).tsM == 1
    assert cluster(1, nsm) == 8 and cluster(B, nsm) == 1
    X, th = model(N, r, T, 1, exclude=(5,), rep=13)
    cons = constr(r, ROWS70)
    ref = O.em_kalman(X, *th, p=1, max_iter=3, constr=cons)
    one = lib.em_kalman(X, *th, p=1, max_iter=3, constr=cons)
    compare_full(one, ref, cons)
    many = lib.em_kalman(np.stack([X] * B), *(np.stack([t] * B) for t in th), p=1, max_iter=3, constr=cons)
    for b in (0, B - 1):
        mine = {n: many[n][b] for n in OUTS + ("iters", "status")}
        for n in OUTS:
            _close(mine[n], one[n], 1e-10, (n, b))
        compare_full(mine, ref, cons)


# ---------------------------------------------------------------------------------------------------- 3. stopping, rows
def crossing_tol(X, th, p, cons, max_iter=40):
    """(tol, j): a tol at which the spec stops at iteration j with a margin -- its relative change at j is <= tol / 2 and at
    every iteration 2 .. j - 1 > 2 tol."""
    ll = O.em_kalman(X, *th, p=p, max_iter=max_iter, constr=cons)["loglik"]
    d = np.abs(np.diff(ll)) / (0.5 * (np.abs(ll[1:]) + np.abs(ll[:-1])))      # d[j - 2]: the change at iteration j
    for j in range(3, max_iter + 1):
        lo, hi = 2.0 * d[j - 2], 0.5 * d[:j - 2].min()
        if lo < hi:
            return float(np.sqrt(lo * hi)), j
    raise AssertionError("no iteration with a margin: %s" % d)


@em_constr_case("tol_stop", MIXED_C)
def _(lib, nsm, alloc):
    # (40, 12, 2, 120): tol > 0 on a balanced (multi-CTA) and a 5 %-missing (k_em_mstep_series) panel: the device stops at the
    # spec's iteration (NaN log-likelihood beyond it)
    T, N, r, p = 120, 40, 12, 2
    assert emb_plan(T, N, r, 1, nsm).on
    cons = constr(r, ((0, 12, True), (7, 3, False), (39, 1, True)))
    for miss, rep in ((0.0, 14), (0.05, 15)):
        X, th = model(N, r, T, p, miss=miss, rep=rep)
        tol, j = crossing_tol(X, th, p, cons)
        ref = O.em_kalman(X, *th, p=p, max_iter=40, tol=tol, constr=cons)
        assert ref["iters"] == j
        compare_full(lib.em_kalman(X, *th, p=p, max_iter=40, tol=tol, constr=cons), ref, cons)


def _interleave(cons):
    """The rows of cons with the series dealt round-robin (each series' own rows in their order)."""
    idx = np.asarray(cons[0])
    groups = [list(np.flatnonzero(idx == i)) for i in sorted(set(idx.tolist()))]
    order = [g[k] for k in range(max(map(len, groups))) for g in groups if k < len(g)]
    assert order != sorted(order)
    return idx[order], cons[1][order], cons[2][order]


@em_constr_case("row_order", EMB_C)
def _(lib, nsm, alloc):
    # (70, 12, 1, 60): rows of different series interleaved, each series' own order kept, give the grouped call's bits
    # (constr_csr builds the same CSR); series 63's 11 rows reversed: 1e-12 of the grouped call, and the spec
    T, N, r = 60, 70, 12
    X, th = model(N, r, T, 1, exclude=(5,), rep=16)
    cons = constr(r, ROWS70)
    base, _ = check(lib, X, th, 1, cons)
    mixed = lib.em_kalman(X, *th, p=1, max_iter=3, constr=_interleave(cons))
    for n in OUTS:
        np.testing.assert_array_equal(mixed[n], base[n], err_msg=n)
    idx, H, h = cons
    sel = np.flatnonzero(idx == 63)
    order = np.arange(len(idx)); order[sel] = sel[::-1]
    rev = (idx[order], H[order], h[order])
    got, _ = check(lib, X, th, 1, rev)
    for n in OUTS:
        _close(got[n], base[n], 1e-12, n)


def near_rows(r, series, delta, seed=17):
    """Two rows on `series`: u and u + delta v (u, v orthonormal), with values c and c + delta d: the solution stays O(1)
    while the rows' relative Gram pivot (the pivot of H H') is delta^2 / (1 + delta^2)."""
    rng = np.random.default_rng(seed)
    U, _ = np.linalg.qr(rng.standard_normal((r, 2)))
    u, v = U[:, 0], U[:, 1]
    c, d = 0.3 * rng.standard_normal(2)
    return np.array([series, series], np.int32), np.vstack([u, u + delta * v]), np.array([c, c + delta * d])


@em_constr_case("near_dependent_rows", MIXED_C)
def _(lib, nsm, alloc):
    # (40, 12, 1, 60) balanced (multi-CTA) and 5 %-missing (k_em_mstep_series): rows 1e-3 apart on series 2 (relative pivot
    # of H H' 1e-6, of G = H S^-1 H' near it: far above the 1e-12 test) are accepted and match the spec; rows 1e-9 apart
    # (relative pivot 1e-18, rounding leaves ~1e-16) give status 3 on the device and ConstraintSingular in the spec
    T, N, r = 60, 40, 12
    assert emb_plan(T, N, r, 1, nsm).on
    for delta, ok in ((1e-3, True), (1e-9, False)):
        _, H, _ = cons = near_rows(r, 2, delta)
        G = H @ H.T
        piv = (G[1, 1] - G[0, 1] ** 2 / G[0, 0]) / G[1, 1]
        assert (piv > 1e-7) if ok else (piv < 1e-15), piv
        for miss, rep in ((0.0, 18), (0.05, 19)):
            X, th = model(N, r, T, 1, miss=miss, rep=rep)
            if ok:
                check(lib, X, th, 1, cons)
            else:
                try:
                    O.em_kalman(X, *th, p=1, max_iter=1, constr=cons)
                    raise AssertionError("the spec accepted rows %g apart" % delta)
                except O.ConstraintSingular:
                    pass
                assert lib.em_kalman(X, *th, p=1, max_iter=3, constr=cons)["status"] == 3


@em_constr_case("mem_device_emb", EMB_C)
def _(lib, nsm, alloc):
    # (70, 12, 2, 80) balanced, the multi-CTA path: every input and output in device memory gives the host call's bits
    T, N, r, p, it = 80, 70, 12, 2, 3
    k = r * p
    assert emb_plan(T, N, r, 1, nsm).on
    X, th = model(N, r, T, p, exclude=(5,), rep=22)
    cons = constr(r, ROWS70)
    ref, _ = check(lib, X, th, p, cons, iters=it)
    ins = dict(X=to_cm(X), Lam=to_cm(th[0]), R=np.ascontiguousarray(th[1]), A=to_cm(th[2]), Q=to_cm(th[3]))
    dev = {n: alloc(a)[0] for n, a in ins.items()}
    size = dict(Lam=N * r, R=N, A=r * k, Q=r * r, P0=k * k, F=T * r, PF=T * r * r, loglik=it)
    outs = {n: alloc(np.full(s, np.nan)) for n, s in size.items()}
    outs.update(iters=alloc(np.zeros(1, np.int32)), status=alloc(np.ones(1, np.int32)))
    lib.em_kalman_raw(dev["X"], T, N, r, p, 1, it, 0.0, {n: dev[n] for n in ("Lam", "R", "A", "Q")},
                      {n: o[0] for n, o in outs.items()}, MEM_DEVICE, constr=cons)
    lib.sync()
    got = {n: o[1]() for n, o in outs.items()}
    shape = dict(Lam=(N, r), A=(r, k), Q=(r, r), P0=(k, k), F=(T, r))
    for n in size:
        g = from_cm(got[n], *shape[n]) if n in shape else got[n].reshape(np.shape(ref[n]))
        np.testing.assert_array_equal(g, ref[n], err_msg=n)
    assert int(got["status"][0]) == 0 and int(got["iters"][0]) == it
