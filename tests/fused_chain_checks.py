"""Oracle checks of the fused EM kernels (k_em_fused2, path 3; k_em_fused, path 2) in the regimes their covariance chain
selects.  Both kernels run the covariance recursion explicitly only until P_{t|t-1} stops changing (relative 1e-14) and
treat the rest of the panel as a frozen range; the number of explicit steps nE then picks code paths inside the kernel:
  - explicit steps read from the idle ring (t < F2_NEXS(r)) or from global scratch (path 3);
  - a chain that never freezes (nE == T): no frozen-range scans, per-period likelihood over all T;
  - the likelihood of the explicit periods in two stages (`split`) or one thread per period (path 3);
  - the chunking of the parallel-in-time scans over the frozen range n = T - nE (blk_recur: 28 eight-lane groups and a
    Kogge-Stone boundary scan on path 3, 16 groups and a serial boundary chain on path 2);
  - the backward convergence point tb (-1 when the smoothed chain has not converged by lo = nE - 1).
Strong-signal panels freeze after 5..8 steps, so the ordinary parity tests reach none of these.  chain_plan restates the
kernels' freeze rules, chain_model builds state-space models with a chosen Riccati speed, and CASES runs each regime
against the oracle: test_emu_fused_chain.py on the host-emulation build, test_gpu_fused_chain.py on the H100 with the
kernel-set assertion.  The geometry constants are read from the kernel sources, so a change of the stage geometry fails
the planner's assertions instead of moving the cases quietly into other branches."""
import collections
import functools
import os
import re

import numpy as np

from oracle import kalman_em as K
import dispatch_checks as DC
import parity_checks as P

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynamic_factor_models_b200", "csrc")
EPS = 1e-14                                       # freeze tolerance of chain_fwd / chain_bwd
MARGIN = 1.5                                      # dmax / (EPS pmax) must clear 1 by this factor around the freeze


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _grab(src, pattern, what):
    m = re.search(pattern, src, re.M)
    assert m, "kernel source changed (%s): update tests/fused_chain_checks.py" % what
    return m.groups()


def _geometry():
    f2, f1, api = _src("dfm_kernels_fused2.cuh"), _src("dfm_kernels_fused.cuh"), _src("dfm_api.cu")
    g = {}
    g["SBS"] = int(_grab(f2, r"^#define F2_SBS (\d+)\b", "F2_SBS")[0])
    s_num, = _grab(f2, r"^#define F2_S \((\d+) / F2_SBS\)", "F2_S")
    g["S"] = int(s_num) // g["SBS"]
    g["TC"] = int(_grab(f2, r"^#define F2_TC (\d+)\b", "F2_TC")[0])
    _grab(f2, r"^#define F2_TS F2_TC\b", "F2_TS")
    g["NCW"] = int(_grab(f2, r"^#define F2_NCW (\d+)\b", "F2_NCW")[0])
    g["GPARTS_S"] = int(_grab(f2, r"^#define F2_GPARTS_S (\d+)\b", "F2_GPARTS_S")[0])
    _grab(f2, r"^#define F2_GPARTS \(\(R == 8\) \? \(F2_NCW \+ 1\) : F2_GPARTS_S\)", "F2_GPARTS")
    _grab(f2, r"^#define F2_PNT_GPU \(\(F2_NCW \+ 1\) \* 32\)", "F2_PNT_GPU")
    _grab(f2, r"^#define F2_NEXS\(R_\) \(\(F2_S \* F2_STG - 4 \* \(R_\) \* \(R_\)\) / FUSED_SCR\(R_\)\)", "F2_NEXS")
    a, c = _grab(f1, r"^#define FUSED_SCR\(R_\) \((\d+) \* \(R_\) \* \(R_\) \+ (\d+)\)", "FUSED_SCR")
    g["SCR"] = (int(a), int(c))
    g["BND"], = _grab(f2, r"const bool split = gram && 2 \* nE \* R <= \((\d+) \* R \+ RR\) - \(F2_GPARTS \+ 1\) \* RR;", "split")
    g["BND"] = int(g["BND"])
    g["F2_THREADS"], g["F2_MINB"] = map(int, _grab(f2, r"__launch_bounds__\((\d+), (\d+)\)", "k_em_fused2 launch bounds"))
    g["F1_THREADS"], g["F1_MINB"] = map(int, _grab(f1, r"__launch_bounds__\((\d+), (\d+)\)", "k_em_fused launch bounds"))
    _grab(f1, r"blk_recur<R>\(Z, Tp, Phinf, T1, T2, bnd, \(nE > 0 \? nE : 1\), T - \(nE > 0 \? nE : 1\), \+1, (128)\)", "k_em_fused scan")
    g["SMEM_CAP"] = int(_grab(api, r"return need <= (\d+) \* 1024;\s+// two CTAs per SM", "fused2_shape_ok")[0]) * 1024
    return g


G = _geometry()
STG = G["SBS"] * 8 * G["TC"]                      # doubles per ring stage
GROUPS3 = (G["NCW"] + 1) * 32 // 8                # 8-lane groups of blk_recur in k_em_fused2 (warps 0..NCW)
GROUPS2 = G["F1_THREADS"] // 8                    # ... in k_em_fused (the whole CTA)


def fused_scr(r):
    return G["SCR"][0] * r * r + G["SCR"][1]


def nexs(r):
    """Explicit covariance steps k_em_fused2 keeps in its idle ring; later steps live in global scratch."""
    return (G["S"] * STG - 4 * r * r) // fused_scr(r)


def gparts(r):
    return G["NCW"] + 1 if r == 8 else G["GPARTS_S"]


def blk_chunk_len(n, ng):
    Lc = (n + ng - 1) // ng
    return Lc + 1 if Lc > 1 and Lc % 2 == 0 else Lc


def pad4mod16(x):
    return x + ((4 - x % 16) + 16) % 16


def fused2_shape_ok(T, N, r):
    """dfm_api.cu fused2_shape_ok (p = 1): the shared-memory plan of k_em_fused2 fits two CTAs per SM."""
    if r < 1 or r > 8 or T < 4 or T % 2:
        return False
    need = (8 * pad4mod16(T) + r * pad4mod16(N) + 3 * N + 30 * r * r + 2 * r + max(97 * r + r * r, 2 * G["NCW"] * 72) +
            G["S"] * STG + 106) * 8
    return need <= G["SMEM_CAP"]


def als_fused2_shape_ok(T, N, r):
    """dfm_api.cu als_fused2_shape_ok: the shared-memory plan of k_als_fused2."""
    if r < 1 or r > 8 or T < 4 or T % 2:
        return False
    need = (8 * pad4mod16(T) + r * pad4mod16(N) + N + 4 * r * r + 2 * r + 48 + 2 * G["NCW"] * 72 + G["S"] * STG + 32) * 8
    return need <= G["SMEM_CAP"]


def t_max(ok, N, r):
    """Largest even T the shape rule `ok` accepts (the rule is monotone in T)."""
    T = 4
    while ok(T + 2, N, r):
        T += 2
    return T


def fused2_smem_bytes(T, N, r):
    """dfm_kernels_fused2.cuh fused2_smem_doubles, in bytes."""
    return (8 * pad4mod16(T) + r * pad4mod16(N) + 3 * N + 30 * r * r + 2 * r + 40 + 8 + 8 +
            max(97 * r + r * r, 2 * G["NCW"] * 72) + G["S"] * STG + 26) * 8


def fused_smem_bytes(T, N, r):
    """dfm_kernels_fused.cuh fused_smem_doubles, in bytes."""
    return (8 * pad4mod16(T) + r * pad4mod16(N) + 3 * N + 30 * r * r + 2 * r + 40 + 8 + 8 + 64 * r + r * r + 8) * 8


def fused_resident_per_sm(T, N, r, smem_per_sm=228 * 1024, reserved=1024):
    """CTAs of k_em_fused per SM when shared memory is the binding limit (H100: 228 KB per SM, 1 KB reserved per CTA).
    __launch_bounds__(128, 3) guarantees registers for at least F1_MINB CTAs, so between F1_MINB and this count the
    shared memory decides, and cudaOccupancyMaxActiveBlocksPerMultiprocessor (resident_grid) returns exactly it."""
    return smem_per_sm // (fused_smem_bytes(T, N, r) + reserved)


# ------------------------------------------------------------------------------------------------------ the planner
Plan = collections.namedtuple("Plan", "nE frozen frozen_at tb lo spill split n Lc3 nch3 levels3 Lc2 nch2 margin ratios")


def _sym(A):
    return 0.5 * (A + A.T)


def chain_plan(Lam, R, A, Q, P0, T, r):
    """The covariance chain of k_em_fused2 / k_em_fused (chain_fwd, chain_bwd; P2 of k_em_fused) for a balanced panel,
    restated step for step: information form (Pi = Pp^-1, W = Pi + C, Pf = W^-1), freeze test max|Pp_{t+1} - Pp_t| <=
    1e-14 max|Pp_t| at step t (frozen_at), one more step after it (nE = frozen_at + 2), backward convergence test
    max|Ps_t - Ps_{t+1}| <= 1e-14 max|Ps_t| for t > lo.  Returns the branch quantities and the margin: the smaller of
    dmax / (1e-14 pmax) at the step before the freeze and its inverse at the freeze step (for a chain that never freezes,
    the smallest dmax / (1e-14 pmax) of the steps that could still have frozen it).  ratios: dmax / (1e-14 pmax) per step."""
    M = np.asarray(A, float).reshape(r, r)
    C = Lam.T @ (Lam / R[:, None])
    Pp = np.array(P0, float)
    Pfs, Js, ratios = [], [], []
    nE, frozen_at, t, Pfprev = T, -1, 0, None
    Pfinf = Jinf = None
    while t < T:
        Pi = np.linalg.inv(Pp)
        Pf = np.linalg.inv(Pi + C)
        if t >= 1:
            Js.append(Pfprev @ M.T @ Pi)                               # J_{t-1}
        Pn = _sym(M @ Pf @ M.T + Q)
        Pfs.append(Pf)
        ratios.append(np.abs(Pn - Pp).max() / (EPS * np.abs(Pp).max()))
        Pfprev = Pf
        if frozen_at >= 0 and t == frozen_at + 1:
            nE = t + 1
            Pfinf, Jinf = Pf, Pf @ M.T @ Pi
            break
        if frozen_at < 0 and ratios[-1] <= 1.0:
            frozen_at = t
        Pp = Pn
        t += 1
    frozen = nE < T
    if frozen:
        margin = min(ratios[frozen_at - 1] if frozen_at >= 1 else np.inf, 1.0 / max(ratios[frozen_at], 1e-300))
    else:
        margin = min(ratios[:T - 2]) if T > 2 else np.inf
    # backward chain: only its convergence point is needed
    Psn = Pfinf if frozen else Pfs[T - 1]
    lo = nE - 1 if frozen else T
    tb, t = -1, T - 2
    while t > lo:
        pf_t = Pfs[t] if t < nE else Pfinf
        j_t = Js[t] if t < nE - 1 else Jinf
        D = _sym(Psn - (M @ pf_t @ M.T + Q))
        Ps = _sym(j_t @ D @ j_t.T + pf_t)
        conv = np.abs(Ps - Psn).max() <= EPS * np.abs(Ps).max()
        Psn = Ps
        if conv:
            tb = t
            break
        t -= 1
    gram = frozen and 1 <= nE < T
    split = gram and 2 * nE * r <= (G["BND"] * r + r * r) - (gparts(r) + 1) * r * r
    n = T - nE if frozen else 0
    Lc3 = blk_chunk_len(n, GROUPS3) if n else 0
    nch3 = -(-n // Lc3) if n else 0
    Lc2 = blk_chunk_len(n, GROUPS2) if n else 0
    nch2 = -(-n // Lc2) if n else 0
    levels3 = sum(1 for lvl in range(5) if (1 << lvl) < nch3)     # Kogge-Stone levels of the boundary scan
    return Plan(nE, frozen, frozen_at, tb, lo, nE > nexs(r), split, n, Lc3, nch3, levels3, Lc2, nch2, margin, ratios)


def oracle_freeze(X, Lam, R, A, Q, P0):
    """nE from the oracle's own filter: the first t whose predicted covariance Pp[t+1] meets the freeze rule, plus two."""
    es = K.e_step(X, Lam, R, A, Q, P0, 1)
    Pp = es["Pp"]
    for t in range(len(Pp) - 1):
        if np.abs(Pp[t + 1] - Pp[t]).max() <= EPS * np.abs(Pp[t]).max():
            return min(t + 2, len(Pp))
    return len(Pp)


# ------------------------------------------------------------------------------------------------- the model builder
Model = collections.namedtuple("Model", "X Lam R A Q P0 plan scale")


def _orth(rng, n, k):
    q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    return q


def model_params(r, N, scale, a, spec, seed):
    """State-space parameters with spectrum(C = Lam' R^-1 Lam) = scale * spec, transition A = U diag(a) U' (eigenvalues
    a, rotated: not diagonal), Q = U diag(1 - a^2) U' (unit stationary variance), P0 = the oracle's Lyapunov doubling."""
    rng = np.random.default_rng(seed)
    U = _orth(rng, r, r)
    A = U @ np.diag(a) @ U.T
    Q = _sym(U @ np.diag(1.0 - np.asarray(a) ** 2) @ U.T)
    R = rng.uniform(0.5, 1.5, N)
    Lam = np.sqrt(R)[:, None] * (_orth(rng, N, r) * np.sqrt(scale * np.asarray(spec))) @ _orth(rng, r, r).T
    P0 = K.lyapunov_doubling(A, Q)
    return Lam, R, A, Q, P0


def simulate(Lam, R, A, Q, P0, T, seed):
    """A panel drawn from the model itself (f_0 ~ N(0, P0)), so that the EM iterations stay near its parameters."""
    rng = np.random.default_rng(seed + 7919)
    r, N = A.shape[0], Lam.shape[0]
    f = np.linalg.cholesky(P0) @ rng.standard_normal(r)
    Lq = np.linalg.cholesky(Q)
    F = np.empty((T, r))
    for t in range(T):
        if t:
            f = A @ f + Lq @ rng.standard_normal(r)
        F[t] = f
    return F @ Lam.T + rng.standard_normal((T, N)) * np.sqrt(R)


def _spec(r):
    return np.geomspace(1.0, 0.4, r)


def _slow(r, lo=0.93, hi=0.985):
    return np.linspace(hi, lo, r)


@functools.lru_cache(maxsize=None)
def chain_model(r, N, want, T=None, n=None, even=False, a=None, seed=0, Tplan=1200, margin=MARGIN):
    """A model whose chain meets `want` (a predicate name of WANTS) with the margin, and a panel simulated from it.
    T: fixed panel length; n: frozen-range length instead (T = nE + n); even: T must be even (k_em_fused2).  The signal
    scale is bisected for the target and then scanned in 1 % steps around it.  margin: MARGIN, or 0 for a case whose
    branches hold for every nE its predicate allows, with room on both sides (a chain that slows by only a few per cent
    per step near the freeze cannot have the margin)."""
    a = _slow(r) if a is None else np.asarray(a)
    pred, target = WANTS[want]
    Tp = T if T is not None else Tplan
    target = Tp - 1 if target is None else target

    def plan(s):
        Lam, R, A, Q, P0 = model_params(r, N, s, a, _spec(r), seed)
        return chain_plan(Lam, R, A, Q, P0, Tp, r)

    lo_s, hi_s = 1e-6, 1e4                                       # nE falls as the signal scale grows
    for _ in range(60):
        mid = np.sqrt(lo_s * hi_s)
        if plan(mid).nE > target:
            lo_s = mid
        else:
            hi_s = mid
    for k in sorted(range(-150, 151), key=abs):
        s = hi_s * 1.01 ** k
        p = plan(s)
        if p.margin < margin or not pred(p):
            continue
        TT = T if T is not None else p.nE + n
        if even and TT % 2:
            continue
        Lam, R, A, Q, P0 = model_params(r, N, s, a, _spec(r), seed)
        p = chain_plan(Lam, R, A, Q, P0, TT, r)
        if p.margin < margin or not pred(p):
            continue
        X = simulate(Lam, R, A, Q, P0, TT, seed)
        return Model(X, Lam, R, A, Q, P0, p, s)
    raise AssertionError("no signal scale gives %s at r = %d" % (want, r))


WANTS = {
    # name: (predicate on the plan, nE the bisection aims at)
    "fast": (lambda p: p.frozen and 5 <= p.nE <= 8, 6),
    "short": (lambda p: p.frozen and 7 <= p.nE <= 11, 9),
    "nE16": (lambda p: p.frozen and 14 <= p.nE <= 18, 16),
    "nE20": (lambda p: p.frozen and 18 <= p.nE <= 22, 20),
    "nE35": (lambda p: p.frozen and 33 <= p.nE <= 37, 35),
    "nE40": (lambda p: p.frozen and 36 <= p.nE <= 44, 40),
    "nE700": (lambda p: p.frozen and 700 < p.nE < 760, 720),
    "never": (lambda p: not p.frozen, None),          # (aims at nE = T)
}


# ------------------------------------------------------------------------------------------------------ the checks
def compare_tight(got, ref, X):
    """compare_em plus the bars of this module: log-likelihood rtol 1e-11, F and PF max-abs <= 1e-10 max|ref|."""
    P.compare_em(got, ref, P.ll_atol(X, 1e-13))
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=1e-11, atol=0)
    for g, rf in (("F", "F"), ("PF", "PsF")):
        err = np.abs(got[g] - ref[rf]).max()
        assert err <= 1e-10 * np.abs(ref[rf]).max(), "%s: max abs error %.3g, max |ref| %.3g" % (g, err, np.abs(ref[rf]).max())


def run_em(lib, m, path, iters):
    ref = K.em_kalman(m.X, m.Lam, m.R, m.A, m.Q, p=1, P0=m.P0, max_iter=iters, tol=0.0)
    got = lib.em_kalman(m.X, m.Lam, m.R, m.A, m.Q, p=1, P0=m.P0, max_iter=iters, tol=0.0, path=path)
    assert got["status"] == 0 and got["iters"] == iters, (got["status"], got["iters"])
    compare_tight(got, ref, m.X)
    return got


Case = collections.namedtuple("Case", "id path model expect iters")
CASES = []
F2 = DC.em(("k_em_fused2<RT>",), ("k_em_fused<RT>", DC.FS))
F1 = DC.em(("k_em_fused<RT>",), ("k_em_fused2<RT>", DC.FS))
KERNELS = {0: F1, 2: F1, 3: F2}                  # (path 0 takes k_em_fused at odd T)


def case(id_, path, model, iters=3, **expect):
    """model: keyword arguments of chain_model; expect: Plan fields and the values they must have at iteration 0."""
    CASES.append(Case(id_, path, model, expect, iters))


# r = 8 on both kernels: explicit steps spilled to global scratch with the two-stage likelihood (nE ~ 16), without it
# (nE ~ 40), a chain that never freezes, and frozen ranges around the scan chunking of each kernel
for _p in (3, 2):
    case("p%d_r8_nE16" % _p, _p, dict(r=8, N=20, want="nE16", n=60, even=_p == 3), spill=True, split=True, frozen=True)
    case("p%d_r8_nE40" % _p, _p, dict(r=8, N=20, want="nE40", n=60, even=_p == 3), spill=True, split=False, frozen=True)
    case("p%d_r8_never" % _p, _p, dict(r=8, N=20, want="never", T=60), frozen=False, tb=-1)
# (the long frozen ranges on a chain with nE ~ 16: its Phi_inf^16 is large enough that a scan level left out shows)
for _n in (1, 2, 27, 28, 29, 57):                 # 28 groups: Lc = 1 up to n = 28 (28 chunks: all five levels), then 3
    case("p3_r8_n%d" % _n, 3, dict(r=8, N=20, want="short" if _n < 16 else "nE16", n=_n, even=True), n=_n)
for _n in (1, 15, 16, 17, 33):                    # 16 groups: Lc = 1 up to n = 16, then 3 (17: 6 chunks; 33: 11)
    case("p2_r8_n%d" % _n, 2, dict(r=8, N=20, want="short", n=_n), n=_n)
case("p3_r7_nE20", 3, dict(r=7, N=18, want="nE20", n=80, even=True), spill=True, split=True)
case("p3_r5_nE35", 3, dict(r=5, N=16, want="nE35", n=80, even=True), spill=True, split=True)
case("p3_r3_never_T150", 3, dict(r=3, N=12, want="never", T=150, a=tuple(_slow(3, 0.985, 0.995))), frozen=False)
case("p0_r3_never_T151", 0, dict(r=3, N=12, want="never", T=151, a=tuple(_slow(3, 0.985, 0.995))), frozen=False)
# r = 1 past the 687 ring steps: the chain slows by ~5 % per step near the freeze, so nE may move by a step or two between
# the planner and the device; every nE above 700 takes the same branches
case("p3_r1_nE700", 3, dict(r=1, N=10, want="nE700", n=180, even=True, a=(0.998,), Tplan=2000, margin=0.0), spill=True,
     split=False, iters=2)


def plan_case(c):
    m = chain_model(**c.model)
    for k, v in c.expect.items():
        assert getattr(m.plan, k) == v, "%s: planned %s = %r, wanted %r (%s)" % (c.id, k, getattr(m.plan, k), v, m.plan[:13])
    return m


def run_case(lib, c):
    m = plan_case(c)
    run_em(lib, m, c.path, c.iters)


# ------------------------------------------------------------------------ the existing fused-path shapes freeze early
# (N, r, T) of the fused-path parity and dispatch tests, started as P.check_em starts them (PCA factors of the panel)
EXISTING_SHAPES = ((24, 3, 70), (40, 8, 90), (12, 1, 50), (37, 5, 102), (24, 4, 300), (45, 8, 278), (16, 8, 264),
                   (19, 5, 62), (33, 2, 44), (27, 7, 150), (50, 6, 36), (16, 2, 150), (21, 4, 150), (31, 6, 151),
                   (40, 7, 150), (16, 2, 264), (27, 6, 150), (40, 7, 302))


def existing_shape_nE(N, r, T, iters=3, rep=9):
    """nE of the chain at the parameters of each of the first `iters` EM iterations of a P.check_em run."""
    from oracle import dfm_ref as R
    from oracle.dgp import simulate_panel
    X, _ = simulate_panel(N, r, T, rep=rep)
    Lam, Rv, A, Q = K.init_from_factors(X, R.pca_score(X, r), 1)
    P0 = K.lyapunov_doubling(A, Q)
    out = []
    for _ in range(iters):
        out.append(chain_plan(Lam, Rv, A, Q, P0, T, r).nE)
        es = K.e_step(X, Lam, Rv, A, Q, P0, 1)
        Lam, Rv, A, Q = K.m_step(X, es, r, 1)
    return out


# ---------------------------------------------------------------------------- stage geometry at the 172-period box
# (T, N, r): T at one, one + 2, one + 4, two and three stage widths and the largest even T the shape rule accepts (None);
# N with N % 8 in {0, 1, 7} and 1, 2, 25 and 26 series blocks (the M pass starts on the ragged last block)
GEOM_EM = ((172, 8, 3), (174, 9, 3), (176, 15, 5), (344, 200, 8), (516, 207, 7), (344, 193, 4), (None, 201, 8),
           (None, 199, 2))
GEOM_ALS = ((172, 8, 3), (174, 9, 3), (176, 15, 5), (344, 200, 8), (516, 207, 7), (344, 193, 4), (None, 201, 8),
            (None, 15, 1))
ALS_KERNELS = {"estimate_factor": (("k_als_fused2<RT>",), ("k_als_masked<RT>", "k_als_factor"))}


def geom_T(T, N, r, ok):
    return t_max(ok, N, r) if T is None else T


def check_geom_em(lib, T, N, r):
    """k_em_fused2 vs the oracle on an ordinary strong-signal panel of this stage geometry (as P.check_em)."""
    T = geom_T(T, N, r, fused2_shape_ok)
    assert fused2_shape_ok(T, N, r) and not fused2_shape_ok(T + 2, N, r) or T < t_max(fused2_shape_ok, N, r)
    P.check_em(lib, N=N, r=r, T=T, p=1, iters=2, path=3, ll_cell_tol=1e-12)


def check_geom_als(lib, T, N, r, B=3):
    """k_als_fused2 vs the oracle, panel by panel (P.check_als_balanced), and each panel of a batched call against its
    one-panel call.  With many series every start converges in the same number of sweeps, so the different stopping
    sweeps P.check_als_balanced asks of per_panel only hold on the narrow panels."""
    T = geom_T(T, N, r, als_fused2_shape_ok)
    assert als_fused2_shape_ok(T, N, r)
    P.check_als_balanced(lib, N=N, r=r, T=T, B=B, per_panel=N < 100)
    from oracle.dgp import simulate_panel
    Xb = np.stack([simulate_panel(N, r, T, rep=70 + b, standardize=False)[0] for b in range(B)])
    got = lib.estimate_factor(Xb, r, nt_min=20, tol=1e-8)
    for b in range(B):
        one = lib.estimate_factor(Xb[b], r, nt_min=20, tol=1e-8)
        assert one["stats"]["iters"] == got["stats"][b]["iters"]
        np.testing.assert_allclose(got["F"][b], one["F"], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(got["Lam"][b], one["Lam"], rtol=1e-12, atol=1e-13)


def check_past_tmax(lib, N=201, r=8):
    """At T_max + 2 path 3 refuses the shape (DFMError 6) and path 0 runs (k_em_fused on the GPU) against the oracle."""
    import dynamic_factor_models_b200 as D
    T = t_max(fused2_shape_ok, N, r) + 2
    from oracle import dfm_ref as R
    from oracle.dgp import simulate_panel
    X, _ = simulate_panel(N, r, T, rep=9)
    Lam, Rv, A, Q = K.init_from_factors(X, R.pca_score(X, r), 1)
    try:
        lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=2, tol=0.0, path=3)
        raise AssertionError("path 3 accepted T = %d > T_max" % T)
    except D.DFMError as e:
        assert e.code == 6, e.code
    ref = K.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=2, tol=0.0)
    got = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=2, tol=0.0, path=0)
    assert got["status"] == 0
    P.compare_em(got, ref, P.ll_atol(X, 1e-12))


# ----------------------------------------------------------------------------------------------- the mixed batch
# one shape for the fast (nE ~ 6), slow (nE ~ 200) and never-frozen panels; T = 900 makes shared memory the binding limit
# of k_em_fused at exactly F1_MINB CTAs per SM, so the resident grid is known without the device's register count
MIX = dict(r=3, N=12, T=900, a=tuple(_slow(3, 0.995, 0.999)))
MIX_WANTS = ("fast", "slow", "never")
WANTS["slow"] = (lambda p: p.frozen and 150 <= p.nE <= 300, 200)


def mixed_models():
    # (the slow chain has no margin; its panels need only stay frozen with a long explicit range)
    return [chain_model(want=w, margin=0.0 if w == "slow" else MARGIN, **MIX) for w in MIX_WANTS]


def mixed_regimes(B, grid):
    """Regime of each panel: b % 3 for the first round, shifted by one for the panels a CTA runs after its first, so that
    every CTA with two panels changes regime on the same scratch and ring."""
    return [b % 3 if b < grid else (b - grid + 1) % 3 for b in range(B)]


def check_mixed_batch(lib, path, grid, iters=2):
    """grid + 5 panels: CTA j < 5 runs panel j and then panel grid + j of another regime.  Those ten panels and the last
    one against their one-panel calls (bit for bit: same kernel, same arithmetic) and against the oracle."""
    ms = mixed_models()
    for m, w in zip(ms, MIX_WANTS):
        assert WANTS[w][0](m.plan), (w, m.plan[:13])
    B = grid + 5
    reg = mixed_regimes(B, grid)
    pick = lambda n: np.stack([getattr(ms[g], n) for g in reg])
    got = lib.em_kalman(pick("X"), pick("Lam"), pick("R"), pick("A"), pick("Q"), p=1, P0=pick("P0"), max_iter=iters, tol=0.0,
                        path=path)
    assert (got["status"] == 0).all() and (got["iters"] == iters).all()
    refs = {}
    for b in sorted(set(range(5)) | set(range(grid, B)) | {grid - 1}):
        m = ms[reg[b]]
        one = lib.em_kalman(m.X, m.Lam, m.R, m.A, m.Q, p=1, P0=m.P0, max_iter=iters, tol=0.0, path=path)
        mine = {n: got[n][b] for n in ("F", "PF", "Lam", "R", "A", "Q", "P0", "loglik")}
        for n in mine:
            assert np.array_equal(mine[n], one[n]), "panel %d (%s): %s differs from the one-panel call" % (b, MIX_WANTS[reg[b]], n)
        if reg[b] not in refs:
            refs[reg[b]] = K.em_kalman(m.X, m.Lam, m.R, m.A, m.Q, p=1, P0=m.P0, max_iter=iters, tol=0.0)
        compare_tight(mine, refs[reg[b]], m.X)
