"""Oracle checks of the narrative sign restrictions (dfm_narrative_sign_restrictions: k_sr_prep -> k_irf -> k_sign_prep ->
k_narr_prep -> k_narr_cand / k_sign_pick per candidate batch -> k_narr_rot -> k_series_resp -> k_narr_omega -> k_narr_weight) and
of the weighted percentiles (dfm_percentiles_weighted: k_wpercentiles) at the sizes and edges their host code accepts.  CASES is
the table; test_gpu_narrative_dispatch.py runs it on the H100 with the kernel-set assertion of dispatch_checks.KernelLog,
test_emu_narrative_dispatch.py on the host-emulation build (no launch profiler there; the cases in GPU_ONLY are left out).
Each case runs as case.run(lib, nsm, alloc), as in history_sign_dispatch_checks.

The host's size rules, restated below:
  - the narrative rows sorted as the kernels read them: kinds 0 and 3 by shock, then kinds 1 and 2; nT = the last shock with
    sign rows or rows of kinds 0 / 3; ncol = r when rows of kinds 1 / 2 exist, else nT; nD = r per kind-0 row and r^2 per
    other row; nC = (h + 1) r per row of kinds 1-3; nP = the periods the rows touch (nP r <= 2^14);
  - k_narr_prep: NR_PT = 128 threads, u_t one thread per period, each G one thread per element (r^2 > 128 at r >= 12);
  - k_narr_cand: narr_cand_smem, k_narr_rot: narr_rot_smem, k_narr_omega: narr_omega_smem, each refused above 220 KiB;
    candidate batches, accept words and pick rounds as dfm_sign_restrictions (history_sign_dispatch_checks.sign_ntile);
  - k_narr_omega: ntl = ceil(n_sim / 128) CTAs per kept slot, simulation s on Philox elements (s nP + pos) r + k;
    k_narr_weight: ceil(S / 128) CTAs over the S = models x n_keep slots of a chunk;
  - model chunks of nb (narr_chunk), the outputs written at offset j0 of each chunk;
  - k_wpercentiles: npad = the power of two >= max(n, 2), NR_PT chunks of ceil(m / 128) counted records in the scan.

Decisions (status, n_accept, cand) and n_ok / weight are compared exactly, n_ok up to the simulations the spec reports within
1e-9 of a decision; rot, resp and fevd relative to each kept candidate's condition number (history_sign_dispatch_checks
.compare_sign), eps relative to |L^-1| (|f_t| + sum_l |A_l| |f_{t-l}|) times that condition number."""
import ctypes as C

import numpy as np

from dynamic_factor_models_b200 import DFMError, api
from dynamic_factor_models_b200._lib import MEM_DEVICE
from dispatch_checks import KernelLog, case  # noqa: F401  (KernelLog: used by the GPU file)
import history_sign_dispatch_checks as HS
import identified_oracle as IO
import narrative_checks as NC
import narrative_oracle as NO
import sign_checks as SC
import sign_oracle as SO

METHODS = ("narrative_sign_restrictions", "narrative_sign_restrictions_raw", "percentiles_weighted")
CASES = []
GPU_ONLY = set()

NR_PT, NR_SIMT, SG_NT = 128, 128, 64
MAX_SMEM = 220 * 1024
ROW_BYTES = 36                         # sizeof(nr_row): nine ints
ALL = ("rot", "resp", "fevd", "n_ok", "weight", "eps")


# ---------------------------------------------------------------------------------------- the host's size rules, restated
def sizes(r, rows, narr):
    """(nT, ncol, nD, nC, nP) of sign rows `rows` (series, h, shock, sign) and narrative rows `narr`."""
    nT = max([j for _, _, j, _ in rows] + [j for kd, j, *_ in narr if kd in (0, 3)] + [0])
    ncol = r if any(kd in (1, 2) for kd, *_ in narr) else nT
    nD = sum(r if kd == 0 else r * r for kd, *_ in narr)
    nC = sum((h + 1) * r for kd, j, i, t, h, s in narr if kd != 0)
    return nT, ncol, nD, nC, len(NO.periods(narr)[0])


def narr_cand_smem(r, rows, narr):
    nT, ncol, nD, _, _ = sizes(r, rows, narr)
    return ((ncol + 1) * r * SG_NT + len(rows) * r + nD) * 8 + ROW_BYTES * len(narr) + 8 * (nT + 1)


def narr_rot_smem(r, rows, narr):
    nT, _, nD, _, _ = sizes(r, rows, narr)
    return ((r + 1) * r + len(rows) * r + nD) * 8 + ROW_BYTES * len(narr) + (2 * (nT + 1) + r) * 4


def narr_omega_smem(r, rows, narr):
    return 8 * sizes(r, rows, narr)[3] + 8


def narr_prep_smem(r, p):
    return (r * r * p + r * r + 1) * 8


def sim_ctas(n_sim):
    return -(-n_sim // NR_SIMT)


def weight_ctas(S):
    return -(-S // NR_PT)


def narr_chunk(n_model, N, r, p, H, Tp, ns, nR, nD, n_keep, n_rot, host, outputs=ALL):
    """Models per chunk of dfm_narrative_sign_restrictions (nb)."""
    k = r * p; kk, rk, rr, Tr = k * k, r * k, r * r, Tp * r
    nout, nE = N * H * ns, Tp * ns
    ntile = HS.sign_ntile(n_rot)
    stage = (N * r + N + rk + rr + Tr + ("rot" in outputs) * n_keep * rr + ("resp" in outputs) * n_keep * nout +
             ("fevd" in outputs) * n_keep * nout + ("eps" in outputs) * n_keep * nE + ("n_ok" in outputs) * n_keep +
             ("weight" in outputs) * n_keep) if host else 0
    per = 8 * (kk + 2 * rk + rr * H + nR * r + 2 + n_keep + n_keep * rr * H + Tr + nD + 2 * n_keep + stage) + 4 * (ntile + 1 + n_keep)
    return min(n_model, max(1, HS.CHUNK_BYTES // per), 65535 // n_keep)


def wp_npad(n):
    npad = 2
    while npad < n:
        npad <<= 1
    return npad


def wp_smem(n):
    return (wp_npad(n) + 2 * (NR_PT + 1) + 1) * 8 + wp_npad(n) * 4


def wp_chunk(m):
    """Counted records per scan chunk of k_wpercentiles."""
    return -(-m // NR_PT)


# ---------------------------------------------------------------------------------------------------- kernel sets
BASE = ("k_sr_prep", "k_irf", "k_sign_prep", "k_narr_prep", "k_narr_cand", "k_sign_pick", "k_narr_rot")
OTHER = ("k_sign_cand", "k_sign_rot", "k_wpercentiles", "k_percentiles")
NR = {"narrative_sign_restrictions": (BASE + ("k_series_resp", "k_narr_omega", "k_narr_weight"), OTHER)}
NR_RAW = {"narrative_sign_restrictions_raw": (BASE + ("k_series_resp", "k_narr_omega", "k_narr_weight"), OTHER)}
NR_NO_RESP = {"narrative_sign_restrictions": (BASE + ("k_narr_omega", "k_narr_weight"), OTHER + ("k_series_resp",))}
NR_NO_OMEGA = {"narrative_sign_restrictions": (BASE + ("k_narr_weight",), OTHER + ("k_series_resp", "k_narr_omega"))}
NR_NO_WEIGHT = {"narrative_sign_restrictions": (BASE + ("k_series_resp",), OTHER + ("k_narr_omega", "k_narr_weight"))}
WP = {"percentiles_weighted": (("k_wpercentiles",), ("k_percentiles", "k_narr_cand"))}


def nd_case(id_, kernels, gpu_only=False):
    if gpu_only:
        GPU_ONLY.add(id_)
    return case(id_, kernels, table=CASES)


# ---------------------------------------------------------------------------------------------------- comparison with the spec
def compare(got, refs, Lam, A, Q, F, p, H, seed, ids, scale, nk=None):
    """Each model of a batched result against the spec's result refs[b], on its first nk slots (all: None)."""
    for b, ref in enumerate(refs):
        nk_ = len(ref["cand"]) if nk is None else nk
        g = {n: v[b][:nk_] if isinstance(v[b], np.ndarray) else v[b] for n, v in got.items()}
        mid = int(ids[b])
        HS.compare_sign(g, ref, Lam[b], A[b], Q[b], p, H, seed, mid, scale)
        kept = ref["cand"] >= 0
        if "eps" in g:
            v, e = g["eps"], ref["eps"]
            assert (np.isnan(v) == np.isnan(e)).all(), ("eps", b)
            if kept.any():
                kap = HS.zcond(seed, mid, ref["cand"][kept], Q.shape[-1])
                se = HS.eps_scale(A[b], Q[b], F[b], p)
                err = np.nanmax(np.abs(v[kept] - e[kept]).reshape(kept.sum(), -1), axis=1)
                assert (err <= HS.TOL * kap * max(se, 1e-300)).all(), ("eps", b, err.max(), se)
        if "n_ok" in g:
            assert (np.abs(g["n_ok"][kept] - ref["n_ok"][kept]) <= ref["n_close"][kept]).all(), (b, g["n_ok"], ref["n_ok"])
            assert (g["n_ok"][~kept] == 0).all()
        if "weight" in g:
            assert np.isnan(g["weight"][~kept]).all()
            exact = kept & (ref["n_close"] == 0)
            np.testing.assert_array_equal(g["weight"][exact], ref["weight"][exact])


def run(lib, Lam, R, A, Q, F, rows, narr, H, ns, n_rot, n_keep, n_sim, seed, ids, scale, outputs=ALL, nk=None, batch=4096):
    """One batched call against the spec, model by model (spec slots: the first nk, all when None); returns (result, the spec's
    results, the smallest decision margin)."""
    got = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), NC.narr_arrays(narr), H, n_rot, n_keep, n_shock=ns,
                                          n_sim=n_sim, seed=seed, ids=ids, scale=scale, outputs=outputs)
    p = A.shape[-1] // Lam.shape[-1]
    refs = [NO.identify(Lam[b], R[b], A[b], Q[b], F[b], p, rows, narr, H, ns, n_rot, n_keep if nk is None else nk, n_sim, seed=seed,
                        mid=int(ids[b]), scale=scale, batch=batch) for b in range(Lam.shape[0])]
    compare(got, refs, Lam, A, Q, F, p, H, seed, ids, scale, nk=nk)
    return got, refs, min(r_["margin"] for r_ in refs)


def code(lib, *a, **kw):
    """The library's error code of a narrative_sign_restrictions call (0: accepted)."""
    try:
        lib.narrative_sign_restrictions(*a, **kw)
        return 0
    except DFMError as e:
        return e.code


# ---------------------------------------------------------------------------------------------------- rows candidate 0 satisfies
def rows_for(Lam, A, Q, F, p, H, seed, mid, spec, sign_rows=()):
    """Narrative rows that candidate 0 of model `mid` satisfies at orientation +1: spec entries (kind, shock, series, t, h); the
    sign of kinds 0 / 3 is candidate 0's, the shock of kinds 1 / 2 (None) the one candidate 0 makes most important (a kind-2
    entry whose window candidate 0 does not make overwhelming becomes kind 1).  sign_rows (series, h, shock): their signs from
    candidate 0 as well.  Returns (sign rows, narrative rows)."""
    r = Lam.shape[1]
    om = SO.omegas(seed, mid, [0], r)[0]
    C = SO.row_vectors(Lam, A, Q, p, [(i, h, j, 1) for i, h, j in sign_rows], H)
    rows = [(i, h, j, int(np.sign(C[q] @ om[:, j - 1]))) for q, (i, h, j) in enumerate(sign_rows)]
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, H)
    narr = []
    for kd, j, i, t, h in spec:
        if kd == 0:
            narr.append((0, j, 0, t, 0, int(np.sign(U[t] @ om[:, j - 1]))))
            continue
        Hk = NO.contributions(np.einsum("a,hab->hb", Lam[i], P), om, U, t, h)
        if kd == 3:
            narr.append((3, j, i, t, h, int(np.sign(Hk[j - 1]))))
        else:
            jj = int(np.argmax(np.abs(Hk)))
            narr.append((kd if kd == 1 or NO._share(2, Hk, jj)[0] else 1, jj + 1, i, t, h, 1))
    return rows, narr


def every_kind(r, p, Tp, H, N):
    """Entries of every kind: kind 0 on shock 1 at rows p and Tp - 1 and on shock r at row p + 1, kind 3 on shocks 1 and r, kinds
    1 and 2 with windows h = 0 and h = H - 1."""
    e = [(0, 1, 0, p, 0), (0, 1, 0, Tp - 1, 0), (3, 1, 1, p, H - 1), (1, None, 2 % N, Tp - 1, 0), (2, None, (N - 1), Tp - H, H - 1)]
    if r >= 2:
        e += [(0, r, 0, p + 1, 0), (3, r, 3 % N, p + 2, 1)]
    return e


def shuffled(narr, seed):
    """The rows in another order: kinds interleaved, shocks descending, periods unsorted (the host sorts them)."""
    return [narr[q] for q in np.random.default_rng(seed).permutation(len(narr))][::-1]


def one_model(r, p, N, Tp, seed):
    Lam, R, A, Q, sc = SC.models(r, p, N, 1, seed=seed)
    F = NC.path(r, Tp, seed)[None]
    return Lam, R, A, Q, F, sc


# ---------------------------------------------------------------------------------------------------- 1. k_narr_prep strides
@nd_case("prep_Tp128_129_300_r12_r16", NR)
def _(lib, nsm, alloc):
    # Tp = 128, 129 and 300 against NR_PT = 128 threads: u_t for t >= 128 on a thread's second (and third) round; a kind-0 row at
    # Tp - 1 and a kind-3 window Tp - 4 .. Tp - 1 read u_t past row 127; r = 12 and 16: the G of a kind-3 row has r^2 = 144 / 256
    # > 128 elements; r = 16, p = 3 (r p = 48, the largest k_narr_prep plan, 8 200 B); eps compared over the whole path
    assert narr_prep_smem(16, 3) == 8200
    for r, p in ((12, 1), (16, 3)):
        for Tp in (128, 129, 300):
            Lam, R, A, Q, F, sc = one_model(r, p, 10, Tp, seed=Tp + r)
            ids = np.array([3], np.uint64)
            rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, 4, 17, 3, [(0, 1, 0, Tp - 1, 0), (3, 1, 2, Tp - 4, 3), (0, 2, 0, p, 0)])
            assert max(t + h for _, _, _, t, h, _ in narr) == Tp - 1 >= NR_PT - 1
            got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, 4, 2, 200, 12, 128, 17, ids, sc)
            assert margin > 1e-9 and got["cand"][0, 0] == 0 and np.isfinite(got["eps"][0, 0, NR_PT:]).all()


# ---------------------------------------------------------------------------------------------------- 2. every kind, r p = 48
@nd_case("every_kind_r16_and_rp48", NR)
def _(lib, nsm, alloc):
    # rows of every kind at r = 16 (p = 1 and p = 3) and at each (r, p) with r p = 48 and r <= 16; n_shock = r
    for r, p in ((16, 1), (1, 48), (2, 24), (3, 16), (4, 12), (6, 8), (8, 6), (12, 4), (16, 3)):
        H, N = 4, 6
        Tp = p + 10
        Lam, R, A, Q, F, sc = one_model(r, p, N, Tp, seed=480 + r)
        ids = np.array([r], np.uint64)
        rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 23, r, every_kind(r, p, Tp, H, N))
        assert {kd for kd, *_ in narr} >= {0, 1, 3}
        got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 150, 10, 200, 23, ids, sc)
        assert margin > 1e-9 and got["cand"][0, 0] == 0, (r, p)


# ---------------------------------------------------------------------------------------------------- 3. largest k_narr_cand plan
@nd_case("cand_smem_r16_256_sign_rows_shuffled", NR)
def _(lib, nsm, alloc):
    # r = 16, ncol = 16, 256 sign rows (shock j: series j + 1 at h = 0 .. 15), kind-0 and kind-3 rows on shocks 1 .. 4 (noff has four
    # non-empty segments, nT = 16) and as many kind-1 rows as fit: 21, narr_cand_smem = 224 924 B <= 220 KiB; a 22nd is refused
    # with code 6.  The same rows shuffled give the same bits.
    r, N, H, Tp, p = 16, 20, 16, 30, 1
    Lam, R, _, Q, sc = SC.models(r, p, N, 1, seed=161)
    A = (0.6 * np.eye(r) + 0.01 * np.random.default_rng(16).standard_normal((r, r)) / np.sqrt(r))[None]
    F = NC.path(r, Tp, 161)[None]
    ids = np.array([5], np.uint64)
    spec = [(0, j, 0, 2 + j, 0) for j in (1, 2, 3, 4)] + [(3, j, j, 4, 2) for j in (1, 2, 3, 4)]
    spec += [(1, None, q % N, 1 + q, q % 3) for q in range(22)]
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 9, 5, spec, [(j + 1, h, j + 1) for j in range(r) for h in range(H)])
    assert len(rows) == 256 and sizes(r, rows, narr[:-1])[:2] == (16, 16)
    assert narr_cand_smem(r, rows, narr[:-1]) == 224924 <= MAX_SMEM < narr_cand_smem(r, rows, narr)
    assert narr_rot_smem(r, rows, narr[:-1]) <= MAX_SMEM and narr_omega_smem(r, rows, narr) <= MAX_SMEM
    assert code(lib, Lam, R, A, Q, F, SC.as_arrays(rows), NC.narr_arrays(narr), H, 64, 2, n_shock=r, n_sim=16, outputs=()) == 6
    narr = narr[:-1]
    got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 300, 6, 64, 9, ids, sc)
    assert margin > 1e-9 and got["cand"][0, 0] == 0
    sh = shuffled(narr, 1)
    assert [kd for kd, *_ in sh] != sorted(kd for kd, *_ in sh)
    got2 = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), NC.narr_arrays(sh), H, 300, 6, n_shock=r, n_sim=64,
                                           seed=9, ids=ids, scale=sc)
    for n in got:
        np.testing.assert_array_equal(got2[n], got[n], err_msg=n)


# ---------------------------------------------------------------------------------------------------- 4. column counts
@nd_case("columns_ncol_nT_below_ns_and_nT0", NR)
def _(lib, nsm, alloc):
    # (a) rows of kinds 0 / 3 on shocks 1 and 2 only, n_shock = 4: ncol = nT = 2 < n_shock; (b) only kinds 1 / 2: nT = 0,
    # ncol = r (every column drawn for the share rows), rows given shuffled
    r, p, N, H, Tp = 4, 2, 7, 4, 16
    Lam, R, A, Q, F, sc = one_model(r, p, N, Tp, seed=44)
    ids = np.array([11], np.uint64)
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 4, 11, [(0, 1, 0, 3, 0), (3, 2, 1, 5, 2), (0, 2, 0, 9, 0)])
    assert sizes(r, rows, narr)[:2] == (2, 2)
    got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, 4, 300, 20, 256, 4, ids, sc)
    assert margin > 1e-9 and got["n_accept"][0] > 20
    _, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 4, 11, [(1, None, 1, 4, 1), (2, None, 5, 8, 3), (1, None, 6, 12, 0)])
    assert sizes(r, [], narr)[:2] == (0, r)
    got, refs, margin = run(lib, Lam, R, A, Q, F, [], shuffled(narr, 2), H, 4, 300, 20, 256, 4, ids, sc)
    assert margin > 1e-9 and got["cand"][0, 0] == 0


@nd_case("columns_no_rows_weight_one", NR_NO_OMEGA)
def _(lib, nsm, alloc):
    # nR = nN = 0: ncol = 0, every candidate kept, n_ok = n_sim and weight 1 without k_narr_omega; no resp / fevd: no k_series_resp
    r, p = 3, 1
    Lam, R, A, Q, F, sc = one_model(r, p, 5, 10, seed=3)
    assert sizes(r, [], [])[:2] == (0, 0) and narr_cand_smem(r, [], []) == r * SG_NT * 8 + 8
    got, refs, _ = run(lib, Lam, R, A, Q, F, [], [], 3, 2, 50, 60, 77, 8, np.array([0], np.uint64), sc,
                       outputs=("rot", "n_ok", "weight", "eps"))
    assert got["n_accept"][0] == 50 and (got["cand"][0, :50] == np.arange(50)).all() and (got["cand"][0, 50:] == -1).all()
    assert (got["weight"][0, :50] == 1.0).all() and (got["n_ok"][0, :50] == 77).all() and np.isnan(got["weight"][0, 50:]).all()


@nd_case("no_weight_requested", NR_NO_WEIGHT)
def _(lib, nsm, alloc):
    # narrative rows, but neither weight nor n_ok requested: no k_narr_omega, no k_narr_weight
    r, p, H, Tp = 3, 2, 4, 12
    Lam, R, A, Q, F, sc = one_model(r, p, 6, Tp, seed=8)
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 2, 0, every_kind(r, p, Tp, H, 6))
    got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 200, 10, 64, 2, np.array([0], np.uint64), sc,
                            outputs=("rot", "resp", "fevd", "eps"))
    assert margin > 1e-9 and got["cand"][0, 0] == 0


# ---------------------------------------------------------------------------------------------------- 5. largest k_narr_omega plan
@nd_case("omega_smem_27_rows_h64_r16", NR_NO_RESP)
def _(lib, nsm, alloc):
    # r = 16, 27 kind-3 rows over one shared window t .. t + 64 (h = 64) on 27 series: nC = 27 * 65 * 16 doubles,
    # narr_omega_smem = 224 648 B <= 220 KiB; a 28th row is refused with code 6; nP = 65
    r, p, N, H, Tp = 16, 1, 28, 65, 72
    Lam, R, A, Q, F, sc = one_model(r, p, N, Tp, seed=27)
    spec = [(3, 1, i, 2, 64) for i in range(28)]
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 6, 1, spec)
    assert narr_omega_smem(r, [], narr[:27]) == 224648 <= MAX_SMEM < narr_omega_smem(r, [], narr)
    assert narr_cand_smem(r, [], narr) <= MAX_SMEM and sizes(r, [], narr)[4] == 65
    assert code(lib, Lam, R, A, Q, F, SC.as_arrays([]), NC.narr_arrays(narr), H, 64, 2, n_shock=1, n_sim=16, outputs=()) == 6
    got, refs, margin = run(lib, Lam, R, A, Q, F, [], narr[:27], H, 1, 100, 4, 128, 6, np.array([1], np.uint64), sc,
                            outputs=("rot", "n_ok", "weight", "eps"))
    assert margin > 1e-9 and got["cand"][0, 0] == 0


# ---------------------------------------------------------------------------------------------------- 6. nP r = 2^14
@nd_case("nP_r_2_14_overlaps_duplicate_shared_positions", NR_NO_RESP)
def _(lib, nsm, alloc):
    # r = 16, Tp = 1 100: a kind-3 row with h = 1 023 (rows 10 .. 1 033: nP = 1 024, nP r = 2^14), a kind-3 window and a kind-1
    # window inside it (500 .. 600, 970 .. 1 030), the kind-1 row twice, and a kind-0 row inside the kind-1 window (two rows on
    # one position); nC = (1 024 + 101 + 2 * 61) 16 doubles
    r, p, N, H, Tp = 16, 1, 8, 1030, 1100
    Lam, R, A, Q, F, sc = one_model(r, p, N, Tp, seed=1100)
    spec = [(3, 1, 0, 10, 1023), (3, 1, 3, 500, 100), (1, None, 5, 970, 60), (0, 1, 0, 1000, 0)]
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 8, 2, spec)
    narr.append(narr[2])
    nT, ncol, nD, nC, nP = sizes(r, rows, narr)
    assert nP * r == 1 << 14 and narr_omega_smem(r, rows, narr) <= MAX_SMEM and (ncol, nT) == (16, 1)
    got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 200, 3, 24, 8, np.array([2], np.uint64), sc,
                            outputs=("rot", "n_ok", "weight", "eps"))
    assert margin > 1e-9 and got["cand"][0, 0] == 0


# ---------------------------------------------------------------------------------------------------- 7. simulation counts
@nd_case("n_sim_1_127_128_129_1000", NR)
def _(lib, nsm, alloc):
    # n_sim around one k_narr_omega CTA (128 simulations): 1, 127 and 128 in one CTA, 129 in two (the second one simulation),
    # 1 000 in eight (the last 104); rows of every kind
    assert [sim_ctas(n) for n in (1, 127, 128, 129, 1000)] == [1, 1, 1, 2, 8]
    r, p, H, Tp = 3, 2, 4, 14
    Lam, R, A, Q, F, sc = one_model(r, p, 6, Tp, seed=129)
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 12, 4, every_kind(r, p, Tp, H, 6))
    for n_sim in (1, 127, 128, 129, 1000):
        got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 200, 8, n_sim, 12, np.array([4], np.uint64), sc)
        assert margin > 1e-9 and got["cand"][0, 0] == 0


@nd_case("n_sim_2_20_element_index_2_34", {"narrative_sign_restrictions": (BASE + ("k_narr_omega", "k_narr_weight"), OTHER)},
         gpu_only=True)
def _(lib, nsm, alloc):
    # n_sim = 2^20 with nP = 8 192 at r = 2 (one kind-3 window of h = 8 191 behind three kind-0 rows): the simulation base index
    # s nP passes 2^32 from s = 2^19 and the element index (s nP + pos) r + k reaches 2^34.  Each simulation's outcome is a fixed
    # function of its index, so n_ok(2^20) - n_ok(2^20 - 128) is the spec on simulations 2^20 - 128 .. 2^20 - 1 alone
    r, p, h = 2, 1, 8191
    H, Tp = h + 1, h + 4
    Lam, R, A, Q, F, sc = one_model(r, p, 4, Tp, seed=34)
    A = A * 0.5
    spec = [(0, 1, 0, 2, 0), (0, 1, 0, 3, 0), (0, 1, 0, 4, 0), (3, 1, 1, 2, h)]
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 3, 1, spec)
    nP = sizes(r, rows, narr)[4]
    assert nP == 8192 and nP * r == 1 << 14 and (1 << 19) * nP == 1 << 32
    ids = np.array([1], np.uint64)
    n = 1 << 20
    out = {}
    for n_sim in (n - 128, n):
        out[n_sim] = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), NC.narr_arrays(narr), H, 40, 2, n_shock=1,
                                                     n_sim=n_sim, seed=3, ids=ids, scale=sc, outputs=("rot", "n_ok", "weight"))
    ref = NO.identify(Lam[0], R[0], A[0], Q[0], F[0], p, rows, narr, H, 1, 40, 2, 1, seed=3, mid=1, scale=sc, batch=64)
    got = out[n]
    assert got["cand"][0, 0] == 0 and ref["margin"] > 1e-9
    np.testing.assert_array_equal(got["cand"][0], ref["cand"])
    np.testing.assert_array_equal(out[n - 128]["cand"], got["cand"])
    P = IO.psi(A[0], Q[0], p, H)
    for q in range(2):
        if got["cand"][0, q] < 0:
            continue
        om = got["rot"][0, q]
        dn, close = NO.omega_sim(lambda i: np.einsum("a,hab->hb", Lam[0][i], P) @ om, narr, r, n, 3, 1, s0=n - 128, s1=n)
        d = int(got["n_ok"][0, q] - out[n - 128]["n_ok"][0, q])
        assert abs(d - dn) <= close and 0 < dn < 128, (q, d, dn, close)
        assert got["weight"][0, q] == n / got["n_ok"][0, q]


# ---------------------------------------------------------------------------------------------------- 8. model ids
@nd_case("ids_2_32_plus_5_and_2_40_minus_1", NR)
def _(lib, nsm, alloc):
    # model ids with a high word (Philox counter word c.w) in the candidate draws and the simulations; rows of every kind
    r, p, H, Tp, N = 4, 2, 4, 15, 6
    Lam, R, A, Q, sc = SC.models(r, p, N, 2, seed=40)
    F = np.stack([NC.path(r, Tp, 40 + b) for b in range(2)])
    ids = HS.IDS_BIG[::-1].copy()
    rows, narr = rows_for(Lam[0], A[0], Q[0], F[0], p, H, 21, int(ids[0]), every_kind(r, p, Tp, H, N))
    got, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, r, 200, 10, 300, 21, ids, sc)
    assert margin > 1e-9 and got["cand"][0, 0] == 0 and all(int(i) >> 32 for i in ids)


# ---------------------------------------------------------------------------------------------------- 9. weight +Inf
@nd_case("weight_inf_when_n_ok_0", NR_NO_RESP)
def _(lib, nsm, alloc):
    # n_sim = 1 and one kind-0 row: the spec picks an id whose one simulation fails the row (n_ok = 0, weight +Inf) and one whose
    # simulation passes it (n_ok = 1, weight 1); api._weighted_bands drops the +Inf draw
    r, p, H, Tp = 2, 1, 3, 8
    Lam, R, A, Q, sc = SC.models(r, p, 4, 2, seed=9)
    F = np.stack([NC.path(r, Tp, 9)] * 2)
    narr = [(0, 1, 0, 3, 0, 1)]
    n_ok = {}
    for mid in range(64):
        n_ok.setdefault(NO.omega_sim(lambda i: None, narr, r, 1, 6, mid)[0], mid)
    ids = np.array([n_ok[0], n_ok[1]], np.uint64)
    got, refs, _ = run(lib, Lam, R, A, Q, F, [], narr, H, 1, 30, 4, 1, 6, ids, sc, outputs=("rot", "n_ok", "weight"))
    assert (got["n_accept"] > 0).all()
    assert np.isposinf(got["weight"][0, 0]) and got["n_ok"][0, 0] == 0 and got["weight"][1, 0] == 1.0
    w = np.r_[got["weight"][0, :1], got["weight"][1, :1]]
    x = np.array([[5.0], [7.0]])
    bands = api._weighted_bands(lib, x, np.where(np.isfinite(w), w, 0.0), (0, 50, 100), (1,))
    assert (bands == 7.0).all()


# ---------------------------------------------------------------------------------------------------- 10. k_narr_weight CTAs
@nd_case("weight_ctas_S129_S300", NR_NO_RESP)
def _(lib, nsm, alloc):
    # S = 3 x 43 = 129 slots (two k_narr_weight CTAs, the second one slot) and 3 x 100 = 300 (three CTAs), weight requested
    assert weight_ctas(129) == 2 and weight_ctas(300) == 3
    r, p, H, Tp = 2, 1, 3, 10
    Lam, R, A, Q, sc = SC.models(r, p, 5, 3, seed=129)
    F = np.stack([NC.path(r, Tp, 60 + b) for b in range(3)])
    ids = np.array([0, 1, 2], np.uint64)
    narr = [(0, 1, 0, 2, 0, 1), (3, 2, 1, 4, 2, 1)]
    for n_keep in (43, 100):
        got, refs, _ = run(lib, Lam, R, A, Q, F, [], narr, H, 2, 400, n_keep, 50, 2, ids, sc, outputs=("rot", "n_ok", "weight"))
        assert (got["n_accept"] >= n_keep).all() and np.isfinite(got["weight"][:, -1]).all()


# ---------------------------------------------------------------------------------------------------- 11. model chunks
@nd_case("chunks_2_2_1_host_and_device", {**NR, **NR_RAW})
def _(lib, nsm, alloc):
    # n_keep = 30 000: nb = 65 535 // 30 000 = 2, so five models run in chunks of 2, 2 and 1; model 2 (a NaN path row) in the
    # middle chunk; every output.  Each model against the spec on its first 4 slots and against the bits of a one-model call; the
    # device-memory call (outputs in place at offset j0) gives the host call's bits
    r, p, N, H, Tp, B, n_keep, n_rot = 2, 1, 4, 3, 10, 5, 30000, 1 << 15
    assert [min(2, B - j) for j in range(0, B, 2)] == [2, 2, 1]
    Lam, R, A, Q, sc = SC.models(r, p, N, B, seed=225)
    F = np.stack([NC.path(r, Tp, 80 + b) for b in range(B)])
    F[2, 5, 1] = np.nan
    narr = [(0, 1, 0, 3, 0, 1), (1, 2, 1, 6, 1, 1), (3, 1, 2, 4, 2, 1)]
    rows = [(0, 0, 1, 1)]
    nD = sizes(r, rows, narr)[2]
    for host in (True, False):
        assert narr_chunk(B, N, r, p, H, Tp, 2, 1, nD, n_keep, n_rot, host) == 2
    ids = np.arange(B, dtype=np.uint64)
    big, refs, margin = run(lib, Lam, R, A, Q, F, rows, narr, H, 2, n_rot, n_keep, 16, 7, ids, sc, nk=4)
    assert list(big["status"]) == [0, 0, 3, 0, 0] and (big["n_accept"][[0, 1, 3, 4]] > 4).all()
    for b in range(B):
        one = lib.narrative_sign_restrictions(Lam[b], R[b], A[b], Q[b], F[b], SC.as_arrays(rows), NC.narr_arrays(narr), H, n_rot,
                                              n_keep, n_shock=2, n_sim=16, seed=7, ids=[b], scale=sc)
        for n in big:
            np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))
    dev = NC._raw_device(lib, alloc, Lam, R, A, Q, F, rows, narr, H, 2, n_rot, n_keep, 16, 7, scale=sc)
    for n in big:
        np.testing.assert_array_equal(dev[n], big[n], err_msg=n)


# ---------------------------------------------------------------------------------------------------- 12. second batch
@nd_case("second_batch_fill_kind1", NR_NO_RESP)
def _(lib, nsm, alloc):
    # n_rot = 2^20 + 1 000: two candidate batches (2^20, then 1 000 from c0 = 2^20); sign rows on shock 1 pi - 0.0143 apart
    # (0.46 % pass) and a kind-1 row on shock 2 (ncol = 2); n_keep between the accepted count of batch 1 and the total, so the last kept slots are
    # filled in batch 2; the spec decides all 1 049 576 candidates with decide_batch
    n_rot, H, seed = (1 << 20) + 1000, 2, 5
    assert HS.sign_batches(n_rot) == 2
    Lam, R, A, Q, sc, rows = HS._two_rows(2, 1, 3, 77, 0.0143, ns=1)
    F = NC.path(2, 8, 77)[None]
    narr = [(1, 2, 2, 3, 1, 1)]
    ids = np.array([3], np.uint64)
    ref = NO.identify(Lam[0], R[0], A[0], Q[0], F[0], 1, rows, narr, H, 2, n_rot, 1, 8, seed=seed, mid=3, scale=sc, batch=1 << 16)
    Om = SO.omegas(seed, 3, np.arange(1 << 20), 2)
    U = NO.shocks_u(A[0], Q[0], F[0], 1)
    P = IO.psi(A[0], Q[0], 1, H)
    ok1, _, _ = NO.decide_batch(Om, SO.row_vectors(Lam[0], A[0], Q[0], 1, rows, H), [j for _, _, j, _ in rows], narr,
                                lambda i: np.einsum("a,hab->hb", Lam[0][i], P), U, 2)
    n1 = int(ok1.sum())
    n_keep = (n1 + ref["n_accept"]) // 2
    assert 0 < n1 < n_keep < ref["n_accept"] and ref["margin"] > 1e-9, (n1, ref["n_accept"])
    got, refs, _ = run(lib, Lam, R, A, Q, F, rows, narr, H, 2, n_rot, n_keep, 8, seed, ids, sc, outputs=("rot", "n_ok", "weight"),
                       batch=1 << 16)
    assert got["cand"][0, -1] >= 1 << 20


# ---------------------------------------------------------------------------------------------------- 13. refusals
@nd_case("n_keep_65535_accepted_65536_refused", NR_NO_RESP)
def _(lib, nsm, alloc):
    r, p = 1, 1
    Lam, R, A, Q, F, sc = one_model(r, p, 3, 6, seed=1)
    a = (Lam, R, A, Q, F, SC.as_arrays([]), NC.narr_arrays([(0, 1, 0, 2, 0, 1)]), 1, 10)
    assert code(lib, *a, 65536, n_shock=1, n_sim=1, outputs=("n_ok",)) == 6
    got = lib.narrative_sign_restrictions(*a, 65535, n_shock=1, n_sim=1, outputs=("n_ok", "weight"))
    assert got["n_accept"] == 10 and (got["cand"][10:] == -1).all() and np.isnan(got["weight"][10:]).all()


# ---------------------------------------------------------------------------------------------------- weighted percentiles
Q11 = (0, 5, 10, 16, 25, 50, 75, 84, 90, 95, 100)
WP_N = (1, 2, 3, 127, 128, 129, 255, 256, 257, 4097, 16383, 16384)


def wp_check(lib, x, w, q, near=False):
    got = lib.percentiles_weighted(x, w, q)
    if near:
        lo, hi = NO.weighted_percentiles(x, w, q, near=True)
        assert ((lo <= got) & (got <= hi) | (np.isnan(lo) & np.isnan(got))).all()
    else:
        np.testing.assert_array_equal(got, NO.weighted_percentiles(x, w, q))
    return got


@nd_case("wp_equal_weights_are_unweighted_inverted_cdf", WP)
def _(lib, nsm, alloc):
    # equal weights n_sim / n_ok (the weights of kind-0-only narratives) at every size edge of the sort (npad) and of the scan
    # chunks (ceil(m / 128)): the record of numpy's unweighted inverted_cdf
    assert [wp_npad(n) for n in (1, 129, 16384)] == [2, 256, 16384] and wp_chunk(16384) == 128 and wp_chunk(129) == 2
    assert wp_smem(16384) <= MAX_SMEM < wp_smem(16385)
    rng = np.random.default_rng(5)
    for n in WP_N:
        x = rng.standard_normal((n, 2))
        for nok in (3, 7, 37, 100, 511, 1000, 12345):
            got = wp_check(lib, x, np.full(n, 2.0 ** 20 / nok), Q11)
            np.testing.assert_array_equal(got, np.percentile(x, Q11, axis=0, method="inverted_cdf"), err_msg=str((n, nok)))


@nd_case("wp_repeated_spanning_special_tied", WP)
def _(lib, nsm, alloc):
    # weights with repeated values (a few n_ok values), weights spanning 2^40 (outside the exact range: either neighbour within
    # 2^-100 of the total), zero / +Inf / NaN weights and NaN values, a column with no counted record, tied values
    rng = np.random.default_rng(6)
    for n in WP_N:
        x = rng.standard_normal((n, 4))
        x[:, 2] = np.round(x[:, 2] * 2)                    # ties
        x[:, 3] = np.nan                                   # (no counted record)
        wp_check(lib, x, 2.0 ** 20 / rng.choice([3, 5, 37, 1000], n), Q11)
        wp_check(lib, x, 2.0 ** rng.uniform(-20, 20, n), Q11, near=True)
        w = rng.random(n) + 0.5
        sp = rng.random(n)
        w[sp < 0.1] = 0.0; w[(sp >= 0.1) & (sp < 0.15)] = np.inf; w[(sp >= 0.15) & (sp < 0.2)] = np.nan
        xx = x.copy(); xx[rng.random(n) < 0.1, 0] = np.nan
        got = wp_check(lib, xx, w, Q11)
        assert np.isnan(got[:, 3]).all()


@nd_case("wp_nq64_d70000_device_memory", WP)
def _(lib, nsm, alloc):
    # 64 quantiles; d = 70 000 > 65 535 statistics (CTAs); the raw call on device memory
    rng = np.random.default_rng(7)
    q = np.linspace(0, 100, 64)
    x = rng.standard_normal((300, 3)); w = 2.0 ** 20 / rng.choice([7, 9, 11], 300)
    ref = wp_check(lib, x, w, q)
    xb = np.tile(rng.standard_normal((5, 7)), (1, 10000))
    got = wp_check(lib, xb, np.full(5, 3.0), (0, 50, 90))
    assert got.shape == (3, 70000)
    dx, dw, do = alloc(np.ascontiguousarray(x)), alloc(w), alloc(np.zeros(64 * 3))
    qq = np.ascontiguousarray(q)
    rc = lib.lib.dfm_percentiles_weighted(lib.h, C.c_void_p(dx[0]), C.c_void_p(dw[0]), 300, 3, qq.ctypes.data_as(C.c_void_p), 64,
                                          MEM_DEVICE, C.c_void_p(do[0]))
    assert rc == 0
    lib.sync()
    np.testing.assert_array_equal(do[1]().reshape(64, 3), ref)
