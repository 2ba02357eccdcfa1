"""Oracle checks of the historical decompositions (dfm_historical_decomposition: k_sr_prep -> k_hd_paths -> k_hd_series<RM>) and
the sign-restriction search (dfm_sign_restrictions: k_sr_prep -> k_irf -> k_sign_prep -> k_sign_cand / k_sign_pick per candidate
batch -> k_sign_rot -> k_series_resp) at the sizes and edges their host code accepts.  CASES is the table;
test_gpu_history_sign_dispatch.py runs it on the H100 with the kernel-set assertion of dispatch_checks.KernelLog,
test_emu_history_sign_dispatch.py on the host-emulation build (no launch profiler there).  Each case runs as
case.run(lib, nsm, alloc): nsm = the device's SM count, alloc(a) = (address, fetch) of a copy of the array a in device memory.

Branches inside a kernel or a host loop cannot be seen from the launch profiler (it records k_hd_series<RM>, not the width
chosen); each case's comment gives the predicate and the numbers that decide them, with the host's rules restated below:
  - k_hd_series: loadings in RM = 8 / 16 / 32 / 48 registers for r <= 8 / 16 / 32 / 48 (hd_rm); HD_NS = 64 series per CTA;
    the recursions staged in passes of tc rows (hd_tc);
  - k_hd_paths: HD_PT = 128 threads, eps one thread per period, the recursions over a ring of p + 1 rows in hd_paths_smem;
  - dfm_historical_decomposition: chunks of nb models (hd_chunk);
  - k_sign_cand: SG_NT = 64 candidates per CTA, a batch of ntile SG_TILE candidates (sign_ntile), at most 2^20; shared memory
    sign_cand_smem; k_sign_pick: SG_PT SG_PW = 1 024 accept words per round (sign_pick_rounds), the kept count carried from
    one batch to the next in nacc; k_sign_rot: sign_rot_smem; k_series_resp: SR_NS = 128 series per CTA.

The tolerances are relative to each output's cancellation scale, not only to its size: for the decompositions the largest
|scale_i| |lam_i|' |y_t| over the factor-level recursions y (and |L^-1| (|f_t| + sum_l |A_l| |f_{t-l}|) for eps); for the
sign search the largest |scale_i| |c_{i,h}| times the condition number of the candidate's Z (Omega is Z's orthogonal factor)."""
import numpy as np

from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
from dispatch_checks import KernelLog, case  # noqa: F401  (KernelLog: used by the GPU file)
from oracle.dgp import rng_normal
from sampling_dispatch_checks import CHUNK_BYTES
import history_checks as HC
import history_oracle as HO
import identified_oracle as IO
import sign_checks as SC
import sign_oracle as SO

METHODS = ("historical_decomposition", "historical_decomposition_raw", "sign_restrictions", "sign_restrictions_raw")
CASES = []

HD_NS, HD_PT = 64, 128
SG_NT, SG_TILE, SG_PT, SG_PW, SG_BATCH = 64, 32, 256, 4, 1 << 20
SR_NS = 128
DEFAULT_SMEM = 48 * 1024               # dynamic shared memory a launch may use before the kernel's attribute is raised
TOL = 1e-12


# ---------------------------------------------------------------------------------------- the host's size rules, restated
def hd_rm(r):
    """Register width of k_hd_series."""
    return 8 if r <= 8 else 16 if r <= 16 else 32 if r <= 32 else 48


def hd_tc(r, ns, Tp):
    """Rows of the recursions per pass of k_hd_series."""
    nc = ns + 2
    budget = max(2048, r * HD_NS + nc * r)
    return min(Tp, (budget - r * HD_NS) // (nc * r))


def hd_passes(r, ns, Tp):
    return -(-Tp // hd_tc(r, ns, Tp))


def hd_paths_smem(r, p, ns):
    """Shared memory of k_hd_paths (hd_paths_smem_doubles * 8)."""
    return (r * r * p + r * r + (ns + 2) * (p + 1) * r + 1) * 8


def hd_chunk(n_model, N, r, p, Tp, ns, host, outputs=("contrib", "rest", "base")):
    """Models per chunk of dfm_historical_decomposition (nb)."""
    k = r * p; kk, rk, rr, Tr = k * k, r * k, r * r, Tp * r
    nY, nC, nB = (ns + 2) * Tr, N * Tp * ns, N * Tp
    stage = (N * r + N + rk + rr + Tr + (nC if "contrib" in outputs else 0) + (nB if "rest" in outputs else 0) +
             (nB if "base" in outputs else 0)) if host else 0
    per = 8 * (kk + 2 * rk + nY + Tr + stage) + 8
    return min(n_model, max(1, CHUNK_BYTES // per), 65535)


def chunks(n, nb):
    return [min(nb, n - j0) for j0 in range(0, n, nb)]


def sign_ntile(n_rot):
    """Accept words per model and candidate batch."""
    return min(-(-n_rot // SG_NT), SG_BATCH // SG_NT) * (SG_NT // SG_TILE)


def sign_batches(n_rot):
    return -(-n_rot // (sign_ntile(n_rot) * SG_TILE))


def sign_pick_rounds(n_rot):
    """Rounds of k_sign_pick per batch."""
    return -(-sign_ntile(n_rot) // (SG_PT * SG_PW))


def sign_cand_smem(r, nj, nR):
    return ((nj + 1) * r * SG_NT + nR * r) * 8 + (nj + 1) * 4


def sign_rot_smem(r, nj, nR):
    return ((r + 1) * r + nR * r) * 8 + (nj + 1 + r) * 4


# ---------------------------------------------------------------------------------------------------- kernel sets
HD_K = ("k_sr_prep", "k_hd_paths", "k_hd_series<RM>")
SG_K = ("k_sr_prep", "k_irf", "k_sign_prep", "k_sign_cand", "k_sign_pick", "k_sign_rot")
HD = {"historical_decomposition": (HD_K, SG_K[2:] + ("k_irf", "k_series_resp"))}
HD_RAW = {"historical_decomposition_raw": (HD_K, SG_K[2:] + ("k_irf", "k_series_resp"))}
SG = {"sign_restrictions": (SG_K + ("k_series_resp",), ("k_hd_paths", "k_hd_series<RM>"))}
SG_NO_RESP = {"sign_restrictions": (SG_K, ("k_series_resp", "k_hd_paths", "k_hd_series<RM>"))}


def hs_case(id_, kernels):
    return case(id_, kernels, table=CASES)


# ---------------------------------------------------------------------------------------------------- decompositions vs spec
def _close(g, e, s, what):
    """NaN pattern equal, |g - e| <= TOL max(s, |e|) (s: the cancellation scale)."""
    assert g.shape == e.shape, (what, g.shape, e.shape)
    assert (np.isnan(g) == np.isnan(e)).all(), what
    if np.isfinite(e).any():
        err = np.nanmax(np.abs(g - e))
        assert err <= TOL * max(s, np.nanmax(np.abs(e)), 1e-300), (what, err, s)


def eps_scale(A, Q, F, p):
    """max_t |L^-1| (|f_t| + sum_l |A_l| |f_{t-l}|): the cancellation scale of u_t = L^-1 (f_t - sum_l A_l f_{t-l})."""
    r = Q.shape[0]; Tp = F.shape[0]
    aF = np.abs(F)
    u = aF[p:].copy()
    for l in range(1, p + 1):
        u += aF[p - l:Tp - l] @ np.abs(A[:, (l - 1) * r:l * r]).T
    return float((u @ np.abs(np.linalg.inv(np.linalg.cholesky(Q))).T).max()) if Tp > p else 0.0


def hd_scales(Lam, A, Q, F, p, t0, ns, scale):
    """(eps scale, series scale) of one model: max_t |L^-1| (|f_t| + sum_l |A_l| |f_{t-l}|), and max_{i,t} |scale_i| |lam_i|' y_t
    with y_t the largest |.| over the factor-level recursions (the spec with Lam = I)."""
    r = Q.shape[0]
    se = eps_scale(A, Q, F, p)
    _, yc, yr, yb, _ = HO.decompose(np.eye(r), np.ones(r), A, Q, F, p, t0, n_shock=ns)
    Y = np.maximum(np.maximum(np.abs(yc).max(-1), np.abs(yr)), np.abs(yb))            # (r, Tp)
    sc = np.ones(Lam.shape[0]) if scale is None else np.asarray(scale)
    ss = float(((np.abs(sc)[:, None] * np.abs(np.nan_to_num(Lam))) @ Y).max())
    return se, ss


def compare_hd(got, b, Lam, R, A, Q, F, p, t0, ns, scale, T=None):
    """Model b of a batched result against the spec on rows < T (all: None; the decomposition is causal, so rows < T of a
    call on F are the spec on F[:T] whenever t0 < T)."""
    T = F.shape[1] if T is None else T
    Fb = F[b, :T]
    ref = HO.decompose(Lam[b], R[b], A[b], Q[b], Fb, p, t0, n_shock=ns, scale=scale)
    assert got["status"][b] == ref[-1], (b, got["status"][b], ref[-1])
    se, ss = hd_scales(Lam[b], A[b], Q[b], Fb, p, t0, ns, scale) if ref[-1] == 0 else (0.0, 0.0)
    _close(got["shocks"][b][:T], ref[0], se, ("shocks", b))
    _close(got["contrib"][b][:, :T], ref[1], ss, ("contrib", b))
    _close(got["rest"][b][:, :T], ref[2], ss, ("rest", b))
    _close(got["base"][b][:, :T], ref[3], ss, ("base", b))


def run_hd(lib, Lam, R, A, Q, F, t0, ns, scale):
    """One batched call against the spec, model by model."""
    got = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=scale)
    p = A.shape[-1] // Lam.shape[-1]
    for b in range(Lam.shape[0]):
        compare_hd(got, b, Lam, R, A, Q, F, p, t0, ns, scale)
    return got


def hd_sweep(lib, r, p, N, Tp, t0s, nss, seed, out=True):
    """Two models (HC.models: companion radius <= 0.95, paths simulated from them) at every (n_shock, t0); with `out`, series 0 of
    model 0 has a NaN R and the last series of model 1 (in the last tile) a NaN loading."""
    Lam, R, A, Q, F, sc = HC.models(r, p, N, Tp, 2, seed=seed)
    if out:
        R[0, 0] = np.nan
        Lam[1, N - 1, r - 1] = np.nan
    for ns in nss:
        for t0 in t0s:
            run_hd(lib, Lam, R, A, Q, F, t0, ns, sc)


def _t0s(p, Tp):
    return sorted({p - 1, (p - 1 + Tp) // 2, Tp - 1})


# ---------------------------------------------------------------------------------------------------- 1. k_hd_series widths
@hs_case("hd_rm8_rm16_r8_r9_r16", HD)
def _(lib, nsm, alloc):
    # r = 8 (RM = 8, its largest r), r = 9 and 16 (RM = 16, its smallest and largest r); N = 65, 129 and 64: two series tiles, the
    # second with one series (threads 1 .. 63 idle), three tiles with a one-series last tile, and exactly one full tile;
    # n_shock in {1, r}, t0 in {p - 1, mid, Tp - 1}
    assert [hd_rm(r) for r in (8, 9, 16)] == [8, 16, 16]
    for r, p, N in ((8, 3, 65), (9, 2, 129), (16, 3, 64)):
        assert -(-N // HD_NS) == {64: 1, 65: 2, 129: 3}[N]
        hd_sweep(lib, r, p, N, 30, _t0s(p, 30), (1, r), seed=100 + r)


@hs_case("hd_rm32_r17_r32", HD)
def _(lib, nsm, alloc):
    # r = 17 and 32: RM = 32, its smallest and largest r (no test reached this width before); N = 65 and 129; tc = 1 at r = 32
    # (one row per pass), tc = (2 048 - 1 088) / (19 * 17) = 2 at r = 17 with n_shock = r
    assert hd_rm(17) == hd_rm(32) == 32 and hd_rm(33) == 48
    assert hd_tc(17, 17, 30) == 2 and hd_tc(32, 1, 30) == hd_tc(32, 32, 30) == 1
    for r, p, N in ((17, 2, 65), (32, 1, 129)):
        hd_sweep(lib, r, p, N, 30, _t0s(p, 30), (1, r), seed=100 + r)


@hs_case("hd_rm48_r33_r40_r48", HD)
def _(lib, nsm, alloc):
    # r = 33, 40 and 48: RM = 48, its smallest, a middle and its largest r; tc = 1; N = 65, 64 and 129
    assert all(hd_rm(r) == 48 and hd_tc(r, 1, 20) == 1 for r in (33, 40, 48))
    for r, N in ((33, 65), (40, 64), (48, 129)):
        hd_sweep(lib, r, 1, N, 20, _t0s(1, 20), (1, r), seed=100 + r)


# ---------------------------------------------------------------------------------------------------- 2. row passes
@hs_case("hd_passes_r1_tc661", HD)
def _(lib, nsm, alloc):
    # r = n_shock = 1: budget = 2 048, tc = (2 048 - 64) / 3 = 661: Tp = 661 takes one pass, Tp = 662 two (the second one row);
    # p = 3, so Tp > 128 also sends eps round k_hd_paths' 128 threads six times
    assert hd_tc(1, 1, 10 ** 6) == 661 and hd_passes(1, 1, 661) == 1 and hd_passes(1, 1, 662) == 2
    for Tp in (661, 662):
        hd_sweep(lib, 1, 3, 5, Tp, _t0s(3, Tp), (1,), seed=Tp)


@hs_case("hd_passes_r8_ns8_tc19", HD)
def _(lib, nsm, alloc):
    # r = n_shock = 8: tc = (2 048 - 512) / 80 = 19: Tp = 19 in one pass, Tp = 20 in two (the second one row); also n_shock = 1
    # (tc = (2 048 - 512) / 24 = 64 >= Tp: one pass)
    assert hd_tc(8, 8, 100) == 19 and hd_passes(8, 8, 19) == 1 and hd_passes(8, 8, 20) == 2 and hd_passes(8, 1, 20) == 1
    for Tp in (19, 20):
        hd_sweep(lib, 8, 2, 13, Tp, _t0s(2, Tp), (1, 8), seed=Tp)


@hs_case("hd_passes_r32_r48_tc1", HD)
def _(lib, nsm, alloc):
    # r >= 32: budget = 64 r + nc r, tc = 1: Tp = 1 (t0 = 0, one pass of one row: nothing after the base row) and Tp = 2 (two
    # passes), at r = 32 (RM = 32) and r = 48 (RM = 48)
    assert all(hd_tc(r, ns, 2) == 1 for r in (32, 48) for ns in (1, r))
    for r in (32, 48):
        for Tp in (1, 2):
            hd_sweep(lib, r, 1, 65, Tp, _t0s(1, Tp), (1, r), seed=r + Tp)


@hs_case("hd_paths_Tp300_t0_first", HD)
def _(lib, nsm, alloc):
    # Tp = 300 > 2 HD_PT: eps on three rounds of k_hd_paths' threads; t0 = p - 1 = 3, so 296 steps of the ring of p + 1 = 5 rows;
    # n_shock in {1, 2, 3}, the rest recursion nonzero for n_shock < r
    hd_sweep(lib, 3, 4, 70, 300, (3,), (1, 2, 3), seed=300)


# ---------------------------------------------------------------------------------------------------- 3. k = 48
K48 = ((1, 48), (2, 24), (3, 16), (4, 12), (6, 8), (8, 6), (12, 4), (16, 3), (24, 2), (48, 1))


@hs_case("hd_k48_every_r_p", HD)
def _(lib, nsm, alloc):
    # every (r, p) with r p = 48; the ring of p + 1 rows up to 49 rows (p = 48); Tp = 150 > HD_PT at p >= 24; n_shock in {1, r},
    # t0 in {p - 1, mid}; the largest k_hd_paths plan, r = 48, p = 1, n_shock = 48: 9 409 doubles = 75 272 B > 48 KiB
    assert hd_paths_smem(48, 1, 48) == 75272 > DEFAULT_SMEM
    assert max(hd_paths_smem(r, p, r) for r, p in K48) == 75272
    for r, p in K48:
        Tp = 150 if p >= 24 else 40
        hd_sweep(lib, r, p, 20, Tp, sorted({p - 1, (p - 1 + Tp) // 2}), sorted({1, r}), seed=1000 + r)


# ---------------------------------------------------------------------------------------------------- 4. model chunks
@hs_case("hd_chunks_2_2_1_host_and_device", {**HD, **HD_RAW})
def _(lib, nsm, alloc):
    # r = 8, p = 1, n_shock = 4, N = 3, Tp = 404 000, 5 models: about 181 MB of device records per model and 265 MB with the host
    # staging, so nb = 2 either way and the chunks hold 2, 2 and 1 models; model 2 (a NaN in its path) in the middle chunk,
    # series 1 out of model 0 (NaN loading), series 2 out of model 3 (NaN loading), series 0 out of model 4 (NaN R).  Each model
    # against the spec on the first 200 rows (t0 = 50), and against the bits of a one-model call; the device-memory call gives
    # the host call's bits
    r, p, ns, N, Tp, B, t0, T = 8, 1, 4, 3, 404000, 5, 50, 200
    assert chunks(B, hd_chunk(B, N, r, p, Tp, ns, host=True)) == [2, 2, 1]
    assert chunks(B, hd_chunk(B, N, r, p, Tp, ns, host=False)) == [2, 2, 1]
    rng = np.random.default_rng(404)
    Lam = rng.standard_normal((B, N, r)); R = 0.5 + rng.random((B, N))
    A = np.stack([HO.stable_lags(rng.standard_normal((r, r)) / np.sqrt(r), 1, 0.9) for _ in range(B)])
    Q = np.empty((B, r, r))
    for b in range(B):
        G = rng.standard_normal((r, r)); Q[b] = G @ G.T / r + 0.5 * np.eye(r)
    F = rng.standard_normal((B, Tp, r))
    sc = 0.5 + rng.random(N)
    F[2, 150, 3] = np.nan
    Lam[0, 1, 2] = np.nan; Lam[3, 2, 0] = np.nan; R[4, 0] = np.nan
    big = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=sc)
    assert list(big["status"]) == [0, 0, 3, 0, 0]
    for b in range(B):
        compare_hd(big, b, Lam, R, A, Q, F, p, t0, ns, sc, T=T)
        one = lib.historical_decomposition(Lam[b], R[b], A[b], Q[b], F[b], t0, n_shock=ns, scale=sc)
        assert one["status"] == big["status"][b]
        for n in HC.NAMES:
            np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))
    assert np.isnan(big["contrib"][0, 1]).all() and np.isnan(big["base"][3, 2]).all() and np.isnan(big["rest"][4, 0]).all()
    assert np.isfinite(big["base"][4, 1:]).all() and np.isfinite(big["contrib"][1]).all()
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dF, dsc = alloc(to_cm(F)), alloc(np.ascontiguousarray(sc))
    size = dict(shocks=Tp * r, contrib=N * Tp * ns, rest=N * Tp, base=N * Tp)
    shape = dict(shocks=(B, r, Tp), contrib=(B, ns, Tp, N), rest=(B, Tp, N), base=(B, Tp, N))
    o = {n: alloc(np.zeros(B * size[n])) for n in HC.NAMES}
    st = alloc(np.zeros(B, np.int32))
    lib.historical_decomposition_raw({n: ins[n][0] for n in ins}, dF[0], N, r, p, Tp, t0, ns, B, dsc[0], MEM_DEVICE,
                                     status=st[0], **{n: o[n][0] for n in HC.NAMES})
    lib.sync()
    np.testing.assert_array_equal(st[1](), big["status"])
    for n in HC.NAMES:
        v = o[n][1]().reshape(shape[n])
        v = v.transpose(0, 3, 2, 1) if v.ndim == 4 else v.transpose(0, 2, 1)
        np.testing.assert_array_equal(v, big[n], err_msg=n)


# ---------------------------------------------------------------------------------------------------- sign search vs spec
def zcond(seed, mid, cand, r):
    """Condition numbers of the Z of candidates `cand` of model id `mid` (sign_oracle.omegas' draws)."""
    c = np.asarray(cand, dtype=np.uint64).reshape(-1)
    e = c[:, None] * np.uint64(r * r) + np.arange(r * r, dtype=np.uint64)[None, :]
    return np.linalg.cond(rng_normal(seed, mid, SO.RNG_SIGN, e.ravel()).reshape(len(c), r, r))


def compare_sign(got, ref, Lam, A, Q, p, H, seed, mid, scale, b=None):
    """One model of a sign_restrictions result (index b of a batch, or a one-model result) against the spec's result `ref`:
    status, n_accept and every kept id exactly; rot, fevd to TOL kappa_s and resp to TOL kappa_s max_{i,h} |scale_i| |c_{i,h}|,
    kappa_s the condition number of slot s's Z."""
    g = (lambda n: got[n][b]) if b is not None else (lambda n: got[n])
    assert g("status") == ref["status"], (g("status"), ref["status"])
    assert g("n_accept") == ref["n_accept"], (g("n_accept"), ref["n_accept"])
    np.testing.assert_array_equal(g("cand"), ref["cand"])
    r = Q.shape[0]
    kept = ref["cand"] >= 0
    kap = np.ones(len(kept))
    if kept.any():
        kap[kept] = zcond(seed, mid, ref["cand"][kept], r)
    sc = np.ones(Lam.shape[0]) if scale is None else np.asarray(scale)
    if ref["status"] == 0:
        c = np.einsum("ia,hab->ihb", np.nan_to_num(Lam), IO.psi(A, Q, p, H))
        cs = float((np.abs(sc)[:, None] * np.linalg.norm(c, axis=2)).max())
    else:
        cs = 1.0
    for n, s in (("rot", 1.0), ("resp", cs), ("fevd", 1.0)):
        if n not in got:
            continue
        v, e = g(n), ref[n]
        assert v.shape == e.shape and (np.isnan(v) == np.isnan(e)).all(), n
        for q in np.flatnonzero(kept):
            err = np.abs(v[q] - e[q])
            assert np.nanmax(err) <= TOL * kap[q] * max(s, 1e-300), (n, q, np.nanmax(err), kap[q], s)


def run_sign(lib, Lam, R, A, Q, rows, H, ns, n_rot, n_keep, seed, ids, scale, outputs=SC.NAMES):
    """One batched call against the spec, model by model; returns (result, the spec's results, the smallest decision margin)."""
    got = lib.sign_restrictions(Lam, R, A, Q, SC.as_arrays(rows), H, n_rot, n_keep, n_shock=ns, seed=seed, ids=ids, scale=scale,
                                outputs=outputs)
    p = A.shape[-1] // Lam.shape[-1]
    refs, margin = [], np.inf
    for b in range(Lam.shape[0]):
        ref = SO.identify(Lam[b], R[b], A[b], Q[b], p, rows, H, ns, n_rot, n_keep, seed=seed, mid=int(ids[b]), scale=scale)
        compare_sign(got, ref, Lam[b], A[b], Q[b], p, H, seed, int(ids[b]), scale, b=b)
        refs.append(ref)
        margin = min(margin, ref["margin"])
    return got, refs, margin


def rows_at_angle(Lam, A, Q, i0, i1, gap, rel=1.3):
    """Loadings of series i0 set so that rows (i0, h = 0) and (i1, h = 0) (both sign +1) are pi - gap apart: gap / pi of the
    Haar candidates pass them.  Returns the angle the spec sees."""
    L = np.linalg.cholesky(Q)
    u1 = Lam[i1] @ L
    v = Lam[i0] @ L
    v = v - (v @ u1) / (u1 @ u1) * u1                      # (a direction orthogonal to u1)
    th = np.pi - gap
    u0 = rel * np.linalg.norm(u1) * (np.cos(th) * u1 / np.linalg.norm(u1) + np.sin(th) * v / np.linalg.norm(v))
    Lam[i0] = np.linalg.solve(L.T, u0)
    C = SO.row_vectors(Lam, A, Q, A.shape[1] // Q.shape[0], [(i0, 0, 1, 1), (i1, 0, 1, 1)], 1)
    return np.arccos(C[0] @ C[1] / np.linalg.norm(C[0]) / np.linalg.norm(C[1]))


SEED_BIG = (1 << 63) + 12345
IDS_BIG = np.array([(1 << 40) - 1, (1 << 32) + 5], np.uint64)


# ---------------------------------------------------------------------------------------------------- 5. sign: r 13 .. 16
@hs_case("sign_r13_r16_big_ids_N130", SG)
def _(lib, nsm, alloc):
    # r = 13 (p = 2, k = 26) and r = 16 = SG_RMAX (p = 3, k = 48), n_shock in {1, r}: candidate columns for every restricted shock
    # up to 16 in k_sign_cand; model ids 2^40 - 1 and 2^32 + 5 (the high word of the id in Philox word c.w) and seed
    # 2^63 + 12 345 (key word k1 = 2^31); N = 130 > SR_NS: k_series_resp's second tile holds series 128 (out of the model: NaN
    # loading) and 129 (restricted at h = H - 1 when n_shock >= 2)
    N, H, n_rot, n_keep = 130, 5, 400, 48
    assert -(-N // SR_NS) == 2 and SEED_BIG >> 32 >= 1 << 31 and all(int(i) >> 32 for i in IDS_BIG)
    for r, p in ((13, 2), (16, 3)):
        Lam, R, A, Q, sc = SC.models(r, p, N, 2, seed=1300 + r)
        Lam[:, 128, 1] = np.nan
        for ns in (1, r):
            rows = SC.case_rows(Lam[0], A[0], Q[0], p, ns, H, SEED_BIG, int(IDS_BIG[0]))
            assert max(j for _, _, j, _ in rows) == ns
            got, refs, margin = run_sign(lib, Lam, R, A, Q, rows, H, ns, n_rot, n_keep, SEED_BIG, IDS_BIG, sc)
            assert margin > 1e-9, margin
            assert got["cand"][0, 0] == 0
            assert np.isnan(got["resp"][:, :, 128]).all() and np.isfinite(got["resp"][0, 0, 129]).all()


# ---------------------------------------------------------------------------------------------------- 6. sign: largest smem
@hs_case("sign_smem_r16_16_shocks_256_rows", SG)
def _(lib, nsm, alloc):
    # r = 16, 16 restricted shocks, 256 rows: sign_cand_smem = (17 * 16 * 64 + 256 * 16) 8 + 17 * 4 = 172 100 B, the largest plan
    # k_sign_cand accepts (> 48 KiB, so its attribute is raised); k_sign_rot 35 076 B.  Shock j's 16 rows are series j + 1 at
    # horizons 0 .. 15, signs those of candidate 0; A = 0.6 I + 0.01 G / 4 keeps a series' rows near one direction, so 435 of the
    # 2 000 candidates pass all 16 shocks
    r, N, H, n_rot, n_keep = 16, 20, 16, 2000, 64
    assert sign_cand_smem(r, 16, 256) == 172100 and sign_rot_smem(r, 16, 256) == 35076
    Lam, R, _, Q, sc = SC.models(r, 1, N, 1, seed=161)
    A = (0.6 * np.eye(r) + 0.01 * np.random.default_rng(16).standard_normal((r, r)) / np.sqrt(r))[None]
    ids = IDS_BIG[:1]
    rows = [(j + 1, h, j + 1, 1) for j in range(r) for h in range(H)]
    om = SO.omegas(SEED_BIG, int(ids[0]), [0], r)[0]
    C = SO.row_vectors(Lam[0], A[0], Q[0], 1, rows, H)
    rows = [(i, h, j, int(np.sign(C[q] @ om[:, j - 1]))) for q, (i, h, j, s) in enumerate(rows)]
    assert len(rows) == 256
    got, refs, margin = run_sign(lib, Lam, R, A, Q, rows, H, r, n_rot, n_keep, SEED_BIG, ids, sc)
    assert margin > 1e-9, margin
    assert got["cand"][0, 0] == 0 and got["n_accept"][0] > n_keep, got["n_accept"]


# ---------------------------------------------------------------------------------------------------- 7. sign: pick rounds
def _two_rows(r, p, N, seed, gap, ns=2):
    """One model with rows (0, 0, 1, +1), (1, 0, 1, +1) pi - gap apart, and (2, 1, ns, +1) when ns >= 2 (one row: always passed,
    the column flipped for about half of the candidates)."""
    Lam, R, A, Q, sc = SC.models(r, p, N, 1, seed=seed)
    ang = rows_at_angle(Lam[0], A[0], Q[0], 0, 1, gap)
    assert abs(ang - (np.pi - gap)) < 1e-9, ang
    rows = [(0, 0, 1, 1), (1, 0, 1, 1)] + ([(2, 1, ns, 1)] if ns >= 2 else [])
    return Lam, R, A, Q, sc, rows


@hs_case("sign_pick_three_rounds_slots_past_word_1024", SG)
def _(lib, nsm, alloc):
    # n_rot = 70 000: ntile = 2 * 1 094 = 2 188 words, three rounds of k_sign_pick (1 024, 1 024, 140 words); two rows on shock 1
    # at right angles (half the candidates pass), so the 20 000 slots are not full after round 1 (32 768 candidates), fill
    # within round 2, and round 3 only counts; the full id list, rot, resp and fevd against the spec
    n_rot, n_keep, H = 70000, 20000, 3
    assert sign_ntile(n_rot) == 2188 and sign_pick_rounds(n_rot) == 3 and sign_batches(n_rot) == 1
    Lam, R, A, Q, sc, rows = _two_rows(3, 2, 5, 70, np.pi / 2)
    ids = np.array([7], np.uint64)
    got, refs, margin = run_sign(lib, Lam, R, A, Q, rows, H, 2, n_rot, n_keep, 11, ids, sc)
    assert margin > 1e-9, margin
    cand = refs[0]["cand"]
    w = SG_PT * SG_PW * SG_TILE                              # candidates per round
    assert 0 < (cand < w).sum() < n_keep and cand[-1] < 2 * w and refs[0]["n_accept"] > n_keep, (refs[0]["n_accept"], cand[-1])
    assert (refs[0]["rot"][:, :, 1] < 0).any()               # (some shock-2 columns flipped)


# ---------------------------------------------------------------------------------------------------- 8. sign: late fill
LATE = {}


def _late(lib, n_keep):
    # r = 2, rows on shock 1 pi - 0.0143 apart: 0.46 % of the candidates pass; n_rot = 2^20 + 2^17 runs two batches (2^20 and 2^17
    # candidates), with 4 806 accepted in the first and 5 427 in all, so n_keep = 5 000 enters batch 2 with 0 < nacc < n_keep
    # (the kept count carried in `run`, the ids offset by c0 = 2^20) and fills inside it, n_keep = 12 000 never fills
    n_rot, H, ns, seed = (1 << 20) + (1 << 17), 2, 2, 5
    assert sign_batches(n_rot) == 2 and sign_ntile(n_rot) * SG_TILE == SG_BATCH
    Lam, R, A, Q, sc, rows = _two_rows(2, 1, 3, 77, 0.0143, ns=1)
    ids = np.array([3], np.uint64)
    if "ref" not in LATE:                                   # (the spec of 1.2 M candidates takes seconds: shared by both cases)
        LATE["ref"] = SO.identify(Lam[0], R[0], A[0], Q[0], 1, rows, H, ns, n_rot, 12000, seed=seed, mid=3, scale=sc)
    full = LATE["ref"]
    acc = full["cand"][full["cand"] >= 0]
    assert full["n_accept"] == len(acc) == 5427 and (acc < SG_BATCH).sum() == 4806 and full["margin"] > 1e-9
    ref = {n: (v[:n_keep] if isinstance(v, np.ndarray) else v) for n, v in full.items()}
    got = lib.sign_restrictions(Lam, R, A, Q, SC.as_arrays(rows), H, n_rot, n_keep, n_shock=ns, seed=seed, ids=ids, scale=sc)
    compare_sign(got, ref, Lam[0], A[0], Q[0], 1, H, seed, 3, sc, b=0)


@hs_case("sign_late_fill_in_batch_2", SG)
def _(lib, nsm, alloc):
    _late(lib, 5000)


@hs_case("sign_late_never_full", SG)
def _(lib, nsm, alloc):
    _late(lib, 12000)


# ---------------------------------------------------------------------------------------------------- 9. sign: edges
@hs_case("sign_edges_no_rows_last_shock_only_empty_slots", SG)
def _(lib, nsm, alloc):
    # (a) no rows: nj = 0, k_sign_cand tests nothing, every candidate is accepted and Omega is never flipped (sign_cand_smem =
    # 3 * 64 * 8 + 4 B); (b) rows only on shock n_shock = 3 (shocks 1 and 2 have empty row ranges, nj = 3); (c) n_keep = 100 >
    # n_rot = 40 with one row: slots 40 .. 99 empty (cand -1, k_sign_rot's sst = 3, NaN resp and fevd from k_series_resp); N = 130
    # > SR_NS throughout
    r, p, N, H = 3, 2, 130, 4
    Lam, R, A, Q, sc = SC.models(r, p, N, 2, seed=33)
    ids = np.array([0, 9], np.uint64)
    assert sign_cand_smem(r, 0, 0) == 3 * 64 * 8 + 4
    got, refs, _ = run_sign(lib, Lam, R, A, Q, [], H, 2, 100, 60, 4, ids, sc)
    assert (got["n_accept"] == 100).all() and (got["cand"] == np.arange(60)).all()
    rows = SC.expand([(1, 3, 1, (0, 1)), (N - 1, 3, -1, 2)])
    got, refs, margin = run_sign(lib, Lam, R, A, Q, rows, H, 3, 300, 40, 4, ids, sc)
    assert margin > 1e-9 and (got["n_accept"] > 0).all()
    got, refs, _ = run_sign(lib, Lam, R, A, Q, [(5, 0, 1, 1)], H, 1, 40, 100, 4, ids, sc)
    assert (got["n_accept"] == 40).all() and (got["cand"][:, 40:] == -1).all()
    assert np.isnan(got["resp"][:, 40:]).all() and np.isnan(got["fevd"][:, 40:]).all() and np.isfinite(got["fevd"][:, :40, 0]).all()


@hs_case("sign_no_series_outputs", SG_NO_RESP)
def _(lib, nsm, alloc):
    # outputs () and ("rot",): k_sign_rot still runs (it writes the records), k_series_resp does not; cand and rot against the spec
    Lam, R, A, Q, sc = SC.models(4, 2, 6, 2, seed=44)
    ids = np.array([2, 1 << 33], np.uint64)
    rows = SC.expand([(0, 1, 1, (0, 2)), (2, 2, -1, 1)])
    for outputs in ((), ("rot",)):
        got, refs, margin = run_sign(lib, Lam, R, A, Q, rows, 3, 2, 500, 30, 6, ids, sc, outputs=outputs)
        assert margin > 1e-9 and (got["n_accept"] > 0).all() and "resp" not in got
