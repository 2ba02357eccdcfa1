"""Oracle checks of the identified-shock entry points at the sizes and edges they accept: dfm_gibbs_constrained
(k_gibbs_draw_constr) at k = r p up to 48 and r up to 36, with up to r rows on a series, restricted series past the thread
loop's first round and a sub-batch capped by memory; dfm_series_responses (k_sr_prep -> k_irf -> k_series_resp) at r up to 64,
k up to 128 and beyond, several passes over the horizons, several series tiles and several chunks of models; and dfm_irf's and
dfm_series_responses' shared memory for k_irf.  CASES is the table; test_gpu_identified_dispatch.py runs it on the H100 with
the kernel-set assertion of dispatch_checks.KernelLog, test_emu_identified_dispatch.py on the host-emulation build (no launch
profiler there).  Each case runs as case.run(lib, nsm, alloc): nsm = the device's SM count (132 on an H100 and in the
emulation build), alloc(a) = (address, fetch) of a copy of the array a in device memory.

Branches inside a kernel or a host loop cannot be seen from the launch profiler; each case's comment gives the predicate and
the numbers that decide them, with the host's rules restated below:
  - k_gibbs_draw_constr: one thread per series (GB_NT = 128 threads, series i on thread i % 128 in round i / 128) factors
    kap I + S_i and leaves the restricted series; thread 0 then draws them in series order with lam_constr_correct (m rows:
    an m x m packed G); shared memory gibbs_draw_smem + gibbs_constr_smem, 84 784 B at (r, p) = (12, 4), 162 640 B at (36, 1);
  - k_series_resp: Psi staged in passes of hc horizons, hc = min(H, (kMaxSmem / 8 - (r + ns + 1) SR_NS) / r^2) (sr_hc); series
    tiles of SR_NS = 128 threads;
  - k_irf: 64 threads, row i of the k-vector on thread i % 64; shared (2k + 8) 8 B, above the 48 KiB default from k = 3 069,
    refused (status 6) from k = 14 077;
  - dfm_series_responses: chunks of nb models (sr_chunk), at most 65 535 (grid.y).

dfm_gibbs_constrained's refusal `smDc > kMaxSmem` and dfm_series_responses' "r too large" cannot fire (the enumerations of
test_emu_identified_dispatch.py check this)."""
import numpy as np

from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, to_cm
from dispatch_checks import KernelLog, case  # noqa: F401  (KernelLog: used by the GPU file)
from sampling_dispatch_checks import CHUNK_BYTES, GB_NT, KMAX_SMEM, _code, _same_as_fresh_handle, gibbs_draw_smem, ss_accepts, ssb_batch
import gibbs_checks as GC
import identified_checks as IC
import identified_oracle as IO

METHODS = ("gibbs", "series_responses", "irf")
CASES = []

SR_NS = 128
DEFAULT_SMEM = 48 * 1024               # dynamic shared memory a launch may use before the kernel's attribute is raised


# ---------------------------------------------------------------------------------------- the host's size rules, restated
def gibbs_constr_smem(r):
    """gibbs_constr_smem_doubles * 8: lam_constr_correct's scratch (r r + r (r + 1) / 2 + r) and three r-vectors."""
    return (r * r + r * (r + 1) // 2 + r + 3 * r) * 8


def gibbs_draw_constr_smem(r, p):
    """Shared memory of k_gibbs_draw_constr (smDc of gibbs_impl)."""
    return gibbs_draw_smem(r, p) + gibbs_constr_smem(r)


def gibbs_accepts(nsm, T, N, r, p):
    """dfm_gibbs' size rules before its own smem guards: k <= 48 and ss_check at the sub-batch size."""
    return r * p <= 48 and ss_accepts(nsm, ssb_batch(nsm, T, N, r, p), r, p)


def sr_smem0(r, ns):
    """series_resp_smem_doubles(r, ns, 0) * 8."""
    return (r + ns + 1) * SR_NS * 8


def sr_hc(r, ns, H):
    """Horizons per pass of k_series_resp."""
    return min(H, (KMAX_SMEM // 8 - (r + ns + 1) * SR_NS) // (r * r))


def sr_accepts(r, ns):
    """dfm_series_responses' `(sm0 + r r) 8 <= kMaxSmem`."""
    return sr_smem0(r, ns) + r * r * 8 <= KMAX_SMEM


def sr_chunk(n_model, N, r, p, H, ns, host, resp=True, fevd=True):
    """Models per chunk of dfm_series_responses (nb)."""
    k = r * p; kk = k * k; rk = r * k; rr = r * r; nout = N * H * ns
    per = 8 * (kk + 2 * rk + rr * H + ((N * r + N + rk + rr + (nout if resp else 0) + (nout if fevd else 0)) if host else 0)) + 8
    return min(n_model, max(1, CHUNK_BYTES // per), 65535)


def irf_smem(k):
    """Shared memory of k_irf (irf_smem_doubles * 8)."""
    return (2 * k + 8) * 8


def chunks(n, nb):
    return [min(nb, n - j0) for j0 in range(0, n, nb)]


# ---------------------------------------------------------------------------------------------------- kernel sets
FS = "k_em_filter_smooth"
FUSED = ("k_em_fused<RT>", "k_em_fused2<RT>")
GIBBS_C = {"gibbs": ((FS, "k_sim_gains", "k_gibbs_paths", "k_gibbs_stats", "k_gibbs_draw_constr", "k_sim_project", "k_ss_fc_rows"),
                     FUSED + ("k_gibbs_draw", "k_sim_paths", "k_ss_align", "k_irf"))}
GIBBS_IRF = {"gibbs": ((FS, "k_gibbs_draw", "k_ss_align", "k_irf"), FUSED + ("k_gibbs_draw_constr",))}
SR = {"series_responses": (("k_sr_prep", "k_irf", "k_series_resp"), ())}
IRF = {"irf": (("k_irf",), ())}


def identified_case(id_, kernels):
    return case(id_, kernels, table=CASES)


# ---------------------------------------------------------------------------------------------------- restrictions
def _rows(r, m, rng, orth=True):
    """m rows on one series: rows of a random orthogonal r x r matrix scaled by 1 .. 1.5 (well conditioned, not e_j), or
    Gaussian rows."""
    if orth:
        U, _ = np.linalg.qr(rng.standard_normal((r, r)))
        return U[:m] * (1.0 + 0.5 * rng.random(m))[:, None]
    return rng.standard_normal((m, r))


def constr(r, spec, seed=11):
    """constr = (index, H, h) from spec = ((series, m, orth), ...): m rows on each named series."""
    rng = np.random.default_rng(seed)
    idx, H, h = [], [], []
    for i, m, orth in spec:
        idx += [i] * m
        H.append(_rows(r, m, rng, orth))
        h.append(0.3 * rng.standard_normal(m))
    return np.array(idx, np.int32), np.vstack(H), np.concatenate(h)


def _restricted_chains(lib, N, r, p, T, spec, miss=0.05):
    X, th = GC.model(N=N, r=r, T=T, p=p, miss=miss, exclude=(4,), ragged=3)
    c = constr(r, spec)
    IC.check_chains(lib, X, th, p, c, n_chain=2, n_burn=1, n_keep=2, H_fc=2, fc_rows=3, chain0=1, sweep0=2)
    return X, th, c


# ---------------------------------------------------------------------------------------------------- 1. restricted Gibbs
@identified_case("gibbs_constr_k48_r12_p4", GIBBS_C)
def _(lib, nsm, alloc):
    # k = 48, r = 12 > 8: k_gibbs_draw_constr with gibbs_draw_smem + gibbs_constr_smem = 82 624 + 2 160 = 84 784 B > 48 KiB (the
    # attribute set per call); series 0 pinned (m = r = 12: a 12 x 12 G, lam = H^-1 h), series 2 with m = r - 1 = 11, three
    # Gaussian rows on series 7, one row on the last series (39) and one on the excluded series 4 (ignored); missing cells and a
    # ragged edge of 3 rows on series 0 .. 19
    assert gibbs_accepts(nsm, 200, 40, 12, 4) and gibbs_draw_constr_smem(12, 4) == 84784 > DEFAULT_SMEM
    _restricted_chains(lib, 40, 12, 4, 200, ((0, 12, True), (2, 11, True), (7, 3, False), (39, 1, True), (4, 1, True)))


@identified_case("gibbs_constr_k36_r12_p3", GIBBS_C)
def _(lib, nsm, alloc):
    # k = 36 (rows 32 .. 35 of k_gibbs_paths on lanes 0 .. 3), r = 12: 62 144 + 2 160 B of shared memory (> 48 KiB); the same
    # rows as the k = 48 case
    assert gibbs_accepts(nsm, 200, 40, 12, 3) and gibbs_draw_constr_smem(12, 3) > DEFAULT_SMEM
    _restricted_chains(lib, 40, 12, 3, 200, ((0, 12, True), (2, 11, True), (7, 3, False), (39, 1, True), (4, 1, True)))


@identified_case("gibbs_constr_r36_p1", GIBBS_C)
def _(lib, nsm, alloc):
    # r = 36, p = 1, the largest r ss_check takes: 162 640 B of shared memory, the most any accepted shape asks for; series 0
    # pinned by a random invertible 36 x 36 H (lam_constr_correct's packed G is 36 x 36, 666 doubles), series 3 with m = 35, one
    # row on the excluded series 4 and on the last series (119)
    assert gibbs_accepts(nsm, 150, 120, 36, 1) and gibbs_draw_constr_smem(36, 1) == 162640
    _restricted_chains(lib, 120, 36, 1, 150, ((0, 36, True), (3, 35, True), (4, 1, True), (119, 1, False)))


@identified_case("gibbs_constr_N200_past_GB_NT", GIBBS_C)
def _(lib, nsm, alloc):
    # N = 200 > GB_NT = 128: the restricted series 130 and 199 are factored on the thread loop's second round (threads 2 and 71)
    # with their missing-cell downdates of kap I + S_i, leave it, and are drawn by thread 0's serial pass after series 0 (m = r)
    T, N, r, p = 60, 200, 5, 1
    X, th, c = _restricted_chains(lib, N, r, p, T, ((0, 5, True), (130, 2, False), (199, 1, True), (4, 1, True)), miss=0.1)
    for i in (130, 199):
        assert i >= GB_NT and np.isnan(X[:, i]).any() and not np.isnan(th["Lam"][i]).any(), i


@identified_case("gibbs_constr_every_series", GIBBS_C)
def _(lib, nsm, alloc):
    # every series restricted, one row each, N = 140 > GB_NT (series 128 .. 139 on the second round): the thread loop draws no
    # series, thread 0 draws all 139 in the model (series 4 is out of it)
    N, r = 140, 3
    assert N > GB_NT
    _restricted_chains(lib, N, r, 2, 40, tuple((i, 1, i % 2 == 0) for i in range(N)), miss=0.1)


@identified_case("gibbs_constr_chain_split_capped_batch", GIBBS_C)
def _(lib, nsm, alloc):
    # N = 1 300, T = 200, r = 2 (gibbs_chain_split_capped_batch's shape): ssb_batch = 225 < 2 nsm = 264, a sub-batch capped by
    # memory; restrictions on series 0 (m = r), 700, 1 299 and the excluded series 4; a call on chains [0, C + 10) runs two
    # sub-batches, and calls on [0, 20) and on [C - 8, C + 8), which straddles its boundary, give the same bits
    T, N, r, p = 200, 1300, 2, 1
    C = ssb_batch(nsm, T, N, r, p)
    assert C < 2 * nsm and gibbs_accepts(nsm, T, N, r, p), C
    X, th = GC.model(N=N, r=r, T=T, p=p, miss=0.05, exclude=(4,), ragged=2)
    cs = constr(r, ((0, 2, True), (700, 1, False), (1299, 1, True), (4, 1, True)))
    base = GC._inits(th, C + 10)
    kw = dict(p=p, sweep0=2, n_burn=1, n_keep=1, seed=GC.SEED, H_fc=1, fc_rows=2, prior=GC.PRIOR, constr=cs,
              outputs=("Lam", "R", "F", "X"))
    sub = lambda c0, n: {m: base[m][c0:c0 + n] for m in base}
    big = lib.gibbs(X, sub(0, C + 10), n_chain=C + 10, chain0=0, **kw)
    assert (big["status"] == 0).all()
    for i in (0, 700, 1299):
        Hi, hi = IO.rows_of(cs, i)
        assert np.abs(np.einsum("qa,cja->cjq", Hi, big["Lam"][:, :, i]) - hi).max() <= 1e-12
    for c0, n in ((0, 20), (C - 8, 16)):
        got = lib.gibbs(X, sub(c0, n), n_chain=n, chain0=c0, **kw)
        for m in got:
            np.testing.assert_array_equal(got[m], big[m][c0:c0 + n], err_msg="%s [%d, %d)" % (m, c0, c0 + n))


# ---------------------------------------------------------------------------------------------------- 2. series responses
def sr_models(B, N, r, p, seed=1, rho=0.9, out=(3,), out_R=()):
    """B models (Lam (B, N, r), R (B, N), A (B, r, k), Q (B, r, r)) with sum_l |A_l|_2 = rho < 1 (stable, so long horizons stay
    bounded); series `out` have a NaN loading row, series `out_R` a NaN R (both out of the model)."""
    rng = np.random.default_rng(seed)
    Lam = 0.5 * rng.standard_normal((B, N, r))
    R = 0.2 + rng.random((B, N))
    A = np.empty((B, r, r * p))
    Q = np.empty((B, r, r))
    for b in range(B):
        for l in range(p):
            A[b, :, l * r:(l + 1) * r] = rho / p * np.linalg.qr(rng.standard_normal((r, r)))[0]
        W = rng.standard_normal((r, r))
        Q[b] = W @ W.T / r + 0.5 * np.eye(r)
    for i in out:
        Lam[:, i] = np.nan
    for i in out_R:
        R[:, i] = np.nan
    return Lam, R, A, Q


def _spec_close(g, e, what):
    assert (np.isnan(g) == np.isnan(e)).all(), what
    if not np.isnan(e).all():
        err = np.nanmax(np.abs(g - e))
        assert err <= 1e-12 * max(1.0, np.nanmax(np.abs(e))), (what, err)


def check_sr(got, Lam, R, A, Q, H, ns, scale=None, models=None, bad=()):
    """got (a series_responses result of the batch) against IO.responses for the models in `models` (all: None); the models in
    `bad` have status 3, the others 0."""
    B, N, r = Lam.shape
    p = A.shape[-1] // r
    st = np.asarray(got["status"])
    assert list(np.flatnonzero(st)) == sorted(bad) and (st[list(bad)] == 3).all(), np.flatnonzero(st)
    for b in (range(B) if models is None else models):
        rr, rf, s = IO.responses(Lam[b], R[b], A[b], Q[b], p, H, ns, scale)
        assert s == st[b], b
        _spec_close(got["resp"][b], rr, ("resp", b))
        _spec_close(got["fevd"][b], rf, ("fevd", b))


def sr_device(lib, alloc, Lam, R, A, Q, H, ns, scale=None):
    """dfm_series_responses with every input and output in device memory; the result shaped as series_responses'."""
    B, N, r = Lam.shape
    p = A.shape[-1] // r
    ins = {n: alloc(a_)[0] for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    sc = alloc(np.ascontiguousarray(scale, dtype=float))[0] if scale is not None else 0
    o = {n: alloc(np.zeros(B * N * H * ns)) for n in ("resp", "fevd")}
    st = alloc(np.zeros(B, np.int32))
    lib.series_responses_raw(ins, N, r, p, B, H, ns, sc, MEM_DEVICE, resp=o["resp"][0], fevd=o["fevd"][0], status=st[0])
    lib.sync()
    res = {n: o[n][1]().reshape(B, ns, H, N).transpose(0, 3, 2, 1) for n in o}
    res["status"] = st[1]()
    return res


def _sr(lib, B, N, r, p, H, ns, scale=True, **kw):
    Lam, R, A, Q = sr_models(B, N, r, p, **kw)
    sc = 0.5 + np.random.default_rng(2).random(N) if scale else None
    got = lib.series_responses(Lam, R, A, Q, H, n_shock=ns, scale=sc)
    check_sr(got, Lam, R, A, Q, H, ns, sc)


@identified_case("sr_r36_ns36_three_passes", SR)
def _(lib, nsm, alloc):
    # r = n_shock = 36: sm0 = 73 * 128 doubles, hc = (28 160 - 9 344) / 1 296 = 14, so H = 40 runs passes of 14, 14 and 12
    # horizons, the running FEV sums carried across them; k_sr_prep's chol at r = 36
    assert sr_hc(36, 36, 40) == 14
    _sr(lib, 2, 30, 36, 1, 40, 36)


@identified_case("sr_r64_ns64_last_pass_one", SR)
def _(lib, nsm, alloc):
    # r = n_shock = 64, the largest r: hc = (28 160 - 16 512) / 4 096 = 2, so H = 7 runs passes of 2, 2, 2 and 1; k_sr_prep's
    # chol at r = 64 (64 threads, (64^2 + 8) 8 = 32 832 B of shared memory); k_series_resp at (16 512 + 2 * 4 096) 8 = 197 632 B
    assert sr_hc(64, 64, 7) == 2 and sr_smem0(64, 64) + 2 * 64 * 64 * 8 == 197632 <= KMAX_SMEM
    _sr(lib, 2, 20, 64, 1, 7, 64)


@identified_case("sr_r20_ns1_last_pass_one", SR)
def _(lib, nsm, alloc):
    # r = 20, n_shock = 1: hc = (28 160 - 2 816) / 400 = 63, so H = 64 runs a pass of 63 and one of 1
    assert sr_hc(20, 1, 64) == 63
    _sr(lib, 2, 25, 20, 1, 64, 1)


@identified_case("sr_N300_three_series_tiles", SR)
def _(lib, nsm, alloc):
    # N = 300: three SR_NS = 128 series tiles of k_series_resp, the last with 44 series (threads 44 .. 127 idle); series 5 (NaN
    # loadings) in the first tile and 270 (NaN R) in the last are NaN columns
    N = 300
    assert -(-N // SR_NS) == 3 and N % SR_NS == 44
    _sr(lib, 3, N, 4, 2, 9, 2, out=(5,), out_R=(270,))


@identified_case("sr_k128_r64_p2", SR)
def _(lib, nsm, alloc):
    # k = 128 > 64: k_irf's rows go around its 64 threads twice; (2 * 128 + 8) 8 = 2 112 B
    _sr(lib, 2, 20, 64, 2, 5, 3)


@identified_case("sr_k48_r12_p4", SR)
def _(lib, nsm, alloc):
    # k = 48, r = 12 > 8: k_sr_prep's companion at k = 48, k_series_resp with all r shocks
    _sr(lib, 2, 30, 12, 4, 10, 12)


@identified_case("sr_chunks_host_and_device", SR)
def _(lib, nsm, alloc):
    # r = 64, p = 1, H = 1 000, N = 20, n_shock = 2, 40 models: in device memory nb = 2^29 / 32 866 312 B = 16 (chunks of 16, 16
    # and 8), in host memory the staging buffers add to a model's bytes and nb = 2^29 / 33 582 248 B = 15 (chunks of 15, 15
    # and 10); model 17 (NaN A and Q) and model 22 (Q not positive definite) sit in the second chunk either way; every model
    # against the spec, the device call's bits equal the host call's; hc = 4 (250 passes)
    B, N, r, p, H, ns = 40, 20, 64, 1, 1000, 2
    assert chunks(B, sr_chunk(B, N, r, p, H, ns, host=False)) == [16, 16, 8]
    assert chunks(B, sr_chunk(B, N, r, p, H, ns, host=True)) == [15, 15, 10]
    Lam, R, A, Q = sr_models(B, N, r, p, out=(3,), out_R=(11,))
    A[17] = np.nan; Q[17] = np.nan
    Q[22] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    sc = 0.5 + np.random.default_rng(2).random(N)
    got = lib.series_responses(Lam, R, A, Q, H, n_shock=ns, scale=sc)
    check_sr(got, Lam, R, A, Q, H, ns, sc, bad=(17, 22))
    dev = sr_device(lib, alloc, Lam, R, A, Q, H, ns, sc)
    for n in ("resp", "fevd", "status"):
        np.testing.assert_array_equal(dev[n], got[n], err_msg=n)


@identified_case("sr_grid_y_cap_70000_models", SR)
def _(lib, nsm, alloc):
    # 70 000 one-series models (r = p = 1, H = 3): nb = 65 535 (the grid.y cap; memory allows far more), chunks of 65 535 and
    # 4 465; models 65 534, 65 535 (the first of the second chunk) and 69 999 against the spec, and models 65 540 (NaN Q) and
    # 68 000 (Q < 0) of the second chunk have status 3
    B, N, r, p, H = 70000, 1, 1, 1, 3
    assert chunks(B, sr_chunk(B, N, r, p, H, 1, host=True)) == [65535, 4465]
    rng = np.random.default_rng(4)
    Lam = rng.standard_normal((B, N, r))
    R = 0.1 + rng.random((B, N))
    A = rng.uniform(-0.9, 0.9, (B, r, r))
    Q = 0.5 + rng.random((B, r, r))
    Q[65540] = np.nan
    Q[68000] = -0.5
    got = lib.series_responses(Lam, R, A, Q, H, n_shock=1)
    check_sr(got, Lam, R, A, Q, H, 1, models=(0, 65534, 65535, 65540, 68000, B - 1), bad=(65540, 68000))


# ---------------------------------------------------------------------------------------------------- 3. k_irf's shared memory
def irf_spec(M, Q, G, H, ids):
    """Q_sel M^h G[:, ids], (r, H, n_shock) (dfm_irf's output for one model)."""
    x = G[:, ids]
    out = []
    for _ in range(H):
        out.append(Q @ x)
        x = M @ x
    return np.stack(out, axis=1)


def check_irf(lib, r, p, H, ids, seed=6):
    """dfm_irf on the companion form of one sr_models model against irf_spec (1e-12 relative)."""
    Lam, R, A, Qm = sr_models(1, 2, r, p, seed=seed, out=())
    k = r * p
    M = np.zeros((k, k)); M[:r] = A[0]; M[r:, :k - r] = np.eye(k - r)
    Qs = np.zeros((r, k)); Qs[:, :r] = np.eye(r)
    G = np.zeros((k, r)); G[:r] = np.linalg.cholesky(Qm[0])
    got = lib.irf(M, Qs, G, H, ids)
    ref = irf_spec(M, Qs, G, H, list(ids))
    assert got.shape == ref.shape
    assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref)), np.max(np.abs(got - ref))


def check_sr_one(lib, r, p, H, ns, seed=7):
    _sr(lib, 1, 3, r, p, H, ns, seed=seed, out=())


@identified_case("irf_smem_k3069", {**SR, **IRF})
def _(lib, nsm, alloc):
    # r = 1, p = 3 069: k_irf needs (2 * 3 069 + 8) 8 = 49 168 B > 48 KiB, so its attribute must be raised (it was not: status 5
    # from both entry points); k_sr_prep's 3 069 x 3 069 companion, k_irf's rows 48 times around its 64 threads
    k = 3069
    assert irf_smem(k) > DEFAULT_SMEM >= irf_smem(k - 1)
    check_sr_one(lib, 1, k, 4, 1)
    check_irf(lib, 1, k, 4, [0])


@identified_case("irf_smem_set_per_call", {**SR, **IRF, **GIBBS_IRF})
def _(lib, nsm, alloc):
    # k_irf's attribute belongs to the kernel for the whole process; every launch site sets it to its own need on every call:
    # series responses at k = 1 set 80 B, then Gibbs impulse responses at k = 6 need 160 B; dfm_irf at k = 2 sets 96 B, then
    # series responses at k = 8 need 192 B and dfm_irf at k = 100 1 664 B; series responses at k = 3 069 (49 168 B) after them
    check_sr_one(lib, 1, 1, 3, 1)
    X, th = GC.model()
    GC.check_chains(lib, X, th, 2, n_chain=2, n_burn=1, n_keep=1, H_fc=1, fc_rows=2, H_irf=3)
    check_irf(lib, 2, 1, 3, [1, 0])
    check_sr_one(lib, 4, 2, 5, 2)
    check_irf(lib, 2, 50, 6, [1])
    check_sr_one(lib, 1, 3069, 3, 1)
    check_irf(lib, 1, 5, 3, [0])
    assert irf_smem(1) < irf_smem(6) and irf_smem(2) < irf_smem(8) < irf_smem(100)


@identified_case("irf_k14077_refused", SR)
def _(lib, nsm, alloc):
    # k = 14 077: (2 k + 8) 8 = 225 296 B > kMaxSmem = 225 280 B: both entry points refuse with status 6 before any allocation
    # (M alone would take 1.6 GB per model); the next call on the handle gives a fresh handle's bits
    k = 14077
    assert irf_smem(k) > KMAX_SMEM >= irf_smem(k - 1)
    Lam, R, A, Q = sr_models(1, 3, 1, 1, out=())
    Ab = np.full((1, k), 0.5 / k)
    assert _code(lambda: lib.series_responses(Lam[0], R[0], Ab, Q[0], 3)) == 6
    M = np.zeros(k * k)                   # (never touched: the refusal comes before any copy)
    Qs, G, out = np.zeros(k), np.zeros(k), np.zeros(3)
    assert _code(lambda: lib.irf_raw(M.ctypes.data, Qs.ctypes.data, G.ctypes.data, k, 1, 3, [0], 1, MEM_HOST, out.ctypes.data)) == 6
    Lam, R, A, Q = sr_models(3, 40, 3, 2, out=(5,))
    _same_as_fresh_handle(lib, lambda L: L.series_responses(Lam, R, A, Q, 6, n_shock=2))
