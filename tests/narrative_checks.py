"""Parity checks of dfm_narrative_sign_restrictions and dfm_percentiles_weighted against the NumPy spec
tests/narrative_oracle.py.  Each function takes a `Library` (CUDA on an H100, or the host-emulation build of the same kernel
source)."""
import ctypes as C

import numpy as np

from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, EmInit, NarrOpts, NarrOut, NarrRestr, SignRestr, to_cm
import narrative_oracle as NO
import sign_checks as SC
import sign_oracle as SO
import identified_oracle as IO

NAMES = ("rot", "resp", "fevd", "eps")


def path(r, Tp, seed):
    return np.random.default_rng(seed).standard_normal((Tp, r))


def narr_arrays(narr):
    """rows (kind, shock, series, t, h, sign) -> the six sequences of Library.narrative_sign_restrictions."""
    return [np.array([rw[q] for rw in narr], np.int64) for q in range(6)]


def compare(got, Lam, R, A, Q, F, p, rows, narr, H, ns, n_rot, n_keep, n_sim, seed, ids, scale):
    """Every model of a batched call against the spec; returns the spec's smallest decision margin."""
    margin = np.inf
    for b in range(Lam.shape[0]):
        ref = NO.identify(Lam[b], R[b], A[b], Q[b], F[b], p, rows, narr, H, ns, n_rot, n_keep, n_sim, seed=seed, mid=int(ids[b]),
                          scale=scale)
        assert got["status"][b] == ref["status"], (b, got["status"][b], ref["status"])
        assert got["n_accept"][b] == ref["n_accept"], (b, got["n_accept"][b], ref["n_accept"])
        np.testing.assert_array_equal(got["cand"][b], ref["cand"], err_msg=str(b))
        for n in NAMES:
            if n in got:
                SC._close(got[n][b], ref[n], (n, b))
        if "n_ok" in got:
            kept = ref["cand"] >= 0
            assert (np.abs(got["n_ok"][b][kept] - ref["n_ok"][kept]) <= ref["n_close"][kept]).all(), (b, got["n_ok"][b], ref["n_ok"])
            assert (got["n_ok"][b][~kept] == 0).all()
        if "weight" in got:
            kept = ref["cand"] >= 0
            assert np.isnan(got["weight"][b][~kept]).all()
            if (ref["n_close"][kept] == 0).all():
                np.testing.assert_array_equal(got["weight"][b][kept], ref["weight"][kept])
        margin = min(margin, ref["margin"])
    return margin


def case(Lam, A, Q, F, p, H, seed, mid, kinds=(0, 1, 2, 3)):
    """Sign rows on shock 1 (sign_checks.case_rows) and narrative rows that candidate 0 of model `mid` satisfies: kind 0 on
    shock 1 at row p (sign rows fix its orientation), kind 0 on shock 2 at row Tp - 1 with the sign that makes the flip group
    flip it, kind 3 on shock 1 over p .. p + H - 1, kinds 1 and 2 at rows p (h = 0) and Tp - 1 - (H - 1) (h = H - 1) on the shock
    that candidate 0 makes most important (overwhelming when it is, most important otherwise)."""
    N, r = Lam.shape
    Tp = F.shape[0]
    rows = SC.case_rows(Lam, A, Q, p, 1, H, seed, mid)
    om = SO.omegas(seed, mid, [0], r)[0]
    C = SO.row_vectors(Lam, A, Q, p, rows, H)
    f1 = 1 if (C @ om[:, 0] > 0).all() else -1
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, H)
    c_of = lambda i: np.einsum("a,hab->hb", Lam[i], P)
    narr = []
    if 0 in kinds:
        narr.append((0, 1, 0, p, 0, int(np.sign(f1 * (U[p] @ om[:, 0])))))
        if r >= 2:
            narr.append((0, 2, 0, Tp - 1, 0, -int(np.sign(U[Tp - 1] @ om[:, 1]))))
    if 3 in kinds:
        Hk = NO.contributions(c_of(2), om, U, p, H - 1)
        narr.append((3, 1, 2, p, H - 1, int(np.sign(Hk[0]))))
    for kd in (1, 2):
        if kd not in kinds:
            continue
        i, t, h = (1, p, 0) if kd == 1 else (N - 1, Tp - H, H - 1)
        Hk = NO.contributions(c_of(i), om, U, t, h)
        j = int(np.argmax(np.abs(Hk)))
        ok2 = NO._share(2, Hk, j)[0]
        narr.append((kd if ok2 or kd == 1 else 1, j + 1, i, t, h, 1))
    return rows, narr


def check_against_spec(lib, r, p, N=9, H=4, n_rot=300, n_keep=40, n_sim=512):
    Lam, R, A, Q, sc = SC.models(r, p, N, 2, seed=10 * r + p)
    Tp = p + H + 3
    F = np.stack([path(r, Tp, 5 + b) for b in range(2)])
    ids = np.array([5, (3 << 24) + 77], np.uint64)
    seed = 1000 + r
    for kinds in ((0, 1, 2, 3), (0,), (1,), (2,), (3,)):
        rows, narr = case(Lam[0], A[0], Q[0], F[0], p, H, seed, int(ids[0]), kinds)
        got = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), narr_arrays(narr), H, n_rot, n_keep, n_shock=r,
                                              n_sim=n_sim, seed=seed, ids=ids, scale=sc)
        margin = compare(got, Lam, R, A, Q, F, p, rows, narr, H, r, n_rot, n_keep, n_sim, seed, ids, sc)
        assert margin > 1e-9, margin
        assert got["n_accept"][0] > 0 and got["cand"][0, 0] == 0, (kinds, got["n_accept"])
        sign = lib.sign_restrictions(Lam, R, A, Q, SC.as_arrays(rows), H, n_rot, n_rot, n_shock=r, seed=seed, ids=ids, outputs=())
        for b in range(2):                                     # the narrative set is a subset of the sign set
            assert set(got["cand"][b][got["cand"][b] >= 0]) <= set(sign["cand"][b][sign["cand"][b] >= 0])


def check_no_narrative_rows(lib):
    """No narrative rows: dfm_sign_restrictions' bits, weight 1, n_ok = n_sim."""
    for r, p in ((3, 2), (8, 1)):
        Lam, R, A, Q, sc = SC.models(r, p, 9, 2, seed=r)
        F = np.stack([path(r, 12, b) for b in range(2)])
        rows = SC.case_rows(Lam[0], A[0], Q[0], p, min(2, r), 4, 7, 0)
        got = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), narr_arrays([]), 4, 500, 50, n_shock=min(2, r),
                                              n_sim=100, seed=7, scale=sc)
        ref = lib.sign_restrictions(Lam, R, A, Q, SC.as_arrays(rows), 4, 500, 50, n_shock=min(2, r), seed=7, scale=sc)
        for n in ("n_accept", "cand", "rot", "resp", "fevd", "status"):
            np.testing.assert_array_equal(got[n], ref[n], err_msg=n)
        kept = got["cand"] >= 0
        assert kept.any() and (got["weight"][kept] == 1.0).all() and (got["n_ok"][kept] == 100).all()
        assert np.isnan(got["weight"][~kept]).all() and (got["n_ok"][~kept] == 0).all()


def check_kind0_probability(lib):
    """Kind-0 rows only, on K = 3 distinct (shock, period) pairs: n_ok / n_sim within 5 sigma of 2^-3."""
    r, p, H = 3, 1, 3
    Lam, R, A, Q, sc = SC.models(r, p, 6, 1, seed=3)
    F = path(r, 10, 1)
    narr = [(0, 1, 0, 2, 0, 1), (0, 2, 0, 2, 0, -1), (0, 1, 0, 5, 0, 1)]
    n_sim = 1 << 14
    got = lib.narrative_sign_restrictions(Lam[0], R[0], A[0], Q[0], F, SC.as_arrays([]), narr_arrays(narr), H, 2000, 8, n_shock=2,
                                          n_sim=n_sim, seed=4, outputs=("n_ok", "weight"))
    assert got["n_accept"] > 0
    kept = got["cand"] >= 0
    sd = np.sqrt(0.125 * 0.875 / n_sim)
    assert (np.abs(got["n_ok"][kept] / n_sim - 0.125) < 5 * sd).all(), got["n_ok"]
    # the simulations are common to every candidate of the model: kind-0 rows do not depend on Omega
    assert len(set(got["n_ok"][kept].tolist())) == 1


def check_weighted_percentiles(lib):
    rng = np.random.default_rng(1)
    q = (0, 5, 16, 50, 84, 95, 100)
    for n in (1, 7, 64, 300, 1000, 5000, 16384):
        x = rng.standard_normal((n, 5 if n <= 1000 else 2))
        for w in (np.ones(n), rng.random(n) + 0.1, np.where(rng.random(n) < 0.3, 0.0, rng.random(n))):
            xx = x.copy()
            if n > 3:
                xx[1, 0] = np.nan; xx[::3, -1] = np.nan
            if 3 < n <= 1000:
                xx[:, 4] = np.nan                              # (a statistic with no counted record: NaN)
            got = lib.percentiles_weighted(xx, w, q)
            ref = NO.weighted_percentiles(xx, w, q)
            np.testing.assert_array_equal(got, ref, err_msg=str((n, w[:3])))


def failing_batch(r=3, p=2, N=8, Tp=10):
    """Seven models: 1 a NaN A, 2 a Q that is not positive definite, 3 a NaN path row, 4 a narrative series out of the model (NaN
    R), 6 both a NaN path row and a narrative series out of the model (the NaN path ranks first: status 3); series 6 of every
    model out (NaN loading, unrestricted)."""
    Lam, R, A, Q, sc = SC.models(r, p, N, 6, seed=21)
    Lam, R, A, Q = (np.concatenate([x, x[:1]]) for x in (Lam, R, A, Q))          # model 6: a copy of model 0
    F = np.stack([path(r, Tp, 30 + b) for b in range(6)] + [path(r, Tp, 30)])
    A[1, 0, 1] = np.nan
    Q[2] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    F[3, 4, 1] = np.nan
    R[4, 3] = np.nan
    F[6, 2, 0] = np.nan; R[6, 3] = np.nan
    Lam[:, 6, 1] = np.nan
    return Lam, R, A, Q, F, sc


FAIL_ROWS = SC.expand([(2, 1, 1, (0, 1))])
FAIL_NARR = [(0, 1, 0, 3, 0, 1), (1, 2, 3, 4, 1, 1)]


def check_failed_models(lib):
    Lam, R, A, Q, F, sc = failing_batch()
    p, H, ns, n_rot, n_keep = 2, 4, 2, 300, 12
    got = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(FAIL_ROWS), narr_arrays(FAIL_NARR), H, n_rot, n_keep, n_shock=ns,
                                          n_sim=256, seed=9, scale=sc)
    assert list(got["status"]) == [0, 3, 3, 3, 1, 0, 3], got["status"]
    compare(got, Lam, R, A, Q, F, p, FAIL_ROWS, FAIL_NARR, H, ns, n_rot, n_keep, 256, 9, np.arange(7), sc)
    for b in (1, 2, 3, 4, 6):
        assert got["n_accept"][b] == 0 and (got["cand"][b] == -1).all() and all(np.isnan(got[n][b]).all() for n in NAMES), b
    for b in (0, 5):
        assert got["n_accept"][b] > 0
        one = lib.narrative_sign_restrictions(Lam[b], R[b], A[b], Q[b], F[b], SC.as_arrays(FAIL_ROWS), narr_arrays(FAIL_NARR), H, n_rot,
                                              n_keep, n_shock=ns, n_sim=256, seed=9, ids=[b], scale=sc)
        for n in ("n_accept", "cand", "n_ok", "weight") + NAMES:
            np.testing.assert_array_equal(one[n], got[n][b], err_msg=(n, b))


def _raw_device(lib, alloc, Lam, R, A, Q, F, rows, narr, H, ns, n_rot, n_keep, n_sim, seed, scale=None):
    B, N, r = Lam.shape; p = A.shape[2] // r; Tp = F.shape[1]
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dF = alloc(to_cm(F))
    dsc = alloc(np.ascontiguousarray(scale)) if scale is not None else None
    size = dict(rot=n_keep * r * r, resp=n_keep * N * H * ns, fevd=n_keep * N * H * ns, eps=n_keep * Tp * ns, weight=n_keep)
    o = {n: alloc(np.zeros(B * size[n])) for n in size}
    na, ca, st = alloc(np.zeros(B, np.int64)), alloc(np.zeros(B * n_keep, np.int64)), alloc(np.zeros(B, np.int32))
    nok = alloc(np.zeros(B * n_keep, np.int64))
    lib.narrative_sign_restrictions_raw({n: ins[n][0] for n in ins}, dF[0], None, N, r, p, B, H, ns, n_rot, n_keep, seed, Tp, n_sim,
                                        SC.as_arrays(rows), narr_arrays(narr), dsc[0] if dsc else 0, MEM_DEVICE, n_accept=na[0],
                                        cand=ca[0], status=st[0], n_ok=nok[0], **{n: o[n][0] for n in size})
    lib.sync()
    res = dict(n_accept=na[1](), cand=ca[1]().reshape(B, n_keep), status=st[1](), n_ok=nok[1]().reshape(B, n_keep),
               weight=o["weight"][1]().reshape(B, n_keep), rot=o["rot"][1]().reshape(B, n_keep, r, r).transpose(0, 1, 3, 2),
               eps=o["eps"][1]().reshape(B, n_keep, ns, Tp).transpose(0, 1, 3, 2))
    for n in ("resp", "fevd"):
        res[n] = o[n][1]().reshape(B, n_keep, ns, H, N).transpose(0, 1, 4, 3, 2)
    return res


def check_device_equals_host(lib, alloc):
    Lam, R, A, Q, F, sc = failing_batch()
    H, ns, n_rot, n_keep = 4, 2, 200, 10
    host = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(FAIL_ROWS), narr_arrays(FAIL_NARR), H, n_rot, n_keep, n_shock=ns,
                                           n_sim=300, seed=3, scale=sc)
    dev = _raw_device(lib, alloc, Lam, R, A, Q, F, FAIL_ROWS, FAIL_NARR, H, ns, n_rot, n_keep, 300, 3, scale=sc)
    for n in ("n_accept", "cand", "status", "n_ok", "weight") + NAMES:
        np.testing.assert_array_equal(dev[n], host[n], err_msg=n)


def check_chunks(lib):
    """Two model chunks (n_keep = 30 000 puts two models in a chunk) and a partial second candidate batch (n_rot = 2^20 + 1000):
    every model has the bits of a one-model call."""
    r, p, N, H, B = 2, 1, 4, 3, 3
    n_rot, n_keep = (1 << 20) + 1000, 30000
    Lam, R, A, Q, sc = SC.models(r, p, N, B, seed=48)
    F = np.stack([path(r, 8, b) for b in range(B)])
    rows = SC.expand([(0, 1, 1, 0)])
    narr = [(0, 2, 0, 3, 0, 1)]
    big = lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), narr_arrays(narr), H, n_rot, n_keep, n_shock=2, n_sim=64,
                                          seed=5, scale=sc, outputs=("rot", "n_ok", "eps"))
    assert (big["status"] == 0).all() and (big["n_accept"] > n_keep).all(), big["n_accept"]
    for b in range(B):
        one = lib.narrative_sign_restrictions(Lam[b], R[b], A[b], Q[b], F[b], SC.as_arrays(rows), narr_arrays(narr), H, n_rot, n_keep,
                                              n_shock=2, n_sim=64, seed=5, ids=[b], scale=sc, outputs=("rot", "n_ok", "eps"))
        assert one["n_accept"] == big["n_accept"][b]
        for n in ("cand", "rot", "n_ok", "eps"):
            np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))


def check_bounds(lib):
    """The largest accepted and the first refused narrative row count, nP r, n_sim and r."""
    def code(r=3, p=1, nN=1, kind=0, Tp=20, n_sim=16, H=2, spread=False, nsign=0, h=1):
        Lam, R, A, Q, _ = SC.models(r, p, 4, 1, seed=r)
        F = path(r, Tp, 1)
        narr = [(kind, 1, 0, (p + q if spread else p), 0 if kind == 0 else h, 1) for q in range(nN)]
        rows = [(q % 4, q % 2, 1 + q % r, 1) for q in range(nsign)]
        try:
            lib.narrative_sign_restrictions(Lam, R, A, Q, F, SC.as_arrays(rows), narr_arrays(narr), H, 64, 2, n_shock=r, n_sim=n_sim,
                                            seed=1, outputs=())
            return 0
        except DFMError as e:
            return e.code
    assert code(nN=64) == 0 and code(nN=65) == 6
    assert code(r=16, nN=25, kind=2, nsign=256) == 0 and code(r=16, nN=26, kind=2, nsign=256) == 6     # k_narr_cand's shared memory
    assert code(r=16, p=1, nN=64, Tp=1100, spread=True) == 0                                            # nP r = 1024
    assert code(r=16, nN=1, kind=1, h=1023, H=1030, Tp=1100) == 0                                       # nP r = 2^14
    assert code(r=16, nN=1, kind=1, h=1024, H=1030, Tp=1100) == 6                                       # nP r = 1025 * 16
    assert code(n_sim=1 << 20) == 0 and code(n_sim=(1 << 20) + 1) == 6
    assert code(r=17) == 6


def check_args(lib):
    Lam, R, A, Q, sc = SC.models(3, 2, 6, 2, seed=5)
    B, N, r = Lam.shape; p, H, Tp = 2, 3, 10
    F = np.stack([path(r, Tp, b) for b in range(B)])
    bufs = dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R).ravel(), A=to_cm(A), Q=to_cm(Q))
    Fb = to_cm(F)
    na = np.zeros(B, np.int64); st = np.zeros(B, np.int32)
    good = [(0, 1, 0, 2, 0, 1), (1, 2, 3, 4, 2, 1)]

    def code(narr=good, F_=Fb.ctypes.data, **kw):
        a = dict(n_shock=2, n_sim=10, Tp=Tp, H=H); a.update(kw)
        try:
            lib.narrative_sign_restrictions_raw({n: v.ctypes.data for n, v in bufs.items()}, F_, None, N, r, p, B, a["H"], a["n_shock"], 10,
                                                2, 1, a["Tp"], a["n_sim"], SC.as_arrays([]), narr_arrays(narr), 0, MEM_HOST,
                                                n_accept=na.ctypes.data, status=st.ctypes.data)
            return 0
        except DFMError as e:
            return e.code
    assert code() == 0 and code(narr=[]) == 0
    assert code(narr=[(4, 1, 0, 2, 0, 1)]) == 1 and code(narr=[(-1, 1, 0, 2, 0, 1)]) == 1      # kind
    assert code(narr=[(0, 1, 0, 2, 0, 0)]) == 1 and code(narr=[(3, 1, 0, 2, 0, 2)]) == 1       # sign on kinds 0 / 3
    assert code(narr=[(1, 1, 0, 2, 0, 0)]) == 0                                                # (sign unused on kinds 1 / 2)
    assert code(narr=[(0, 1, 0, p - 1, 0, 1)]) == 1 and code(narr=[(0, 1, 0, Tp, 0, 1)]) == 1  # row < p, row >= Tp
    assert code(narr=[(1, 1, 0, Tp - 2, 2, 1)]) == 1 and code(narr=[(1, 1, 0, Tp - 3, 2, 1)]) == 0   # row + h >= Tp
    assert code(narr=[(1, 1, 0, 2, H, 1)]) == 1 and code(narr=[(1, 1, 0, 2, -1, 1)]) == 1      # h outside [0, H)
    assert code(narr=[(0, 3, 0, 2, 0, 1)]) == 1 and code(narr=[(0, 0, 0, 2, 0, 1)]) == 1       # shock outside [1, n_shock]
    assert code(narr=[(1, 1, N, 2, 0, 1)]) == 1 and code(narr=[(1, 1, -1, 2, 0, 1)]) == 1      # series outside [0, N)
    assert code(n_sim=0) == 1 and code(Tp=0) == 1 and code(F_=0) == 1
    ini = EmInit(**{n: C.c_void_p(v.ctypes.data) for n, v in bufs.items()})
    o = NarrOpts(N=N, r=r, p=p, n_model=B, H=H, n_shock=1, n_rot=10, n_keep=2, seed=1, mem=MEM_HOST, Tp=Tp, n_sim=4)
    rs = SignRestr(0, None, None, None, None)
    nr0 = NarrRestr(0, None, None, None, None, None, None)
    nr_null = NarrRestr(1, None, None, None, None, None, None)
    ou = NarrOut(n_accept=C.c_void_p(na.ctypes.data))
    f = lib.lib.dfm_narrative_sign_restrictions
    Fp = C.c_void_p(Fb.ctypes.data)
    assert f(lib.h, C.byref(ini), Fp, None, None, C.byref(o), C.byref(rs), C.byref(nr0), C.byref(ou)) == 0
    assert f(lib.h, C.byref(ini), Fp, None, None, C.byref(o), C.byref(rs), None, C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), Fp, None, None, C.byref(o), C.byref(rs), C.byref(nr_null), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), Fp, None, None, C.byref(o), None, C.byref(nr0), C.byref(ou)) == 1
    w = np.ones(4); x = np.zeros((4, 2)); out = np.zeros(2); qq = np.array([50.0])
    g = lib.lib.dfm_percentiles_weighted
    P = lambda a_: a_.ctypes.data_as(C.c_void_p)
    assert g(lib.h, P(x), P(w), 4, 2, P(qq), 1, MEM_HOST, P(out)) == 0
    assert g(lib.h, P(x), None, 4, 2, P(qq), 1, MEM_HOST, P(out)) == 1
    assert g(lib.h, P(x), P(w), 0, 2, P(qq), 1, MEM_HOST, P(out)) == 1
    assert g(lib.h, P(x), P(w), 4, 2, P(np.array([101.0])), 1, MEM_HOST, P(out)) == 1
    big = np.ones(16385)
    assert g(lib.h, P(big), P(big), 16384, 1, P(qq), 1, MEM_HOST, P(out)) == 0
    assert g(lib.h, P(big), P(big), 16385, 1, P(qq), 1, MEM_HOST, P(out)) == 6
