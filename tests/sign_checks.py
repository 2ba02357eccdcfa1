"""Parity checks of dfm_sign_restrictions against the NumPy spec tests/sign_oracle.py.  Each function takes a `Library` (CUDA on an
H100, or the host-emulation build of the same kernel source)."""
import ctypes as C

import numpy as np

from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, EmInit, SignOpts, SignOut, SignRestr, to_cm
import history_oracle as HO
import sign_oracle as SO

NAMES = ("rot", "resp", "fevd")


def models(r, p, N, B, seed):
    """B stationary models (companion spectral radius <= 0.95) and a scale (N,)."""
    rng = np.random.default_rng(seed)
    Lam = rng.standard_normal((B, N, r)); R = 0.5 + rng.random((B, N))
    A = np.empty((B, r, r * p)); Q = np.empty((B, r, r))
    for b in range(B):
        A[b] = HO.stable_lags(rng.standard_normal((r, r * p)) / np.sqrt(r * p), p, 0.95)
        G = rng.standard_normal((r, r))
        Q[b] = G @ G.T / r + 0.5 * np.eye(r)
    return Lam, R, A, Q, 0.5 + rng.random(N)


def expand(restrictions):
    """[(series, shock, sign, horizons)] with horizons an int or an inclusive (lo, hi) -> rows (i, h, j, s)."""
    rows = []
    for i, j, s, hz in restrictions:
        lo, hi = (hz, hz) if np.isscalar(hz) else hz
        rows += [(i, h, j, s) for h in range(lo, hi + 1)]
    return rows


def as_arrays(rows):
    """rows (i, h, j, s) -> the four sequences of Library.sign_restrictions."""
    return [np.array([rw[q] for rw in rows], np.int64) for q in range(4)]


def _close(g, e, what, tol=1e-10):
    assert (np.isnan(g) == np.isnan(e)).all(), what
    if np.isfinite(e).any():
        err = np.nanmax(np.abs(g - e))
        assert err <= tol * max(1.0, np.nanmax(np.abs(e))), (what, err)


def compare(got, Lam, R, A, Q, p, rows, H, ns, n_rot, n_keep, seed, ids, scale):
    """Every model of a batched call against the spec; returns the spec's smallest decision margin."""
    margin = np.inf
    for b in range(Lam.shape[0]):
        ref = SO.identify(Lam[b], R[b], A[b], Q[b], p, rows, H, ns, n_rot, n_keep, seed=seed, mid=int(ids[b]), scale=scale)
        assert got["status"][b] == ref["status"], b
        assert got["n_accept"][b] == ref["n_accept"], (b, got["n_accept"][b], ref["n_accept"])
        np.testing.assert_array_equal(got["cand"][b], ref["cand"], err_msg=str(b))
        for n in NAMES:
            if n in got:
                _close(got[n][b], ref[n], (n, b))
        margin = min(margin, ref["margin"])
    return margin


def case_rows(Lam, A, Q, p, ns, H, seed, mid):
    """Rows on several shocks with horizon ranges (an unrestricted shock 2 inside n_shock where n_shock >= 3), their signs those
    of candidate 0 of model `mid` with shock n_shock's flipped, so that candidate is accepted (with shock n_shock flipped)."""
    N, r = Lam.shape
    res = [(0, 1, 1, (0, min(1, H - 1))), (3, 1, 1, 0)]
    if ns >= 2:
        res += [(1, ns, 1, (0, H - 1)), (N - 1, ns, 1, H - 1)]
    rows = expand(res)
    om = SO.omegas(seed, mid, [0], r)[0]
    C = SO.row_vectors(Lam, A, Q, p, rows, H)
    return [(i, h, j, int(np.sign(C[q] @ om[:, j - 1])) * (-1 if j == ns and ns > 1 else 1)) for q, (i, h, j, s) in enumerate(rows)]


def check_against_spec(lib, r, p, N=9, H=5, n_rot=300, n_keep=40):
    """n_shock in {1, 2, r}, two models per call with ids that are not 0 .. B-1."""
    Lam, R, A, Q, sc = models(r, p, N, 2, seed=10 * r + p)
    ids = np.array([5, (3 << 24) + 77], np.uint64)
    seed = 1000 + r
    for ns in sorted({1, min(2, r), r}):
        rows = case_rows(Lam[0], A[0], Q[0], p, ns, H, seed, int(ids[0]))
        got = lib.sign_restrictions(Lam, R, A, Q, as_arrays(rows), H, n_rot, n_keep, n_shock=ns, seed=seed, ids=ids, scale=sc)
        margin = compare(got, Lam, R, A, Q, p, rows, H, ns, n_rot, n_keep, seed, ids, sc)
        assert margin > 1e-9, margin
        assert got["n_accept"][0] > 0 and got["cand"][0, 0] == 0


def failing_batch(r=3, p=2, N=8):
    """Five models: 1 a NaN A, 2 a Q that is not positive definite, 3 a restricted series out of the model (NaN R); series 6 of
    every model out (NaN loading, unrestricted)."""
    Lam, R, A, Q, sc = models(r, p, N, 5, seed=21)
    A[1, 0, 1] = np.nan
    Q[2] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    R[3, 2] = np.nan
    Lam[:, 6, 1] = np.nan
    return Lam, R, A, Q, sc


FAIL_ROWS = expand([(2, 1, 1, (0, 1)), (0, 2, -1, 2)])


def check_failed_models(lib):
    Lam, R, A, Q, sc = failing_batch()
    p, H, ns, n_rot, n_keep = 2, 4, 2, 200, 16
    got = lib.sign_restrictions(Lam, R, A, Q, as_arrays(FAIL_ROWS), H, n_rot, n_keep, n_shock=ns, seed=9, scale=sc)
    assert list(got["status"]) == [0, 3, 3, 1, 0]
    compare(got, Lam, R, A, Q, p, FAIL_ROWS, H, ns, n_rot, n_keep, 9, np.arange(5), sc)
    for b in (1, 2, 3):
        assert got["n_accept"][b] == 0 and (got["cand"][b] == -1).all() and all(np.isnan(got[n][b]).all() for n in NAMES), b
    for b in (0, 4):
        assert got["n_accept"][b] > 0 and np.isnan(got["resp"][b, :, 6]).all() and np.isfinite(got["resp"][b, 0, 5]).all()
    one = lib.sign_restrictions(Lam[4], R[4], A[4], Q[4], as_arrays(FAIL_ROWS), H, n_rot, n_keep, n_shock=ns, seed=9, ids=[4],
                                scale=sc)                                       # neighbours unaffected
    assert one["n_accept"] == got["n_accept"][4]
    for n in ("cand",) + NAMES:
        np.testing.assert_array_equal(one[n], got[n][4], err_msg=n)


def _raw_device(lib, alloc, Lam, R, A, Q, rows, H, ns, n_rot, n_keep, seed, ids=None, scale=None):
    B, N, r = Lam.shape; p = A.shape[2] // r
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dsc = alloc(np.ascontiguousarray(scale)) if scale is not None else None
    size = dict(rot=n_keep * r * r, resp=n_keep * N * H * ns, fevd=n_keep * N * H * ns)
    o = {n: alloc(np.zeros(B * size[n])) for n in NAMES}
    na, ca, st = alloc(np.zeros(B, np.int64)), alloc(np.zeros(B * n_keep, np.int64)), alloc(np.zeros(B, np.int32))
    lib.sign_restrictions_raw({n: ins[n][0] for n in ins}, ids, N, r, p, B, H, ns, n_rot, n_keep, seed, as_arrays(rows),
                              dsc[0] if dsc else 0, MEM_DEVICE, n_accept=na[0], cand=ca[0], status=st[0], **{n: o[n][0] for n in NAMES})
    lib.sync()
    res = dict(n_accept=na[1](), cand=ca[1]().reshape(B, n_keep), status=st[1](),
               rot=o["rot"][1]().reshape(B, n_keep, r, r).transpose(0, 1, 3, 2))
    for n in ("resp", "fevd"):
        res[n] = o[n][1]().reshape(B, n_keep, ns, H, N).transpose(0, 1, 4, 3, 2)
    return res


def check_device_equals_host(lib, alloc):
    """The same call through device pointers gives the host call's bits, and NULL outputs leave the others unchanged."""
    Lam, R, A, Q, sc = failing_batch()
    H, ns, n_rot, n_keep = 4, 2, 150, 12
    host = lib.sign_restrictions(Lam, R, A, Q, as_arrays(FAIL_ROWS), H, n_rot, n_keep, n_shock=ns, seed=3, scale=sc)
    dev = _raw_device(lib, alloc, Lam, R, A, Q, FAIL_ROWS, H, ns, n_rot, n_keep, 3, scale=sc)
    for n in ("n_accept", "cand", "status") + NAMES:
        np.testing.assert_array_equal(dev[n], host[n], err_msg=n)
    part = lib.sign_restrictions(Lam, R, A, Q, as_arrays(FAIL_ROWS), H, n_rot, n_keep, n_shock=ns, seed=3, scale=sc, outputs=("fevd",))
    for n in ("n_accept", "cand", "status", "fevd"):
        np.testing.assert_array_equal(part[n], host[n], err_msg=n)


def check_chunks(lib, alloc):
    """Several model chunks and candidate batches: n_keep = 30 000 puts two models in a chunk (the rotated records of all kept slots
    of a chunk sit on one grid axis), n_rot = 2^20 + 1000 takes two candidate batches, the second partial; no rows on shock 2.
    Each model has the bits of a one-model call, a failed model in the first chunk leaves the others alone, and the device-memory
    call gives the host call's bits."""
    r, p, N, H, B, ns = 2, 1, 4, 3, 3, 2
    n_rot, n_keep = (1 << 20) + 1000, 30000
    Lam, R, A, Q, sc = models(r, p, N, B, seed=48)
    A[1, 0, 0] = np.nan
    rows = expand([(0, 1, 1, 0), (1, 1, 1, 0), (2, 1, -1, 0), (3, 1, 1, 0)])
    big = lib.sign_restrictions(Lam, R, A, Q, as_arrays(rows), H, n_rot, n_keep, n_shock=ns, seed=5, scale=sc)
    assert list(big["status"]) == [0, 3, 0]
    assert (big["n_accept"][[0, 2]] > n_keep).all(), big["n_accept"]                  # (the first batch fills the slots)
    for b in range(B):
        one = lib.sign_restrictions(Lam[b], R[b], A[b], Q[b], as_arrays(rows), H, n_rot, n_keep, n_shock=ns, seed=5, ids=[b], scale=sc)
        assert one["n_accept"] == big["n_accept"][b] and one["status"] == big["status"][b]
        for n in ("cand",) + NAMES:
            np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))
    ref = SO.identify(Lam[2], R[2], A[2], Q[2], p, rows, H, ns, n_rot, 4, seed=5, mid=2)
    assert big["n_accept"][2] == ref["n_accept"]
    np.testing.assert_array_equal(big["cand"][2, :4], ref["cand"])
    dev = _raw_device(lib, alloc, Lam, R, A, Q, rows, H, ns, n_rot, n_keep, 5, scale=sc)
    for n in ("n_accept", "cand", "status") + NAMES:
        np.testing.assert_array_equal(dev[n], big[n], err_msg=n)


def check_partial_tiles(lib):
    """n_rot not a multiple of the tile: each prefix n_rot gives the spec's count and the first ids of the larger call."""
    Lam, R, A, Q, sc = models(3, 2, 6, 1, seed=4)
    rows = expand([(0, 1, 1, (0, 2)), (1, 1, 1, 1)])
    full = lib.sign_restrictions(Lam[0], R[0], A[0], Q[0], as_arrays(rows), 4, 1000, 1000, seed=2, outputs=())
    for n_rot in (1, 31, 33, 64, 65, 999):
        got = lib.sign_restrictions(Lam[0], R[0], A[0], Q[0], as_arrays(rows), 4, n_rot, 8, seed=2, outputs=())
        keep = full["cand"][(full["cand"] >= 0) & (full["cand"] < n_rot)]
        assert got["n_accept"] == len(keep), n_rot
        np.testing.assert_array_equal(got["cand"][:min(8, len(keep))], keep[:8])


def check_bounds(lib):
    """The largest accepted and first refused r, n_shock and number of rows."""
    def code(r, ns=1, nrow=1, p=1):
        Lam, R, A, Q, _ = models(r, p, 4, 1, seed=r)
        rows = [(q % 4, q % 2, 1 + q % ns, 1) for q in range(nrow)]
        try:
            lib.sign_restrictions(Lam, R, A, Q, as_arrays(rows), 2, 64, 2, n_shock=ns, seed=1, outputs=())
            return 0
        except DFMError as e:
            return e.code
    assert code(16, ns=16, nrow=256) == 0
    assert code(17) == 6 and code(16, nrow=257) == 6 and code(16, ns=17) == 1
    assert code(8, ns=8, nrow=256) == 0 and code(12, p=4) == 0 and code(7, p=7) == 6   # (k = 48 accepted, 49 refused)


def check_args(lib):
    Lam, R, A, Q, sc = models(3, 2, 6, 2, seed=5)
    B, N, r = Lam.shape; p, H = 2, 3
    bufs = dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R).ravel(), A=to_cm(A), Q=to_cm(Q))
    na = np.zeros(B, np.int64); st = np.zeros(B, np.int32)
    good = [(0, 0, 1, 1), (1, 2, 2, -1)]

    def code(models=None, rows=good, ids=None, mem=MEM_HOST, **kw):
        a = dict(N=N, r=r, p=p, n_model=B, H=H, n_shock=2, n_rot=10, n_keep=2); a.update(kw)
        m = {n: v.ctypes.data for n, v in bufs.items()} if models is None else models
        try:
            lib.sign_restrictions_raw(m, ids, a["N"], a["r"], a["p"], a["n_model"], a["H"], a["n_shock"], a["n_rot"], a["n_keep"], 1,
                                      as_arrays(rows), 0, mem, n_accept=na.ctypes.data, status=st.ctypes.data)
            return 0
        except DFMError as e:
            return e.code

    for n in ("Lam", "R", "A", "Q"):                                            # a NULL required pointer
        assert code(models={m: (0 if m == n else v.ctypes.data) for m, v in bufs.items()}) == 1, n
    assert code(rows=[(-1, 0, 1, 1)]) == 1 and code(rows=[(N, 0, 1, 1)]) == 1  # series outside [0, N)
    assert code(rows=[(0, -1, 1, 1)]) == 1 and code(rows=[(0, H, 1, 1)]) == 1  # horizon outside [0, H)
    assert code(rows=[(0, 0, 0, 1)]) == 1 and code(rows=[(0, 0, 3, 1)]) == 1   # shock outside [1, n_shock]
    assert code(rows=[(0, 0, 1, 0)]) == 1 and code(rows=[(0, 0, 1, 2)]) == 1   # sign not +-1
    assert code(n_shock=0) == 1 and code(n_shock=r + 1, rows=[]) == 1
    assert code(n_rot=0) == 1 and code(n_keep=0) == 1
    assert code(mem=2) == 1 and code(mem=-1) == 1
    assert code(N=0) == 1 and code(n_model=0) == 1 and code(p=0) == 1 and code(H=0) == 1 and code(r=0) == 1
    assert code(ids=np.array([0, 1 << 40], np.uint64)) == 1
    assert code(ids=np.array([0, (1 << 40) - 1], np.uint64)) == 0
    assert code(n_keep=65536) == 6
    assert code(rows=[]) == 0 and code(n_shock=r, rows=[(0, H - 1, r, -1)]) == 0 and (st == 0).all()
    ini = EmInit(**{n: C.c_void_p(v.ctypes.data) for n, v in bufs.items()})
    o = SignOpts(N=N, r=r, p=p, n_model=B, H=H, n_shock=1, n_rot=10, n_keep=2, seed=1, mem=MEM_HOST)
    rs = SignRestr(0, None, None, None, None)
    rs_null = SignRestr(1, None, None, None, None)
    ou = SignOut(n_accept=C.c_void_p(na.ctypes.data))
    f = lib.lib.dfm_sign_restrictions
    assert f(None, C.byref(ini), None, None, C.byref(o), C.byref(rs), C.byref(ou)) == 1
    assert f(lib.h, None, None, None, C.byref(o), C.byref(rs), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), None, None, None, C.byref(rs), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), None, None, C.byref(o), None, C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), None, None, C.byref(o), C.byref(rs), None) == 1
    assert f(lib.h, C.byref(ini), None, None, C.byref(o), C.byref(rs_null), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), None, None, C.byref(o), C.byref(rs), C.byref(ou)) == 0
