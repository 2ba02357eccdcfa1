"""Parity checks of dfm_historical_decomposition against the NumPy spec tests/history_oracle.py.  Each function takes a `Library`
(CUDA on an H100, or the host-emulation build of the same kernel source)."""
import numpy as np

from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, to_cm
import history_oracle as HO

NAMES = ("shocks", "contrib", "rest", "base")


def models(r, p, N, Tp, B, seed):
    """B stationary models (companion spectral radius <= 0.95) and B paths simulated from them; scale (N,)."""
    rng = np.random.default_rng(seed)
    Lam = rng.standard_normal((B, N, r)); R = 0.5 + rng.random((B, N))
    A = np.empty((B, r, r * p)); Q = np.empty((B, r, r)); F = np.empty((B, Tp, r))
    for b in range(B):
        A[b] = HO.stable_lags(rng.standard_normal((r, r * p)) / np.sqrt(r * p), p, 0.95)
        G = rng.standard_normal((r, r))
        Q[b] = G @ G.T / r + 0.5 * np.eye(r)
        F[b] = HO.simulate(Lam[b], A[b], Q[b], p, Tp, p - 1, rng)[0]
    return Lam, R, A, Q, F, 0.5 + rng.random(N)


def _close(g, e, what):
    assert (np.isnan(g) == np.isnan(e)).all(), what
    if np.isfinite(e).any():
        err = np.nanmax(np.abs(g - e))
        assert err <= 1e-12 * max(1.0, np.nanmax(np.abs(e))), (what, err)


def compare(got, Lam, R, A, Q, F, p, t0, ns, scale):
    """Every model of a batched call against the spec."""
    for b in range(Lam.shape[0]):
        ref = HO.decompose(Lam[b], R[b], A[b], Q[b], F[b], p, t0, n_shock=ns, scale=scale)
        assert got["status"][b] == ref[-1], b
        for n, e in zip(NAMES, ref[:-1]):
            _close(got[n][b], e, (n, b))


def check_against_spec(lib, r, p, N=13, Tp=24):
    """n_shock in {1, 2, r}, t0 in {p - 1, mid-sample, Tp - 1}, two models per call."""
    Lam, R, A, Q, F, sc = models(r, p, N, Tp, 2, seed=10 * r + p)
    for ns in sorted({1, min(2, r), r}):
        for t0 in sorted({p - 1, (p - 1 + Tp) // 2, Tp - 1}):
            got = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=sc)
            compare(got, Lam, R, A, Q, F, p, t0, ns, sc)
            inm = np.isfinite(got["base"])
            tot = got["base"] + got["contrib"].sum(-1) + got["rest"]
            common = sc[None, :, None] * np.einsum("bia,bta->bit", Lam, F)
            assert np.abs(tot - common)[inm].max() <= 1e-12 * np.abs(common).max()


def check_k49_refused(lib):
    Lam, R, A, Q, F, sc = models(7, 1, 5, 12, 1, seed=1)
    A7 = np.hstack([A[0] / 7] * 7)                                              # r = 7, p = 7: k = 49
    try:
        lib.historical_decomposition(Lam[0], R[0], A7, Q[0], F[0], 6)
    except DFMError as e:
        assert e.code == 6
    else:
        raise AssertionError("k = 49 accepted")


def failing_batch(r=3, p=2, N=9, Tp=20):
    """Five models: 1 a NaN A, 2 a Q that is not positive definite, 3 a NaN row in its path; series 4 of every model out (NaN R),
    series 6 of model 0 out (NaN loading)."""
    Lam, R, A, Q, F, sc = models(r, p, N, Tp, 5, seed=21)
    A[1, 0, 1] = np.nan
    Q[2] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    F[3, 7] = np.nan
    R[:, 4] = np.nan
    Lam[0, 6, 1] = np.nan
    return Lam, R, A, Q, F, sc


def check_failed_models_and_nan_series(lib):
    Lam, R, A, Q, F, sc = failing_batch()
    p, t0, ns = 2, 5, 2
    got = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=sc)
    assert list(got["status"]) == [0, 3, 3, 3, 0]
    compare(got, Lam, R, A, Q, F, p, t0, ns, sc)
    for b in (1, 2, 3):
        assert all(np.isnan(got[n][b]).all() for n in NAMES), b
    for b in (0, 4):
        assert np.isnan(got["base"][b, 4]).all() and np.isfinite(got["base"][b, 5]).all()
        assert np.isfinite(got["shocks"][b, p:]).all()
    assert np.isnan(got["contrib"][0, 6]).all() and np.isfinite(got["contrib"][4, 6]).all()
    one = lib.historical_decomposition(Lam[4], R[4], A[4], Q[4], F[4], t0, n_shock=ns, scale=sc)   # neighbours unaffected
    for n in NAMES:
        np.testing.assert_array_equal(one[n], got[n][4], err_msg=n)


def check_device_equals_host(lib, alloc):
    """The same call through device pointers gives the host call's bits, and NULL outputs leave the others unchanged."""
    Lam, R, A, Q, F, sc = failing_batch()
    B, N, r = Lam.shape; Tp = F.shape[1]; p, t0, ns = 2, 4, 2
    host = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=sc)
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dF, dsc = alloc(to_cm(F)), alloc(np.ascontiguousarray(sc))
    size = dict(shocks=Tp * r, contrib=N * Tp * ns, rest=N * Tp, base=N * Tp)
    o = {n: alloc(np.zeros(B * size[n])) for n in NAMES}
    st = alloc(np.zeros(B, np.int32))
    lib.historical_decomposition_raw({n: ins[n][0] for n in ins}, dF[0], N, r, p, Tp, t0, ns, B, dsc[0], MEM_DEVICE,
                                     status=st[0], **{n: o[n][0] for n in NAMES})
    lib.sync()
    shape = dict(shocks=(B, r, Tp), contrib=(B, ns, Tp, N), rest=(B, Tp, N), base=(B, Tp, N))
    for n in NAMES:
        v = o[n][1]().reshape(shape[n])
        v = v.transpose(0, 3, 2, 1) if v.ndim == 4 else v.transpose(0, 2, 1)
        np.testing.assert_array_equal(v, host[n], err_msg=n)
    np.testing.assert_array_equal(st[1](), host["status"])
    part = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=ns, scale=sc, outputs=("contrib",))
    np.testing.assert_array_equal(part["contrib"], host["contrib"])
    np.testing.assert_array_equal(part["status"], host["status"])


def check_chunks(lib, alloc):
    """More models than one chunk (r = 48, p = 1, n_shock = r, Tp = 14 000: about 270 MB of recursions per model, so one model
    per chunk in device and host memory): each model has the bits of a one-model call, with a failed model in a later chunk."""
    r, p, N, Tp, t0, B = 48, 1, 2, 14000, 0, 3
    rng = np.random.default_rng(48)
    Lam = rng.standard_normal((B, N, r)); R = 0.5 + rng.random((B, N))
    A = np.stack([0.5 * np.eye(r) + 0.01 * rng.standard_normal((r, r)) for _ in range(B)])
    Q = np.stack([np.eye(r) + 0.1 * np.diag(rng.random(r)) for _ in range(B)])
    F = rng.standard_normal((B, Tp, r))
    F[2, 100, 3] = np.nan
    big = lib.historical_decomposition(Lam, R, A, Q, F, t0, n_shock=r)
    assert list(big["status"]) == [0, 0, 3]
    for b in range(B):
        one = lib.historical_decomposition(Lam[b], R[b], A[b], Q[b], F[b], t0, n_shock=r)
        assert one["status"] == big["status"][b]
        for n in NAMES:
            np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dF = alloc(to_cm(F))
    o = alloc(np.zeros(B * N * Tp * r))
    st = alloc(np.zeros(B, np.int32))
    lib.historical_decomposition_raw({n: ins[n][0] for n in ins}, dF[0], N, r, p, Tp, t0, r, B, 0, MEM_DEVICE, contrib=o[0], status=st[0])
    lib.sync()
    np.testing.assert_array_equal(o[1]().reshape(B, r, Tp, N).transpose(0, 3, 2, 1), big["contrib"])
    np.testing.assert_array_equal(st[1](), big["status"])


def check_args(lib):
    Lam, R, A, Q, F, sc = models(3, 2, 6, 15, 2, seed=5)
    B, N, r = Lam.shape; Tp = F.shape[1]; p = 2
    bufs = dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R).ravel(), A=to_cm(A), Q=to_cm(Q))
    Fb = to_cm(F)
    base = np.zeros(B * N * Tp); st = np.zeros(B, np.int32)

    def code(models=None, F=Fb.ctypes.data, mem=MEM_HOST, **kw):
        a = dict(N=N, r=r, p=p, Tp=Tp, t0=p - 1, n_shock=1, n_model=B); a.update(kw)
        m = {n: v.ctypes.data for n, v in bufs.items()} if models is None else models
        try:
            lib.historical_decomposition_raw(m, F, a["N"], a["r"], a["p"], a["Tp"], a["t0"], a["n_shock"], a["n_model"], 0, mem,
                                             base=base.ctypes.data, status=st.ctypes.data)
            return 0
        except DFMError as e:
            return e.code

    for n in ("Lam", "R", "A", "Q"):                                            # a NULL required pointer
        assert code(models={m: (0 if m == n else v.ctypes.data) for m, v in bufs.items()}) == 1, n
    assert code(F=0) == 1
    assert code(t0=p - 2) == 1 and code(t0=Tp) == 1                             # t0 outside [p - 1, Tp)
    assert code(n_shock=0) == 1 and code(n_shock=r + 1) == 1                     # n_shock outside [1, r]
    assert code(mem=2) == 1 and code(mem=-1) == 1                               # a bad mem
    assert code(N=0) == 1 and code(n_model=0) == 1 and code(p=0) == 1 and code(Tp=0) == 1
    assert code(r=7, p=7, t0=6) == 6                                             # k = 49
    assert code(t0=Tp - 1, n_shock=r) == 0 and (st == 0).all()                  # the edges are accepted; the handle stays usable
    import ctypes as C
    from dynamic_factor_models_b200._lib import EmInit, HdOpts, HdOut
    ini = EmInit(**{n: C.c_void_p(v.ctypes.data) for n, v in bufs.items()})
    o = HdOpts(N=N, r=r, p=p, Tp=Tp, t0=p - 1, n_shock=1, n_model=B, mem=MEM_HOST)
    ou = HdOut(base=C.c_void_p(base.ctypes.data))
    f = lib.lib.dfm_historical_decomposition
    assert f(lib.h, None, C.c_void_p(Fb.ctypes.data), None, C.byref(o), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), C.c_void_p(Fb.ctypes.data), None, None, C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), C.c_void_p(Fb.ctypes.data), None, C.byref(o), None) == 1
    assert f(None, C.byref(ini), C.c_void_p(Fb.ctypes.data), None, C.byref(o), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), C.c_void_p(Fb.ctypes.data), None, C.byref(o), C.byref(ou)) == 0
