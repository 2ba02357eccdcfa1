"""Parity checks of dfm_proxy_identification against the NumPy spec tests/proxy_oracle.py.  Each function takes a `Library` (CUDA on
an H100, or the host-emulation build of the same kernel source)."""
import ctypes as C

import numpy as np

from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, EmInit, ProxyOpts, ProxyOut, to_cm
import proxy_oracle as PO
import sign_checks as SC

NAMES = ("omega", "resp", "fevd", "eps", "n_obs", "reliability", "fs_pi", "fs_F", "status")
BIG = 1 << 30                              # a block length past every n_k: each replicate is the sample itself


def paths(A, Q, p, Tp, seed):
    """Factor paths of the models (B, Tp, r) and their standardized shocks (B, Tp, r)."""
    B, r = Q.shape[0], Q.shape[1]
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((B, Tp, r))
    F = np.zeros((B, Tp, r))
    for b in range(B):
        Lc = np.linalg.cholesky(Q[b]) if not np.isnan(Q[b]).any() and (np.linalg.eigvalsh(Q[b]) > 0).all() else np.eye(r)
        An = np.nan_to_num(A[b])
        for t in range(Tp):
            f = Lc @ e[b, t]
            for l in range(1, min(p, t) + 1):
                f = f + An[:, (l - 1) * r:l * r] @ F[b, t - l]
            F[b, t] = f
    return F, e


def instruments(e, n_inst, seed, lead=4):
    """Tp x n_inst: instrument k = shock (k mod r) of model 0 plus noise, a leading NaN run and two gaps."""
    Tp, r = e.shape
    rng = np.random.default_rng(seed)
    Z = np.stack([e[:, k % r] + 0.5 * rng.standard_normal(Tp) for k in range(n_inst)], axis=1)
    Z[:lead] = np.nan
    Z[Tp // 2, 0] = np.nan
    Z[Tp // 3, n_inst - 1] = np.nan
    return Z


def _close(g, e, what, tol=1e-10):
    assert (np.isnan(g) == np.isnan(e)).all(), what
    if np.isfinite(e).any():
        err = np.nanmax(np.abs(g - e))
        assert err <= tol * max(1.0, np.nanmax(np.abs(e))), (what, err)


def compare(got, Lam, R, A, Q, F, Z, p, H, i0, q, block, n_boot, seed, ids, scale):
    for b in range(Lam.shape[0]):
        ref = PO.identify(Lam[b], R[b], A[b], Q[b], F[b], Z, p, H, i0, q=q, block=block, n_boot=n_boot, seed=seed, mid=int(ids[b]),
                          scale=scale)
        for n in NAMES:
            if n in got:
                if n in ("status", "n_obs"):
                    np.testing.assert_array_equal(got[n][b], ref[n], err_msg=str((n, b)))
                else:
                    _close(got[n][b], ref[n], (n, b))


def case(r, p, N=9, B=2, Tp=48, n_inst=1, seed=0):
    Lam, R, A, Q, sc = SC.models(r, p, N, B, seed=seed)
    F, e = paths(A, Q, p, Tp, seed + 1)
    return Lam, R, A, Q, F, instruments(e[0], n_inst, seed + 2), sc


def check_against_spec(lib, r, p, H=5, n_boot=6):
    """Two models with ids that are not 0 .. B-1; (n_inst, q, block) over one and three instruments, q 0 and 4, blocks 1, 7 and n_k."""
    ids = np.array([7, (5 << 24) + 3], np.uint64)
    for ni, q, block in ((1, 0, 1), (3, 4, 7), (3, 0, BIG), (1, 4, 7)):
        Lam, R, A, Q, F, Z, sc = case(r, p, n_inst=ni, seed=10 * r + p)
        got = lib.proxy_identification(Lam, R, A, Q, F, Z, 2, H, n_boot=n_boot, block=block, q=q, seed=100 + r, ids=ids, scale=sc)
        assert (got["status"] == 0).all(), got["status"]
        compare(got, Lam, R, A, Q, F, Z, p, H, 2, q, block, n_boot, 100 + r, ids, sc)
        if block == BIG:                                   # every replicate is the sample
            _close(got["omega"][:, :, 1:], np.broadcast_to(got["omega"][:, :, :1], got["omega"][:, :, 1:].shape), "omega block n_k")
        assert np.allclose(np.linalg.norm(got["omega"], axis=-1), 1.0)


def failing_batch(r=3, p=2, N=8, Tp=40):
    """Six models: 1 a NaN A, 2 a Q that is not positive definite, 3 a NaN path row inside instrument 0's periods (instrument 1,
    NaN there, is unaffected), 4 series i0 = 2 out of the model (NaN R); series 6 of every model out (NaN loading).  Instrument 2
    has two observations only (n_k < 3)."""
    Lam, R, A, Q, sc = SC.models(r, p, N, 6, seed=21)
    F, e = paths(A, Q, p, Tp, 22)
    A[1, 0, 1] = np.nan
    Q[2] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    F[3, 20, 1] = np.nan
    R[4, 2] = np.nan
    Lam[:, 6, 1] = np.nan
    Z = instruments(e[0], 3, 23)
    Z[18:24, 1] = np.nan                                   # (rows 20 .. 22 use the NaN row of model 3)
    Z[:, 2] = np.nan; Z[10, 2] = 1.0; Z[30, 2] = -1.0
    return Lam, R, A, Q, F, Z, sc


def check_failed_models(lib):
    Lam, R, A, Q, F, Z, sc = failing_batch()
    p, H, nbt = 2, 4, 5
    got = lib.proxy_identification(Lam, R, A, Q, F, Z, 2, H, n_boot=nbt, block=3, q=2, seed=9, scale=sc)
    np.testing.assert_array_equal(got["status"], [[0, 0, 3], [3, 3, 3], [3, 3, 3], [3, 0, 3], [1, 1, 1], [0, 0, 3]])
    compare(got, Lam, R, A, Q, F, Z, p, H, 2, 2, 3, nbt, 9, np.arange(6), sc)
    for b, k in zip(*np.nonzero(got["status"])):
        for n in ("omega", "resp", "fevd", "eps", "reliability", "fs_pi", "fs_F"):
            assert np.isnan(got[n][b, k]).all(), (n, b, k)
    assert np.isnan(got["resp"][0, 0, :, 6]).all() and np.isfinite(got["resp"][0, 0, :, 5]).all()
    for b in (0, 3, 5):                                    # neighbours unaffected
        one = lib.proxy_identification(Lam[b], R[b], A[b], Q[b], F[b], Z, 2, H, n_boot=nbt, block=3, q=2, seed=9, ids=[b], scale=sc)
        for n in NAMES:
            np.testing.assert_array_equal(one[n], got[n][b], err_msg=(n, b))


def _raw_device(lib, alloc, Lam, R, A, Q, F, Z, i0, H, n_boot, block, q, seed, ids=None, scale=None):
    B, N, r = Lam.shape; p = A.shape[2] // r; Tp = F.shape[1]; ni = Z.shape[1]; nr = 1 + n_boot
    ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
    dF, dZ = alloc(to_cm(F)), alloc(to_cm(Z))
    dsc = alloc(np.ascontiguousarray(scale)) if scale is not None else None
    size = dict(omega=ni * nr * r, resp=ni * nr * N * H, fevd=ni * nr * N * H, eps=ni * Tp, n_obs=ni, reliability=ni, fs_pi=ni, fs_F=ni,
                status=ni)
    o = {n: alloc(np.zeros(B * size[n], np.int32 if n in ("n_obs", "status") else np.float64)) for n in NAMES}
    lib.proxy_identification_raw({n: ins[n][0] for n in ins}, dF[0], dZ[0], ids, N, r, p, B, Tp, H, ni, i0, q, block, n_boot, seed,
                                 dsc[0] if dsc else 0, MEM_DEVICE, **{n: o[n][0] for n in NAMES})
    lib.sync()
    res = {n: o[n][1]().reshape(B, ni) for n in ("n_obs", "reliability", "fs_pi", "fs_F", "status")}
    res["omega"] = o["omega"][1]().reshape(B, ni, nr, r)
    res["eps"] = o["eps"][1]().reshape(B, ni, Tp)
    for n in ("resp", "fevd"):
        res[n] = o[n][1]().reshape(B, ni, nr, H, N).transpose(0, 1, 2, 4, 3)
    return res


def check_device_equals_host(lib, alloc):
    """The same call through device pointers gives the host call's bits, and NULL outputs leave the others unchanged."""
    Lam, R, A, Q, F, Z, sc = failing_batch()
    host = lib.proxy_identification(Lam, R, A, Q, F, Z, 2, 4, n_boot=7, block=2, q=1, seed=3, scale=sc)
    dev = _raw_device(lib, alloc, Lam, R, A, Q, F, Z, 2, 4, 7, 2, 1, 3, scale=sc)
    for n in NAMES:
        np.testing.assert_array_equal(dev[n], host[n], err_msg=n)
    part = lib.proxy_identification(Lam, R, A, Q, F, Z, 2, 4, n_boot=7, block=2, q=1, seed=3, scale=sc, outputs=("fevd", "fs_F"))
    for n in ("fevd", "fs_F", "status"):
        np.testing.assert_array_equal(part[n], host[n], err_msg=n)


def check_chunks(lib, alloc):
    """Model chunks and record batches: n_boot = 30 000 at one instrument puts two models in a chunk (chunks of 2, 2 and 1, a failed
    model in the middle one); three instruments put one model in a chunk with its records in two batches.  Each model has the bits
    of a one-model call, replicate rho the bits of a call with a smaller n_boot, and device memory the host's bits."""
    r, p, N, H, Tp = 2, 1, 4, 3, 30
    Lam, R, A, Q, sc = SC.models(r, p, N, 5, seed=48)
    F, e = paths(A, Q, p, Tp, 49)
    A[2, 0, 0] = np.nan
    Z = instruments(e[0], 3, 50)
    for Zc, B, nbt in ((Z[:, :1], 5, 30000), (Z, 2, 30000)):
        big = lib.proxy_identification(Lam[:B], R[:B], A[:B], Q[:B], F[:B], Zc, 1, H, n_boot=nbt, block=4, q=1, seed=5, scale=sc)
        assert (big["status"][2 if B > 2 else 0] == (3 if B > 2 else 0)).all()
        for b in range(B):
            one = lib.proxy_identification(Lam[b], R[b], A[b], Q[b], F[b], Zc, 1, H, n_boot=nbt, block=4, q=1, seed=5, ids=[b], scale=sc)
            for n in NAMES:
                np.testing.assert_array_equal(one[n], big[n][b], err_msg=(n, b))
        small = lib.proxy_identification(Lam[:B], R[:B], A[:B], Q[:B], F[:B], Zc, 1, H, n_boot=50, block=4, q=1, seed=5, scale=sc)
        for n in ("omega", "resp", "fevd"):
            np.testing.assert_array_equal(small[n], big[n][:, :, :51], err_msg=n)
        compare(small, Lam[:1], R[:1], A[:1], Q[:1], F[:1], Zc, p, H, 1, 1, 4, 50, 5, [0], sc)
    dev = _raw_device(lib, alloc, Lam[:2], R[:2], A[:2], Q[:2], F[:2], Z, 1, H, nbt, 4, 1, 5, scale=sc)
    for n in NAMES:
        np.testing.assert_array_equal(dev[n], big[n], err_msg=n)


def check_bounds(lib):
    """The largest accepted and first refused k = r p, n_inst, n_boot and Tp (the bootstrap kernel's shared memory)."""
    def code(r=2, p=1, ni=1, nbt=1, Tp=20):
        Lam, R, A, Q, _ = SC.models(r, p, 4, 1, seed=r)
        F, e = paths(A, Q, p, Tp, 1)
        Z = np.stack([e[0, :, 0] + 0.1 * k for k in range(ni)], axis=1)
        try:
            o = lib.proxy_identification(Lam, R, A, Q, F, Z, 0, 2, n_boot=nbt, block=3, seed=1, outputs=())
            assert (o["status"] == 0).all()
            return 0
        except DFMError as ex:
            return ex.code
    assert code(r=12, p=4) == 0 and code(r=7, p=7) == 6 and code(r=48) == 0 and code(r=49) == 6
    assert code(ni=8) == 0 and code(ni=9) == 6
    assert code(nbt=65535) == 0 and code(nbt=65536) == 6
    assert code(r=8, Tp=3072) == 0 and code(r=8, Tp=3073) == 6


def check_args(lib):
    Lam, R, A, Q, F, Z, sc = case(3, 2, B=2, n_inst=2, seed=5)
    B, N, r = Lam.shape; p, H, Tp = 2, 3, F.shape[1]
    bufs = dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R).ravel(), A=to_cm(A), Q=to_cm(Q))
    Fb, Zb = to_cm(F), to_cm(Z)
    st = np.zeros(B * 2, np.int32)

    def code(models=None, F_=Fb.ctypes.data, Z_=Zb.ctypes.data, ids=None, mem=MEM_HOST, **kw):
        a = dict(N=N, r=r, p=p, n_model=B, Tp=Tp, H=H, n_inst=2, i0=0, q=0, block=2, n_boot=3); a.update(kw)
        m = {n: v.ctypes.data for n, v in bufs.items()} if models is None else models
        try:
            lib.proxy_identification_raw(m, F_, Z_, ids, a["N"], a["r"], a["p"], a["n_model"], a["Tp"], a["H"], a["n_inst"], a["i0"],
                                         a["q"], a["block"], a["n_boot"], 1, 0, mem, status=st.ctypes.data)
            return 0
        except DFMError as e:
            return e.code

    for n in ("Lam", "R", "A", "Q"):                                            # a NULL required pointer
        assert code(models={m: (0 if m == n else v.ctypes.data) for m, v in bufs.items()}) == 1, n
    assert code(F_=0) == 1 and code(Z_=0) == 1
    assert code(i0=-1) == 1 and code(i0=N) == 1 and code(i0=N - 1) == 0
    assert code(q=-1) == 1 and code(block=0) == 1 and code(n_boot=-1) == 1 and code(n_boot=0) == 0
    assert code(n_inst=0) == 1 and code(Tp=0) == 1 and code(H=0) == 1
    assert code(mem=2) == 1 and code(mem=-1) == 1
    assert code(N=0) == 1 and code(n_model=0) == 1 and code(p=0) == 1 and code(r=0) == 1
    assert code(ids=np.array([0, 1 << 40], np.uint64)) == 1
    assert code(ids=np.array([0, (1 << 40) - 1], np.uint64)) == 0 and (st == 0).all()
    ini = EmInit(**{n: C.c_void_p(v.ctypes.data) for n, v in bufs.items()})
    o = ProxyOpts(N=N, r=r, p=p, n_model=B, Tp=Tp, H=H, n_inst=2, i0=0, q=0, block=2, n_boot=1, seed=1, mem=MEM_HOST)
    ou = ProxyOut(status=C.c_void_p(st.ctypes.data))
    f = lib.lib.dfm_proxy_identification
    Fp, Zp = C.c_void_p(Fb.ctypes.data), C.c_void_p(Zb.ctypes.data)
    assert f(None, C.byref(ini), Fp, Zp, None, None, C.byref(o), C.byref(ou)) == 1
    assert f(lib.h, None, Fp, Zp, None, None, C.byref(o), C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), Fp, Zp, None, None, None, C.byref(ou)) == 1
    assert f(lib.h, C.byref(ini), Fp, Zp, None, None, C.byref(o), None) == 1
    assert f(lib.h, C.byref(ini), Fp, Zp, None, None, C.byref(o), C.byref(ou)) == 0
