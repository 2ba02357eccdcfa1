"""ctypes binding of include/dfm_b200.h.  Every symbol the header declares is bound here
(tests/test_abi.py checks the export list against the header)."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

MEM_HOST, MEM_DEVICE = 0, 1
STATUS = {0: "ok", 1: "bad argument", 2: "too few observations", 3: "not positive definite",
          4: "not converged", 5: "CUDA error / no device", 6: "unsupported size", 7: "NCCL error"}

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)


class DFMError(RuntimeError):
    def __init__(self, code, where, detail=""):
        self.code = code
        super().__init__(f"{where}: status {code} ({STATUS.get(code, '?')}) {detail}")


class FactorOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("N", C.c_int), ("r", C.c_int), ("nt_min", C.c_int), ("tol", C.c_double),
                ("max_iter", C.c_longlong), ("compute_r2", C.c_int), ("n_constr", C.c_int),
                ("constr_index", c_ip), ("constr_R", c_dp), ("constr_r", c_dp), ("batch", C.c_int), ("mem", C.c_int)]


class FactorStats(C.Structure):
    _fields_ = [("ssr", C.c_double), ("tss", C.c_double), ("nobs", C.c_longlong), ("iters", C.c_int), ("status", C.c_int)]


class LoadingOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("ns", C.c_int), ("r", C.c_int), ("nt_min", C.c_int), ("n_uarlag", C.c_int),
                ("n_constr", C.c_int), ("constr_index", c_ip), ("constr_R", c_dp), ("constr_r", c_dp),
                ("batch", C.c_int), ("mem", C.c_int)]


class BootOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("ns", C.c_int), ("r", C.c_int), ("p", C.c_int), ("n_uarlag", C.c_int), ("n_resid", C.c_int),
                ("burn", C.c_int), ("batch", C.c_int), ("mem", C.c_int), ("seed", C.c_ulonglong), ("rep0", C.c_longlong)]


class EmOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("N", C.c_int), ("r", C.c_int), ("p", C.c_int), ("max_iter", C.c_int),
                ("tol", C.c_double), ("batch", C.c_int), ("mem", C.c_int), ("path", C.c_int)]


class EmInit(C.Structure):
    _fields_ = [("Lam", C.c_void_p), ("R", C.c_void_p), ("A", C.c_void_p), ("Q", C.c_void_p), ("P0", C.c_void_p)]


class EmOut(C.Structure):
    _fields_ = [("Lam", C.c_void_p), ("R", C.c_void_p), ("A", C.c_void_p), ("Q", C.c_void_p), ("P0", C.c_void_p),
                ("F", C.c_void_p), ("PF", C.c_void_p), ("loglik", C.c_void_p), ("iters", C.c_void_p), ("status", C.c_void_p)]


class SsOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("N", C.c_int), ("r", C.c_int), ("p", C.c_int), ("H", C.c_int), ("batch", C.c_int), ("mem", C.c_int)]


class SsOut(C.Structure):
    _fields_ = [("F", C.c_void_p), ("PF", C.c_void_p), ("common", C.c_void_p), ("xhat", C.c_void_p), ("xvar", C.c_void_p),
                ("loglik", C.c_void_p), ("status", C.c_void_p)]


SS_OUTPUTS = ("F", "PF", "common", "xhat", "xvar")


class SimOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("N", C.c_int), ("r", C.c_int), ("p", C.c_int), ("H", C.c_int), ("n_draw", C.c_longlong),
                ("draw0", C.c_longlong), ("seed", C.c_ulonglong), ("mem", C.c_int)]


class SimOut(C.Structure):
    _fields_ = [("F", C.c_void_p), ("X", C.c_void_p), ("status", C.c_void_p)]


class NewsOpts(C.Structure):
    _fields_ = [("T", C.c_int), ("N", C.c_int), ("r", C.c_int), ("p", C.c_int), ("H", C.c_int), ("news_rows", C.c_int),
                ("n_target", C.c_int), ("target_series", c_ip), ("target_period", c_ip), ("batch", C.c_int), ("mem", C.c_int)]


class NewsOut(C.Structure):
    _fields_ = [("old_est", C.c_void_p), ("new_est", C.c_void_p), ("news", C.c_void_p), ("weight", C.c_void_p),
                ("contrib", C.c_void_p), ("status", C.c_void_p)]


NEWS_OUTPUTS = ("old_est", "new_est", "news", "weight", "contrib")


def default_library_path():
    return os.path.join(HERE, "lib", "libdfm_b200.so")


EXPORTS = ["dfm_version", "dfm_status_string", "dfm_create", "dfm_create_on_stream", "dfm_destroy", "dfm_sync",
           "dfm_launch_count", "dfm_last_error", "dfm_profile_enable", "dfm_profile_query", "dfm_profile_reset",
           "dfm_profile_kernel_name", "dfm_standardize", "dfm_pca_score", "dfm_estimate_factor",
           "dfm_estimate_loading", "dfm_estimate_loading_ex", "dfm_estimate_var", "dfm_irf", "dfm_instability", "dfm_fit_correlation", "dfm_em_kalman", "dfm_kalman_smooth", "dfm_simulation_smoother",
           "dfm_news", "dfm_em_init_from_factors",
           "dfm_simulate_panels", "dfm_bootstrap_panels", "dfm_bootstrap_irf", "dfm_percentiles", "dfm_allgather_results", "dfm_shard_range"]


def _ptr(a):
    """numpy array -> void*; int -> device pointer; None -> NULL."""
    if a is None:
        return None
    if isinstance(a, (int, np.integer)):
        return C.c_void_p(int(a))
    return a.ctypes.data_as(C.c_void_p)


def to_cm(X):
    """(rows, cols) or (B, rows, cols) array -> contiguous buffer holding column-major panels."""
    X = np.asarray(X, dtype=np.float64)
    if X.ndim == 1:
        return np.ascontiguousarray(X)
    if X.ndim == 2:
        return np.ascontiguousarray(X.T)
    return np.ascontiguousarray(X.transpose(0, 2, 1))


def from_cm(buf, rows, cols, batch=None):
    """inverse of to_cm for an output buffer of batch*rows*cols doubles."""
    if batch is None:
        return np.ascontiguousarray(buf.reshape(cols, rows).T)
    return np.ascontiguousarray(buf.reshape(batch, cols, rows).transpose(0, 2, 1))


class Library:
    """One loaded libdfm_b200.so + one dfm_handle.  `path=None` loads the in-tree CUDA build and
    raises if it is absent (no fallback); tests may pass the host-emulation harness explicitly."""

    def __init__(self, path=None, device=0, stream=None):
        path = path or default_library_path()
        if not os.path.exists(path):
            raise DFMError(5, "load", f"{path} not found: build it with __graft_entry__.build() (needs nvcc); "
                                      "there is no CPU fallback")
        self.path = path
        self.lib = C.CDLL(path)
        L = self.lib
        L.dfm_status_string.restype = C.c_char_p
        L.dfm_last_error.restype = C.c_char_p
        L.dfm_last_error.argtypes = [C.c_void_p]
        L.dfm_launch_count.restype = C.c_longlong
        L.dfm_launch_count.argtypes = [C.c_void_p]
        L.dfm_profile_enable.argtypes = [C.c_void_p, C.c_int]
        L.dfm_profile_query.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
        L.dfm_profile_reset.argtypes = [C.c_void_p]
        L.dfm_profile_kernel_name.argtypes = [C.c_void_p, C.c_int]
        L.dfm_profile_kernel_name.restype = C.c_char_p
        L.dfm_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.dfm_create_on_stream.argtypes = [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
        L.dfm_destroy.argtypes = [C.c_void_p]
        L.dfm_sync.argtypes = [C.c_void_p]
        L.dfm_standardize.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.dfm_pca_score.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.dfm_estimate_factor.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(FactorOpts), C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(FactorStats)]
        L.dfm_estimate_loading.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LoadingOpts), C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]
        L.dfm_estimate_loading_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LoadingOpts)] + [C.c_void_p] * 7
        L.dfm_estimate_var.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 6
        L.dfm_irf.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, c_ip,
                              C.c_int, C.c_int, C.c_void_p]
        L.dfm_em_kalman.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(EmOpts), C.POINTER(EmInit), C.POINTER(EmOut)]
        L.dfm_kalman_smooth.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(SsOpts), C.POINTER(EmInit), C.POINTER(SsOut)]
        L.dfm_simulation_smoother.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(SimOpts), C.POINTER(EmInit), C.POINTER(SimOut)]
        L.dfm_news.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(NewsOpts), C.POINTER(EmInit), C.POINTER(NewsOut)]
        L.dfm_simulate_panels.argtypes = [C.c_void_p, C.c_ulonglong, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p]
        L.dfm_bootstrap_panels.argtypes = [C.c_void_p, C.POINTER(BootOpts)] + [C.c_void_p] * 8
        L.dfm_bootstrap_irf.argtypes = [C.c_void_p, C.POINTER(BootOpts)] + [C.c_void_p] * 7 + [C.c_int, C.c_double, C.c_int, C.c_void_p,
                                                                                               C.c_void_p, C.c_void_p]
        L.dfm_percentiles.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.dfm_em_init_from_factors.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                               C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.dfm_allgather_results.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]
        L.dfm_shard_range.argtypes = [C.c_longlong, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
        self.h = C.c_void_p()
        rc = L.dfm_create_on_stream(device, C.c_void_p(stream) if stream else None, C.byref(self.h))
        if rc != 0:
            raise DFMError(rc, "dfm_create", "(a CUDA device is required; there is no CPU fallback)")

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.dfm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc, where):
        if rc != 0:
            raise DFMError(rc, where, self.lib.dfm_last_error(self.h).decode())

    def sync(self):
        self.check(self.lib.dfm_sync(self.h), "dfm_sync")

    @property
    def launches(self):
        return int(self.lib.dfm_launch_count(self.h))

    def profile(self, on=True):
        self.lib.dfm_profile_reset(self.h)
        self.lib.dfm_profile_enable(self.h, int(on))

    def profile_report(self):
        """{kernel name: (total ms, launches)} since profile(True)."""
        out = {}
        i = 0
        while True:
            nm = self.lib.dfm_profile_kernel_name(self.h, i)
            if not nm:
                break
            ms, cnt = C.c_double(), C.c_longlong()
            self.lib.dfm_profile_query(self.h, nm, C.byref(ms), C.byref(cnt))
            out[nm.decode()] = (ms.value, cnt.value)
            i += 1
        return out

    def em_kalman_raw(self, X, T, N, r, p, B, max_iter, tol, init, out, mem, path=0):
        """Pointer-level call (ints = device or pinned-host addresses).  init/out: dicts of
        name -> address (missing = NULL)."""
        o = EmOpts(T=T, N=N, r=r, p=p, max_iter=max_iter, tol=tol, batch=B, mem=mem, path=path)
        ini = EmInit(**{k: C.c_void_p(v) if v else None for k, v in init.items()})
        ou = EmOut(**{k: C.c_void_p(v) if v else None for k, v in out.items()})
        self.check(self.lib.dfm_em_kalman(self.h, C.c_void_p(X), C.byref(o), C.byref(ini), C.byref(ou)), "dfm_em_kalman")

    def kalman_smooth_raw(self, X, T, N, r, p, H, B, params, out, mem):
        """Pointer-level dfm_kalman_smooth (ints = device or host addresses).  params: dict Lam, R, A, Q[, P0]; out: dict of
        F, PF, common, xhat, xvar, loglik, status (missing or 0 = NULL)."""
        o = SsOpts(T=T, N=N, r=r, p=p, H=H, batch=B, mem=mem)
        ini = EmInit(**{k: C.c_void_p(v) if v else None for k, v in params.items()})
        ou = SsOut(**{k: C.c_void_p(v) if v else None for k, v in out.items()})
        self.check(self.lib.dfm_kalman_smooth(self.h, C.c_void_p(X), C.byref(o), C.byref(ini), C.byref(ou)), "dfm_kalman_smooth")

    def simulation_smoother_raw(self, X, T, N, r, p, H, n_draw, draw0, seed, params, out, mem):
        """Pointer-level dfm_simulation_smoother (ints = device or host addresses).  params: dict Lam, R, A, Q[, P0]; out: dict
        of F, X, status (missing or 0 = NULL)."""
        o = SimOpts(T=T, N=N, r=r, p=p, H=H, n_draw=n_draw, draw0=draw0, seed=seed, mem=mem)
        ini = EmInit(**{k: C.c_void_p(v) if v else None for k, v in params.items()})
        ou = SimOut(**{k: C.c_void_p(v) if v else None for k, v in out.items()})
        self.check(self.lib.dfm_simulation_smoother(self.h, C.c_void_p(X), C.byref(o), C.byref(ini), C.byref(ou)),
                   "dfm_simulation_smoother")

    def news_raw(self, X_old, X_new, T, N, r, p, H, B, news_rows, targets, params, out, mem):
        """Pointer-level dfm_news (ints = device or host addresses).  targets: (series, period) pairs, 0-based; params: dict
        Lam, R, A, Q[, P0]; out: dict of old_est, new_est, news, weight, contrib, status (missing or 0 = NULL)."""
        ts = np.ascontiguousarray([t[0] for t in targets], dtype=np.int32)
        tp = np.ascontiguousarray([t[1] for t in targets], dtype=np.int32)
        o = NewsOpts(T=T, N=N, r=r, p=p, H=H, news_rows=news_rows, n_target=len(ts), target_series=ts.ctypes.data_as(c_ip),
                     target_period=tp.ctypes.data_as(c_ip), batch=B, mem=mem)
        ini = EmInit(**{k: C.c_void_p(v) if v else None for k, v in params.items()})
        ou = NewsOut(**{k: C.c_void_p(v) if v else None for k, v in out.items()})
        self.check(self.lib.dfm_news(self.h, C.c_void_p(X_old), C.c_void_p(X_new), C.byref(o), C.byref(ini), C.byref(ou)), "dfm_news")

    def estimate_factor_raw(self, X, T, N, r, B, mem, F=0, Lam=0, nt_min=20, tol=1e-8, max_iter=100000000, F_init=0):
        o = FactorOpts(T=T, N=N, r=r, nt_min=nt_min, tol=tol, max_iter=max_iter, compute_r2=0, batch=B, mem=mem)
        st = (FactorStats * B)()
        vp = lambda a: C.c_void_p(a) if a else None
        self.check(self.lib.dfm_estimate_factor(self.h, C.c_void_p(X), C.byref(o), vp(F_init), vp(F), vp(Lam), None, None, None, st),
                   "dfm_estimate_factor")
        return [dict(ssr=s.ssr, tss=s.tss, nobs=s.nobs, iters=s.iters, status=s.status) for s in st]

    # pointer-level wrappers of the replication pipeline (device-resident C4 step: addresses are ints)
    def bootstrap_panels_raw(self, T, ns, r, p, L, n_resid, burn, B, seed, rep0, ptrs, X, mem=MEM_DEVICE):
        """ptrs = (F0, resid, beta, lam, uar_coef, uar_ser, data) addresses."""
        o = BootOpts(T=T, ns=ns, r=r, p=p, n_uarlag=L, n_resid=n_resid, burn=burn, batch=B, mem=mem, seed=seed, rep0=rep0)
        self.check(self.lib.dfm_bootstrap_panels(self.h, C.byref(o), *[C.c_void_p(a_) for a_ in ptrs], C.c_void_p(X)), "dfm_bootstrap_panels")

    def estimate_var_raw(self, F, T, r, p, withconst, B, mem, betahat=0, resid=0, seps=0, M=0, Q=0, G=0):
        vp = lambda a: C.c_void_p(a) if a else None
        self.check(self.lib.dfm_estimate_var(self.h, C.c_void_p(F), T, r, p, int(withconst), B, mem, vp(betahat), vp(resid), vp(seps),
                                             vp(M), vp(Q), vp(G)), "dfm_estimate_var")

    def irf_raw(self, M, Q, G, k, r, H, shock_ids, B, mem, out):
        ids = np.ascontiguousarray(shock_ids, dtype=np.int32)
        self.check(self.lib.dfm_irf(self.h, C.c_void_p(M), C.c_void_p(Q), C.c_void_p(G), k, r, H, len(ids), ids.ctypes.data_as(c_ip), B, mem,
                                    C.c_void_p(out)), "dfm_irf")

    def percentiles_raw(self, recs, n, d, q, out, mem=MEM_DEVICE):
        qq = np.ascontiguousarray(q, dtype=float)
        self.check(self.lib.dfm_percentiles(self.h, C.c_void_p(recs), n, d, _ptr(qq), len(qq), mem, C.c_void_p(out)), "dfm_percentiles")

    def shard_range(self, n_rep, rank, world):
        b, e = C.c_longlong(), C.c_longlong()
        rc = self.lib.dfm_shard_range(n_rep, rank, world, C.byref(b), C.byref(e))
        if rc != 0:
            raise DFMError(rc, "dfm_shard_range")
        return b.value, e.value

    # ------------------------------------------------------------ numpy-level wrappers (host memory)
    def standardize(self, X):
        X = np.asarray(X, float); b = X.shape[0] if X.ndim == 3 else None
        T, N = X.shape[-2:]; B = b or 1
        xin = to_cm(X); xs = np.empty(B * T * N); mu = np.empty(B * N); sd = np.empty(B * N)
        self.check(self.lib.dfm_standardize(self.h, _ptr(xin), T, N, B, MEM_HOST, _ptr(xs), _ptr(mu), _ptr(sd)), "dfm_standardize")
        return from_cm(xs, T, N, b), (mu.reshape(B, N) if b else mu), (sd.reshape(B, N) if b else sd)

    def pca_score(self, X, r):
        X = np.asarray(X, float); b = X.shape[0] if X.ndim == 3 else None
        T, N = X.shape[-2:]; B = b or 1
        xin = to_cm(X); sc = np.empty(B * T * r)
        self.check(self.lib.dfm_pca_score(self.h, _ptr(xin), T, N, r, B, MEM_HOST, _ptr(sc)), "dfm_pca_score")
        return from_cm(sc, T, r, b)

    def estimate_factor(self, X, r, nt_min=20, tol=1e-8, max_iter=100000000, compute_r2=True, constr=None, F_init=None):
        """X (T,N) or (B,T,N) raw estimation block.  constr = (index[int], R[n_c x r], r[n_c]) or None."""
        X = np.asarray(X, float); b = X.shape[0] if X.ndim == 3 else None
        T, N = X.shape[-2:]; B = b or 1
        xin = to_cm(X)
        o = FactorOpts(T=T, N=N, r=r, nt_min=nt_min, tol=tol, max_iter=max_iter, compute_r2=int(compute_r2), batch=B, mem=MEM_HOST)
        keep = []
        if constr is not None:
            idx = np.ascontiguousarray(constr[0], dtype=np.int32); Rm = to_cm(np.asarray(constr[1], float))
            rv = np.ascontiguousarray(constr[2], dtype=np.float64); keep = [idx, Rm, rv]
            o.n_constr = len(idx); o.constr_index = idx.ctypes.data_as(c_ip); o.constr_R = Rm.ctypes.data_as(c_dp)
            o.constr_r = rv.ctypes.data_as(c_dp)
        F = np.empty(B * T * r); Lam = np.empty(B * N * r); R2 = np.full(B * N, np.nan); mu = np.empty(B * N); sd = np.empty(B * N)
        st = (FactorStats * B)()
        fi = to_cm(F_init) if F_init is not None else None
        self.check(self.lib.dfm_estimate_factor(self.h, _ptr(xin), C.byref(o), _ptr(fi), _ptr(F), _ptr(Lam), _ptr(R2), _ptr(mu),
                                                _ptr(sd), st), "dfm_estimate_factor")
        stats = [dict(ssr=s.ssr, tss=s.tss, nobs=s.nobs, iters=s.iters, status=s.status) for s in st]
        out = dict(F=from_cm(F, T, r, b), Lam=from_cm(Lam, N, r, b), R2=R2.reshape(B, N) if b else R2,
                   xmean=mu.reshape(B, N) if b else mu, xstd=sd.reshape(B, N) if b else sd, stats=stats if b else stats[0])
        del keep
        return out

    def estimate_loading(self, data, F, nt_min=40, n_uarlag=4, constr=None):
        data = np.asarray(data, float); F = np.asarray(F, float); b = data.shape[0] if data.ndim == 3 else None
        T, ns = data.shape[-2:]; r = F.shape[-1]; B = b or 1
        o = LoadingOpts(T=T, ns=ns, r=r, nt_min=nt_min, n_uarlag=n_uarlag, batch=B, mem=MEM_HOST)
        keep = []
        if constr is not None:
            idx = np.ascontiguousarray(constr[0], dtype=np.int32); Rm = to_cm(np.asarray(constr[1], float))
            rv = np.ascontiguousarray(constr[2], dtype=np.float64); keep = [idx, Rm, rv]
            o.n_constr = len(idx); o.constr_index = idx.ctypes.data_as(c_ip); o.constr_R = Rm.ctypes.data_as(c_dp)
            o.constr_r = rv.ctypes.data_as(c_dp)
        din, fin = to_cm(data), to_cm(F)
        lam = np.empty(B * ns * r); r2 = np.empty(B * ns); ac = np.empty(B * ns * n_uarlag); ser = np.empty(B * ns)
        con = np.empty(B * ns); res = np.empty(B * ns * T); st = np.zeros(B, np.int32)
        self.check(self.lib.dfm_estimate_loading_ex(self.h, _ptr(din), _ptr(fin), C.byref(o), _ptr(lam), _ptr(r2), _ptr(ac), _ptr(ser),
                                                    _ptr(con), _ptr(res), _ptr(st)), "dfm_estimate_loading")
        del keep
        return dict(lam=from_cm(lam, ns, r, b), r2=r2.reshape(B, ns) if b else r2, uar_coef=from_cm(ac, ns, n_uarlag, b),
                    uar_ser=ser.reshape(B, ns) if b else ser, constant=con.reshape(B, ns) if b else con,
                    resid=from_cm(res, T, ns, b), status=st if b else int(st[0]))

    def estimate_var(self, F, p, withconst=True):
        F = np.asarray(F, float); b = F.shape[0] if F.ndim == 3 else None
        T, r = F.shape[-2:]; B = b or 1; k = r * p; K = k + int(withconst)
        fin = to_cm(F)
        beta = np.empty(B * K * r); res = np.empty(B * T * r); seps = np.empty(B * r * r)
        M = np.empty(B * k * k); Q = np.empty(B * r * k); G = np.empty(B * k * r)
        self.check(self.lib.dfm_estimate_var(self.h, _ptr(fin), T, r, p, int(withconst), B, MEM_HOST, _ptr(beta), _ptr(res),
                                             _ptr(seps), _ptr(M), _ptr(Q), _ptr(G)), "dfm_estimate_var")
        return dict(betahat=from_cm(beta, K, r, b), resid=from_cm(res, T, r, b), seps=from_cm(seps, r, r, b),
                    M=from_cm(M, k, k, b), Q=from_cm(Q, r, k, b), G=from_cm(G, k, r, b))

    # ------------------------------------------------------------ replication generators / bands
    def simulate_panels(self, rep0, B, N, r, T, seed, want_F=False):
        """(B, T, N) standardised panels of replication ids rep0 .. rep0+B-1 (and the true factors (B, T, r))."""
        X = np.empty(B * T * N); F = np.empty(B * T * r) if want_F else None
        self.check(self.lib.dfm_simulate_panels(self.h, seed, rep0, B, T, N, r, MEM_HOST, _ptr(X), _ptr(F)), "dfm_simulate_panels")
        Xo = from_cm(X, T, N, B)
        return (Xo, from_cm(F, T, r, B)) if want_F else Xo

    def simulate_panels_raw(self, rep0, B, N, r, T, seed, X, F=0, mem=MEM_DEVICE):
        self.check(self.lib.dfm_simulate_panels(self.h, seed, rep0, B, T, N, r, mem, C.c_void_p(X), C.c_void_p(F) if F else None),
                   "dfm_simulate_panels")

    def bootstrap_panels(self, F0, resid, beta, lam, uar_coef, uar_ser, data, rep0, B, seed, burn=50):
        """(B, Tw, ns) residual-bootstrap draws of replication ids rep0 .. rep0+B-1."""
        F0 = np.asarray(F0, float); Tw, r = F0.shape; ns, Lg = np.asarray(uar_coef).shape; K = np.asarray(beta).shape[0]
        o = BootOpts(T=Tw, ns=ns, r=r, p=(K - 1) // r, n_uarlag=Lg, n_resid=np.asarray(resid).shape[0], burn=burn, batch=B, mem=MEM_HOST,
                     seed=seed, rep0=rep0)
        X = np.empty(B * ns * Tw)
        bufs = [to_cm(np.asarray(a_, float)) for a_ in (F0, resid, beta, lam, uar_coef)] + [np.ascontiguousarray(uar_ser, dtype=float),
                                                                                               to_cm(np.asarray(data, float))]
        self.check(self.lib.dfm_bootstrap_panels(self.h, C.byref(o), *[_ptr(b_) for b_ in bufs], _ptr(X)), "dfm_bootstrap_panels")
        return from_cm(X, Tw, ns, B)

    def bootstrap_irf(self, F0, resid, beta, lam, uar_coef, uar_ser, data, rep0, B, seed, H, nt_min=20, tol=1e-8, burn=50):
        """The whole C4 replication step on the device: (B, r, H, r) impulse responses [variable, horizon, shock] of the
        re-estimated models of bootstrap draws rep0 .. rep0+B-1, plus the ALS iteration counts / statuses."""
        F0 = np.asarray(F0, float); Tw, r = F0.shape; ns, Lg = np.asarray(uar_coef).shape; K = np.asarray(beta).shape[0]
        o = BootOpts(T=Tw, ns=ns, r=r, p=(K - 1) // r, n_uarlag=Lg, n_resid=np.asarray(resid).shape[0], burn=burn, batch=B, mem=MEM_HOST,
                     seed=seed, rep0=rep0)
        bufs = [to_cm(np.asarray(a_, float)) for a_ in (F0, resid, beta, lam, uar_coef)] + [np.ascontiguousarray(uar_ser, dtype=float),
                                                                                               to_cm(np.asarray(data, float))]
        out = np.empty(B * r * H * r); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self.check(self.lib.dfm_bootstrap_irf(self.h, C.byref(o), *[_ptr(b_) for b_ in bufs], nt_min, tol, H, _ptr(out), _ptr(it), _ptr(st)),
                   "dfm_bootstrap_irf")
        return np.ascontiguousarray(out.reshape(B, r, H, r).transpose(0, 3, 2, 1)), it, st

    def percentiles(self, recs, q):
        """recs (n, d) -> (len(q), d): numpy.percentile(recs, q, axis=0) on the device, NaN records ignored."""
        recs = np.ascontiguousarray(recs, dtype=float); n, d = recs.shape
        qq = np.ascontiguousarray(q, dtype=float); out = np.empty(len(qq) * d)
        self.check(self.lib.dfm_percentiles(self.h, _ptr(recs), n, d, _ptr(qq), len(qq), MEM_HOST, _ptr(out)), "dfm_percentiles")
        return out.reshape(len(qq), d)

    def irf(self, M, Q, G, H, shock_ids):
        M = np.asarray(M, float); b = M.shape[0] if M.ndim == 3 else None; B = b or 1
        k = M.shape[-1]; r = np.asarray(Q).shape[-2]
        ids = np.ascontiguousarray(shock_ids, dtype=np.int32); ns_ = len(ids)
        out = np.empty(B * r * H * ns_)
        self.check(self.lib.dfm_irf(self.h, _ptr(to_cm(M)), _ptr(to_cm(Q)), _ptr(to_cm(G)), k, r, H, ns_, ids.ctypes.data_as(c_ip),
                                    B, MEM_HOST, _ptr(out)), "dfm_irf")
        o = out.reshape(B, ns_, H, r).transpose(0, 3, 2, 1)      # -> (B, r, H, n_shock)
        return np.ascontiguousarray(o if b else o[0])

    def instability(self, data, F, T_break, q=6, ccut=0.15, min_obs=80, want_q0=False):
        """Chow / QLR statistics (HAC, q lags) of the regression of every column of data (T, ns) on F (T, r); NaN = missing.
        Returns dict(chow, qlr[, qlr0], status)."""
        data = np.asarray(data, float); F = np.asarray(F, float)
        T, ns = data.shape; r = F.shape[1]
        chow = np.empty(ns); qlr = np.empty(ns); qlr0 = np.empty(ns) if want_q0 else None; st = np.zeros(ns, np.int32)
        self.check(self.lib.dfm_instability(self.h, _ptr(to_cm(data)), _ptr(to_cm(F)), T, ns, r, q, T_break, C.c_double(ccut), min_obs, MEM_HOST,
                                            _ptr(chow), _ptr(qlr), _ptr(qlr0), st.ctypes.data_as(c_ip)), "dfm_instability")
        out = dict(chow=chow, qlr=qlr, status=st)
        if want_q0:
            out["qlr0"] = qlr0
        return out

    def fit_correlation(self, data, F, F_alt, T_break, min_obs=80):
        """cor(yhat on F, yhat on F_alt) per column of data (Table 4(a), lower half)."""
        data = np.asarray(data, float); F = np.asarray(F, float); Fa = np.asarray(F_alt, float)
        T, ns = data.shape; r = F.shape[1]
        cor = np.empty(ns); st = np.zeros(ns, np.int32)
        self.check(self.lib.dfm_fit_correlation(self.h, _ptr(to_cm(data)), _ptr(to_cm(F)), _ptr(to_cm(Fa)), T, ns, r, T_break, min_obs, MEM_HOST,
                                                _ptr(cor), st.ctypes.data_as(c_ip)), "dfm_fit_correlation")
        return cor

    def em_init_from_factors(self, Xs, F, p=1):
        Xs = np.asarray(Xs, float); F = np.asarray(F, float); b = Xs.shape[0] if Xs.ndim == 3 else None
        T, N = Xs.shape[-2:]; r = F.shape[-1]; B = b or 1; k = r * p
        Lam = np.empty(B * N * r); R = np.empty(B * N); A = np.empty(B * r * k); Q = np.empty(B * r * r)
        self.check(self.lib.dfm_em_init_from_factors(self.h, _ptr(to_cm(Xs)), _ptr(to_cm(F)), T, N, r, p, B, MEM_HOST, _ptr(Lam),
                                                     _ptr(R), _ptr(A), _ptr(Q)), "dfm_em_init_from_factors")
        return from_cm(Lam, N, r, b), (R.reshape(B, N) if b else R), from_cm(A, r, k, b), from_cm(Q, r, r, b)

    def em_kalman(self, X, Lam, R, A, Q, p=1, P0=None, max_iter=50, tol=0.0, path=0, want_PF=True):
        X = np.asarray(X, float); b = X.shape[0] if X.ndim == 3 else None
        T, N = X.shape[-2:]; r = np.asarray(Lam).shape[-1]; B = b or 1; k = r * p
        o = EmOpts(T=T, N=N, r=r, p=p, max_iter=max_iter, tol=tol, batch=B, mem=MEM_HOST, path=path)
        bufs = dict(X=to_cm(X), Lam=to_cm(Lam), R=np.ascontiguousarray(R, dtype=float), A=to_cm(A), Q=to_cm(Q),
                    P0=to_cm(P0) if P0 is not None else None)
        ini = EmInit(Lam=_ptr(bufs["Lam"]), R=_ptr(bufs["R"]), A=_ptr(bufs["A"]), Q=_ptr(bufs["Q"]), P0=_ptr(bufs["P0"]))
        oL = np.empty(B * N * r); oR = np.empty(B * N); oA = np.empty(B * r * k); oQ = np.empty(B * r * r); oP0 = np.empty(B * k * k)
        oF = np.empty(B * T * r); oPF = np.empty(B * T * r * r) if want_PF else None; oll = np.empty(B * max_iter)
        oit = np.empty(B, dtype=np.int32); ost = np.empty(B, dtype=np.int32)
        out = EmOut(Lam=_ptr(oL), R=_ptr(oR), A=_ptr(oA), Q=_ptr(oQ), P0=_ptr(oP0), F=_ptr(oF), PF=_ptr(oPF), loglik=_ptr(oll),
                    iters=_ptr(oit), status=_ptr(ost))
        self.check(self.lib.dfm_em_kalman(self.h, _ptr(bufs["X"]), C.byref(o), C.byref(ini), C.byref(out)), "dfm_em_kalman")
        res = dict(Lam=from_cm(oL, N, r, b), R=oR.reshape(B, N) if b else oR, A=from_cm(oA, r, k, b), Q=from_cm(oQ, r, r, b),
                   P0=from_cm(oP0, k, k, b), F=from_cm(oF, T, r, b), loglik=oll.reshape(B, max_iter) if b else oll,
                   iters=oit if b else int(oit[0]), status=ost if b else int(ost[0]))
        if want_PF:
            pf = oPF.reshape(B, T, r, r)
            res["PF"] = pf if b else pf[0]
        return res

    def kalman_smooth(self, X, Lam, R, A, Q, p=1, P0=None, H=0, outputs=SS_OUTPUTS):
        """Smoothed factors, forecasts and imputed values at FIXED parameters (dfm_kalman_smooth).  X (T, N) or (B, T, N)
        standardized with NaN; parameters as em_kalman.  Returns F (T+H, r), PF (T+H, r, r), common / xhat / xvar (T+H, N)
        -- those named in `outputs` -- plus loglik and status (per panel for batched input)."""
        X = np.asarray(X, float); b = X.shape[0] if X.ndim == 3 else None
        T, N = X.shape[-2:]; r = np.asarray(Lam).shape[-1]; B = b or 1; Tp = T + H
        o = SsOpts(T=T, N=N, r=r, p=p, H=H, batch=B, mem=MEM_HOST)
        bufs = dict(X=to_cm(X), Lam=to_cm(Lam), R=np.ascontiguousarray(R, dtype=float), A=to_cm(A), Q=to_cm(Q),
                    P0=to_cm(P0) if P0 is not None else None)
        ini = EmInit(Lam=_ptr(bufs["Lam"]), R=_ptr(bufs["R"]), A=_ptr(bufs["A"]), Q=_ptr(bufs["Q"]), P0=_ptr(bufs["P0"]))
        size = dict(F=Tp * r, PF=Tp * r * r, common=Tp * N, xhat=Tp * N, xvar=Tp * N)
        outs = {n: np.empty(B * size[n]) for n in outputs}
        oll = np.empty(B); ost = np.empty(B, dtype=np.int32)
        ou = SsOut(loglik=_ptr(oll), status=_ptr(ost), **{n: _ptr(a_) for n, a_ in outs.items()})
        self.check(self.lib.dfm_kalman_smooth(self.h, _ptr(bufs["X"]), C.byref(o), C.byref(ini), C.byref(ou)), "dfm_kalman_smooth")
        res = dict(loglik=oll if b else float(oll[0]), status=ost if b else int(ost[0]))
        for n, a_ in outs.items():
            if n == "PF":
                pf = a_.reshape(B, Tp, r, r)
                res[n] = pf if b else pf[0]
            else:
                res[n] = from_cm(a_, Tp, r if n == "F" else N, b)
        return res

    def simulation_smoother(self, X, Lam, R, A, Q, p=1, P0=None, H=0, n_draw=1, seed=0, draw0=0, outputs=("F", "X")):
        """Draws draw0 .. draw0 + n_draw - 1 from the joint posterior of the factor path and the missing cells at FIXED
        parameters (dfm_simulation_smoother).  X (T, N) standardized with NaN, one model; parameters as kalman_smooth.  Returns
        F (n_draw, T+H, r) and X (n_draw, T+H, N) -- those named in `outputs` -- and status."""
        X = np.asarray(X, float); T, N = X.shape; r = np.asarray(Lam).shape[-1]; Tp = T + H
        bufs = dict(X=to_cm(X), Lam=to_cm(Lam), R=np.ascontiguousarray(R, dtype=float), A=to_cm(A), Q=to_cm(Q),
                    P0=to_cm(P0) if P0 is not None else None)
        size = dict(F=Tp * r, X=Tp * N)
        outs = {n: np.empty(n_draw * size[n]) for n in outputs}
        ost = np.empty(1, dtype=np.int32)
        self.simulation_smoother_raw(bufs["X"].ctypes.data, T, N, r, p, H, n_draw, draw0, seed,
                                     {n: (bufs[n].ctypes.data if bufs[n] is not None else 0) for n in ("Lam", "R", "A", "Q", "P0")},
                                     {**{n: a_.ctypes.data for n, a_ in outs.items()}, "status": ost.ctypes.data}, MEM_HOST)
        res = dict(status=int(ost[0]))
        for n, a_ in outs.items():
            res[n] = from_cm(a_, Tp, r if n == "F" else N, n_draw)
        return res

    def news(self, X_old, X_new, Lam, R, A, Q, p=1, P0=None, H=0, targets=(), news_rows=1, outputs=NEWS_OUTPUTS):
        """News decomposition of the revision of each target between two vintages at FIXED parameters (dfm_news).  X_old,
        X_new (T, N) or (B, T, N) standardized with NaN, the new vintage only adding cells in the last `news_rows` rows;
        parameters as kalman_smooth; targets: (series, period) pairs, 0-based, period < T + H.  Returns old_est, new_est
        (n_target), news (news_rows, N), weight / contrib (news_rows, N, n_target) -- those named in `outputs` -- and status
        (per pair for batched input)."""
        X_old = np.asarray(X_old, float); b = X_old.shape[0] if X_old.ndim == 3 else None
        T, N = X_old.shape[-2:]; r = np.asarray(Lam).shape[-1]; B = b or 1; nq = len(targets)
        bufs = dict(Xo=to_cm(X_old), Xn=to_cm(X_new), Lam=to_cm(Lam), R=np.ascontiguousarray(R, dtype=float), A=to_cm(A), Q=to_cm(Q),
                    P0=to_cm(P0) if P0 is not None else None)
        size = dict(old_est=nq, new_est=nq, news=news_rows * N, weight=news_rows * N * nq, contrib=news_rows * N * nq)
        outs = {n: np.empty(B * size[n]) for n in outputs}
        ost = np.empty(B, dtype=np.int32)
        self.news_raw(bufs["Xo"].ctypes.data, bufs["Xn"].ctypes.data, T, N, r, p, H, B, news_rows, list(targets),
                      {n: (bufs[n].ctypes.data if bufs[n] is not None else 0) for n in ("Lam", "R", "A", "Q", "P0")},
                      {**{n: a_.ctypes.data for n, a_ in outs.items()}, "status": ost.ctypes.data}, MEM_HOST)
        res = dict(status=ost if b else int(ost[0]))
        for n, a_ in outs.items():
            if n in ("old_est", "new_est"):
                v = a_.reshape(B, nq)
            elif n == "news":
                v = a_.reshape(B, N, news_rows).transpose(0, 2, 1)
            else:
                v = a_.reshape(B, nq, N, news_rows).transpose(0, 3, 2, 1)
            res[n] = np.ascontiguousarray(v if b else v[0])
        return res
