"""Output staging of the single-call entry points: the device-memory path against the host path, outputs left out, and a call in
a workspace that an earlier, larger call grew and used.  Run by tests/test_emu_staging.py on the host-emulation build and by
tests/test_gpu_staging.py on the H100.

A case builds one call from a shape: its inputs (uploaded for device memory), its outputs (zero buffers of the caller's memory),
the optional outputs, outputs the library always writes to host memory, and the call itself.  alloc(a) -> (address, to_numpy)
places a copy of the array `a` in device memory (numpy buffers on the emulation build, torch CUDA tensors on the GPU)."""
import ctypes as C

import numpy as np

from dynamic_factor_models_b200._lib import (BootOpts, EmInit, FactorOpts, GibbsOpts, GibbsOut, GibbsPrior, LoadingOpts, MEM_DEVICE,
                                             MEM_HOST, SsbOpts, SsbOut, gibbs_default_prior)


class Case:
    """ins: name -> input array; outs: name -> zero output array; optional: outputs that may be NULL; host_outs: outputs the
    library writes to host memory whatever mem (zero arrays); call(lib, mem, ptr) -> status, where ptr(name) is the address of
    an input or output (None for an output left out)."""

    def __init__(self, ins, outs, call, optional=(), host_outs=None):
        self.ins, self.outs, self.call, self.optional, self.host_outs = ins, outs, call, tuple(optional), host_outs or {}


def _rng(seed):
    return np.random.default_rng(seed)


def run(lib, case, mem, alloc, drop=()):
    """One call of `case` with inputs and outputs in `mem`; the outputs not in `drop` (and the host outputs) as numpy arrays."""
    assert not set(case.ins) & (set(case.outs) | set(case.host_outs)), "an input and an output share a name"
    keep, bufs = [], {}

    def host(a):
        b = np.array(a, copy=True)
        keep.append(b)
        return b.ctypes.data, (lambda: b.copy())

    for n, a in case.ins.items():
        bufs[n] = (alloc if mem == MEM_DEVICE else host)(a)
    for n, a in case.outs.items():
        if n not in drop:
            bufs[n] = (alloc if mem == MEM_DEVICE else host)(a)
    for n, a in case.host_outs.items():
        bufs[n] = host(a)

    def ptr(n):
        return C.c_void_p(bufs[n][0]) if n in bufs else None

    lib.check(case.call(lib, mem, ptr), "staging case")
    lib.sync()
    res = {n: bufs[n][1]() for n in list(case.outs) + list(case.host_outs) if n in bufs}
    del keep
    return res


def assert_same_bits(a, b, what=""):
    assert set(a) == set(b), (what, sorted(a), sorted(b))
    for n in a:
        assert a[n].dtype == b[n].dtype and a[n].shape == b[n].shape, (what, n)
        assert a[n].tobytes() == b[n].tobytes(), f"{what}: output {n} differs"


def _subset(res, names):
    return {n: v for n, v in res.items() if n in names}


def check_device_equals_host(lib, make, alloc):
    """mem = DEVICE gives, bit for bit, what mem = HOST gives, with every output asked for."""
    case = make("big")
    host = run(lib, case, MEM_HOST, alloc)
    dev = run(lib, case, MEM_DEVICE, alloc)
    assert_same_bits(dev, host, "device vs host")


def check_optional_outputs(lib, make, alloc):
    """Leaving out the optional outputs (all of them, then each one alone) does not change the outputs that were asked for, in
    either memory."""
    case = make("big")
    for mem in (MEM_HOST, MEM_DEVICE):
        full = run(lib, case, mem, alloc)
        drops = [tuple(case.optional)] + [(n,) for n in case.optional] if case.optional else []
        for drop in drops:
            part = run(lib, case, mem, alloc, drop=drop)
            assert_same_bits(part, _subset(full, part), f"mem {mem} without {drop}")


def check_grown_workspace(lib, new_lib, make, alloc):
    """A smaller call on a handle whose workspace a larger call grew and used gives the bits of that call on a fresh handle."""
    big, small = make("big"), make("small")
    for mem in (MEM_HOST, MEM_DEVICE):
        run(lib, big, mem, alloc)
        used = run(lib, small, mem, alloc)
        fresh_lib = new_lib()
        try:
            fresh = run(fresh_lib, small, mem, alloc)
        finally:
            fresh_lib.close()
        assert_same_bits(used, fresh, f"mem {mem}: grown workspace vs fresh handle")


# ---------------------------------------------------------------------------------------------------------- cases
def _panel(B, T, N, seed, miss=0.0):
    """B column-major T x N panels (B * N * T doubles) with a fraction `miss` of NaN."""
    x = _rng(seed).standard_normal(B * N * T)
    if miss:
        x[_rng(seed + 1).random(x.size) < miss] = np.nan
    return x


def standardize(size):
    B, T, N = (3, 40, 14) if size == "big" else (2, 30, 10)
    return Case(dict(X=_panel(B, T, N, 1, 0.05)), dict(Xs=np.zeros(B * T * N), xmean=np.zeros(B * N), xstd=np.zeros(B * N)),
                lambda lib, mem, p: lib.lib.dfm_standardize(lib.h, p("X"), T, N, B, mem, p("Xs"), p("xmean"), p("xstd")),
                optional=("xmean", "xstd"))


def pca_score(size):
    B, T, N, r = (3, 40, 14, 3) if size == "big" else (2, 30, 10, 2)
    return Case(dict(X=_panel(B, T, N, 2)), dict(score=np.zeros(B * T * r)),
                lambda lib, mem, p: lib.lib.dfm_pca_score(lib.h, p("X"), T, N, r, B, mem, p("score")))


def estimate_factor(size):
    B, T, N, r = (3, 40, 14, 3) if size == "big" else (2, 30, 10, 2)

    def call(lib, mem, p):
        o = FactorOpts(T=T, N=N, r=r, nt_min=10, tol=1e-8, max_iter=200, compute_r2=1, batch=B, mem=mem)
        return lib.lib.dfm_estimate_factor(lib.h, p("X"), C.byref(o), None, p("F"), p("Lambda"), p("R2"), p("xmean"), p("xstd"), None)
    X = _panel(B, T, N, 3, 0.05)
    X.reshape(B, N, T)[:, :r + 1] = _rng(30).standard_normal((B, r + 1, T))      # the PCA start needs r fully observed series
    return Case(dict(X=X),
                dict(F=np.zeros(B * T * r), Lambda=np.zeros(B * N * r), R2=np.zeros(B * N), xmean=np.zeros(B * N), xstd=np.zeros(B * N)),
                call, optional=("Lambda", "R2", "xmean", "xstd"))


def estimate_loading_ex(size):
    B, T, ns, r, Lg = (3, 50, 9, 2, 2) if size == "big" else (2, 40, 6, 2, 2)

    def call(lib, mem, p):
        o = LoadingOpts(T=T, ns=ns, r=r, nt_min=20, n_uarlag=Lg, batch=B, mem=mem)
        return lib.lib.dfm_estimate_loading_ex(lib.h, p("data"), p("F"), C.byref(o), p("lambda"), p("r2"), p("uar_coef"), p("uar_ser"),
                                               p("constant"), p("resid"), p("status"))
    return Case(dict(data=_panel(B, T, ns, 4, 0.05), F=_panel(B, T, r, 5)),
                dict(**{"lambda": np.zeros(B * ns * r)}, r2=np.zeros(B * ns), uar_coef=np.zeros(B * ns * Lg), uar_ser=np.zeros(B * ns),
                     constant=np.zeros(B * ns), resid=np.zeros(B * ns * T)),
                call, optional=("constant", "resid"), host_outs=dict(status=np.zeros(B, np.int32)))


def estimate_var(size):
    B, T, r, p_ = (3, 60, 3, 2) if size == "big" else (2, 40, 2, 2)
    k, K = r * p_, r * p_ + 1

    def call(lib, mem, p):
        return lib.lib.dfm_estimate_var(lib.h, p("F"), T, r, p_, 1, B, mem, p("betahat"), p("resid"), p("seps"), p("M"), p("Q"), p("G"))
    return Case(dict(F=_panel(B, T, r, 6)),
                dict(betahat=np.zeros(B * K * r), resid=np.zeros(B * T * r), seps=np.zeros(B * r * r), M=np.zeros(B * k * k),
                     Q=np.zeros(B * r * k), G=np.zeros(B * k * r)),
                call, optional=("betahat", "resid", "seps", "Q", "G"))


def irf(size):
    B, r, p_, H = (3, 3, 2, 6) if size == "big" else (2, 2, 2, 4)
    k = r * p_
    ids = np.array([r - 1, 0], np.int32)
    g = _rng(7)

    def call(lib, mem, p):
        return lib.lib.dfm_irf(lib.h, p("M"), p("Q"), p("G"), k, r, H, len(ids), ids.ctypes.data_as(C.POINTER(C.c_int)), B, mem, p("irf"))
    return Case(dict(M=0.3 * g.standard_normal(B * k * k) / k, Q=g.standard_normal(B * r * k), G=g.standard_normal(B * k * r)),
                dict(irf=np.zeros(B * r * H * len(ids))), call)


def em_init_from_factors(size):
    B, T, N, r, p_ = (3, 40, 14, 3, 1) if size == "big" else (2, 30, 10, 2, 1)

    def call(lib, mem, p):
        return lib.lib.dfm_em_init_from_factors(lib.h, p("Xs"), p("F"), T, N, r, p_, B, mem, p("Lam"), p("R"), p("A"), p("Q"))
    return Case(dict(Xs=_panel(B, T, N, 8, 0.05), F=_panel(B, T, r, 9)),
                dict(Lam=np.zeros(B * N * r), R=np.zeros(B * N), A=np.zeros(B * r * r * p_), Q=np.zeros(B * r * r)),
                call, optional=("R", "A", "Q"))


def simulate_panels(size):
    B, T, N, r = (3, 30, 12, 3) if size == "big" else (2, 20, 8, 2)

    def call(lib, mem, p):
        return lib.lib.dfm_simulate_panels(lib.h, 11, 5, B, T, N, r, mem, p("X"), p("F_true"))
    return Case({}, dict(X=np.zeros(B * T * N), F_true=np.zeros(B * T * r)), call, optional=("F_true",))


def _boot_inputs(size, seed):
    Tw, ns, r, p_, Lg = (60, 12, 2, 1, 2) if size == "big" else (50, 10, 2, 1, 2)
    g = _rng(seed)
    nres, K = Tw - p_, 1 + r * p_
    ins = dict(F0=g.standard_normal(Tw * r), resid=g.standard_normal(nres * r), beta=0.2 * g.standard_normal(K * r),
               lam=g.standard_normal(ns * r), uar_coef=0.1 * g.standard_normal(ns * Lg), uar_ser=0.5 + g.random(ns),
               data=g.standard_normal(Tw * ns))
    return ins, Tw, ns, r, p_, Lg, nres


_BOOT_IN = ("F0", "resid", "beta", "lam", "uar_coef", "uar_ser", "data")


def bootstrap_panels(size):
    ins, Tw, ns, r, p_, Lg, nres = _boot_inputs(size, 10)
    B = 3 if size == "big" else 2

    def call(lib, mem, p):
        o = BootOpts(T=Tw, ns=ns, r=r, p=p_, n_uarlag=Lg, n_resid=nres, burn=10, batch=B, mem=mem, seed=3, rep0=7)
        return lib.lib.dfm_bootstrap_panels(lib.h, C.byref(o), *[p(n) for n in _BOOT_IN], p("X"))
    return Case(ins, dict(X=np.zeros(B * ns * Tw)), call)


def bootstrap_irf(size):
    ins, Tw, ns, r, p_, Lg, nres = _boot_inputs(size, 12)
    B, H = (3, 5) if size == "big" else (2, 4)

    def call(lib, mem, p):
        o = BootOpts(T=Tw, ns=ns, r=r, p=p_, n_uarlag=Lg, n_resid=nres, burn=10, batch=B, mem=mem, seed=4, rep0=2)
        return lib.lib.dfm_bootstrap_irf(lib.h, C.byref(o), *[p(n) for n in _BOOT_IN], 20, 1e-8, H, p("irf"), p("iters"), p("status"))
    return Case(ins, dict(irf=np.zeros(B * r * H * r)), call,
                host_outs=dict(iters=np.zeros(B, np.int32), status=np.zeros(B, np.int32)))


def _ss_model(N, r, seed):
    g = _rng(seed)
    return dict(Lam=g.standard_normal(N * r), R=0.5 + g.random(N), A=(0.5 * np.eye(r)).T.ravel(), Q=np.eye(r).ravel(),
                P0=(np.eye(r) / 0.75).ravel())


def ss_simulate_panels(size):
    B, T, N, r = (3, 30, 10, 2) if size == "big" else (2, 20, 8, 2)
    ins = dict(X=_panel(1, T, N, 13, 0.05), **_ss_model(N, r, 14))

    def call(lib, mem, p):
        ini = EmInit(**{n: p(n) for n in ("Lam", "R", "A", "Q", "P0")})
        return lib.lib.dfm_ss_simulate_panels(lib.h, p("X"), T, N, r, 1, C.byref(ini), 21, 3, B, mem, p("Xout"))
    return Case(ins, dict(Xout=np.zeros(B * T * N)), call)


def gibbs(size):
    nch, T, N, r = (3, 24, 8, 2) if size == "big" else (2, 20, 6, 2)
    nk, Hi, Hf, fr, n_burn = 2, 3, 2, 2, 1
    n_sweep, Tp = n_burn + nk, T + Hf
    m = _ss_model(N, r, 15)
    ins = dict(Xin=_panel(1, T, N, 16, 0.05), **{"init_" + n: np.tile(v, nch) for n, v in m.items()},
               **{"ref_" + n: m[n] for n in ("Lam", "R", "A", "Q")})
    outs = dict(Lam=np.zeros(nch * nk * N * r), R=np.zeros(nch * nk * N), A=np.zeros(nch * nk * r * r), Q=np.zeros(nch * nk * r * r),
                irf=np.zeros(nch * nk * r * Hi * r), F=np.zeros(nch * nk * Tp * r), X=np.zeros(nch * nk * fr * N),
                loglik=np.zeros(nch * n_sweep), status=np.zeros(nch, np.int32))

    def call(lib, mem, p):
        o = GibbsOpts(T=T, N=N, r=r, p=1, H_irf=Hi, H_fc=Hf, fc_rows=fr, n_chain=nch, chain0=1, sweep0=0, n_burn=n_burn, n_keep=nk,
                      thin=1, seed=9, mem=mem, prior=GibbsPrior(**gibbs_default_prior(r)))
        ini = EmInit(**{n: p("init_" + n) for n in ("Lam", "R", "A", "Q", "P0")})
        ref = EmInit(**{n: p("ref_" + n) for n in ("Lam", "R", "A", "Q")})
        ou = GibbsOut(**{n: p(n) for n in outs})
        return lib.lib.dfm_gibbs(lib.h, p("Xin"), C.byref(o), C.byref(ini), C.byref(ref), C.byref(ou))
    return Case(ins, outs, call, optional=("Lam", "irf", "F", "X", "loglik", "status"))


def ss_bootstrap(size):
    """big: one replicate more than a sub-batch (264 replicates of this shape on 132 SMs), so the records of the second
    sub-batch go out from row 264."""
    n_rep, T, N, r = (265, 16, 6, 2) if size == "big" else (5, 12, 5, 2)
    Hi, Hf, fr = 3, 2, 2
    ins = dict(in_X=_panel(1, T, N, 24, 0.05), **{"in_" + n: v for n, v in _ss_model(N, r, 25).items()})
    outs = dict(Lam=np.zeros(n_rep * N * r), R=np.zeros(n_rep * N), A=np.zeros(n_rep * r * r), Q=np.zeros(n_rep * r * r),
                irf=np.zeros(n_rep * r * Hi * r), xhat=np.zeros(n_rep * fr * N), xvar=np.zeros(n_rep * fr * N), loglik=np.zeros(n_rep),
                iters=np.zeros(n_rep, np.int32), status=np.zeros(n_rep, np.int32))

    def call(lib, mem, p):
        o = SsbOpts(T=T, N=N, r=r, p=1, H_irf=Hi, H_fc=Hf, fc_rows=fr, max_iter=2, tol=0.0, n_rep=n_rep, rep0=3, seed=5, mem=mem)
        ini = EmInit(**{n: p("in_" + n) for n in ("Lam", "R", "A", "Q", "P0")})
        ou = SsbOut(**{n: p(n) for n in outs})
        return lib.lib.dfm_ss_bootstrap(lib.h, p("in_X"), C.byref(o), C.byref(ini), C.byref(ou))
    return Case(ins, outs, call, optional=("irf", "xhat", "loglik"))


def instability(size):
    T, ns, r = (80, 6, 2) if size == "big" else (70, 4, 2)

    def call(lib, mem, p):
        return lib.lib.dfm_instability(lib.h, p("data"), p("F"), C.c_int(T), C.c_int(ns), C.c_int(r), C.c_int(2), C.c_int(T // 2),
                                       C.c_double(0.15), C.c_int(20), C.c_int(mem), p("chow"), p("qlr"), p("qlr0"), p("status"))
    return Case(dict(data=_panel(1, T, ns, 17, 0.03), F=_panel(1, T, r, 18)),
                dict(chow=np.zeros(ns), qlr=np.zeros(ns), qlr0=np.zeros(ns), status=np.zeros(ns, np.int32)),
                call, optional=("qlr0", "status"))


def fit_correlation(size):
    T, ns, r = (80, 6, 2) if size == "big" else (70, 4, 2)

    def call(lib, mem, p):
        return lib.lib.dfm_fit_correlation(lib.h, p("data"), p("F"), p("F_alt"), C.c_int(T), C.c_int(ns), C.c_int(r), C.c_int(T // 2),
                                           C.c_int(20), C.c_int(mem), p("cor"), p("status"))
    return Case(dict(data=_panel(1, T, ns, 19, 0.03), F=_panel(1, T, r, 20), F_alt=_panel(1, T, r, 21)),
                dict(cor=np.zeros(ns), status=np.zeros(ns, np.int32)), call, optional=("status",))


_Q = np.array([5.0, 50.0, 95.0])


def percentiles(size):
    n, d = (60, 7) if size == "big" else (40, 5)
    recs = _rng(22).standard_normal(n * d)
    recs[::13] = np.nan

    def call(lib, mem, p):
        return lib.lib.dfm_percentiles(lib.h, p("recs"), n, d, _Q.ctypes.data_as(C.c_void_p), len(_Q), mem, p("out"))
    return Case(dict(recs=recs), dict(out=np.zeros(len(_Q) * d)), call)


def percentiles_weighted(size):
    n, d = (60, 7) if size == "big" else (40, 5)
    g = _rng(23)

    def call(lib, mem, p):
        return lib.lib.dfm_percentiles_weighted(lib.h, p("recs"), p("w"), n, d, _Q.ctypes.data_as(C.c_void_p), len(_Q), mem, p("out"))
    return Case(dict(recs=g.standard_normal(n * d), w=g.random(n) + 0.1), dict(out=np.zeros(len(_Q) * d)), call)


CASES = dict(standardize=standardize, pca_score=pca_score, estimate_factor=estimate_factor, estimate_loading_ex=estimate_loading_ex,
             estimate_var=estimate_var, irf=irf, em_init_from_factors=em_init_from_factors, simulate_panels=simulate_panels,
             bootstrap_panels=bootstrap_panels, bootstrap_irf=bootstrap_irf, ss_simulate_panels=ss_simulate_panels, gibbs=gibbs,
             instability=instability, fit_correlation=fit_correlation, percentiles=percentiles,
             percentiles_weighted=percentiles_weighted, ss_bootstrap=ss_bootstrap)
