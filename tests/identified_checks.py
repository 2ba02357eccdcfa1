"""Parity checks of dfm_gibbs_constrained and dfm_series_responses against the NumPy spec tests/identified_oracle.py.  Each
function takes a `Library` (CUDA on an H100, or the host-emulation build of the same kernel source)."""
import numpy as np

from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
import gibbs_checks as GC
import identified_oracle as IO

SEED = GC.SEED
PRIOR = GC.PRIOR


def constr_for(th):
    """Restrictions on GC.model()'s r = 3 model: series 0 fully pinned (m = r), series 2 one row, series 5 two rows, and a row on
    the excluded series 4 (ignored)."""
    idx = np.array([0, 0, 0, 2, 4, 5, 5], np.int32)
    H = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, -1, 0.5], [1, 0, 0], [0, 1, 0], [0.5, 0, 1]], float)
    h = np.array([0.7, 0.0, 0.0, 0.2, 0.5, 0.1, -0.3])
    assert np.isnan(th["Lam"][4]).all()
    return idx, H, h


def _no_rows(r):
    return np.zeros(0, np.int32), np.zeros((0, r)), np.zeros(0)


def check_chains(lib, X, th, p, constr, n_chain=2, n_burn=2, n_keep=3, thin=1, H_fc=2, fc_rows=4, chain0=3, sweep0=5, tol=1e-8):
    """Every kept draw, the loglik trace and the panel draws against the spec chain; every kept restricted draw on its rows."""
    ini = GC._inits(th, n_chain)
    got = lib.gibbs(X, ini, p=p, n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin, seed=SEED,
                    H_fc=H_fc, fc_rows=fc_rows, prior=PRIOR, constr=constr, outputs=("Lam", "R", "A", "Q", "F", "X"))
    for c in range(n_chain):
        ref = IO.chain(X, GC._chain_init(ini, c), p, PRIOR, SEED, chain0 + c, sweep0, n_burn, n_keep, thin, H=H_fc, constr=constr)
        GC.compare_chain(got, c, ref, tol)
    use = ~np.isnan(th["R"]) & ~np.isnan(th["Lam"]).any(1)
    for i in sorted(set(int(v) for v in constr[0])):
        if not use[i]:
            assert np.isnan(got["Lam"][:, :, i]).all()
            continue
        Hi, hi = IO.rows_of(constr, i)
        res = np.einsum("qa,cja->cjq", Hi, got["Lam"][:, :, i]) - hi
        assert np.max(np.abs(res)) <= 1e-12 * max(np.abs(hi).max(), 1.0), (i, np.max(np.abs(res)))
    return got


def check_no_rows_is_gibbs(lib, X, th, p):
    """n_constr = 0 gives dfm_gibbs' bits, impulse responses included."""
    r = th["Lam"].shape[1]
    kw = dict(p=p, n_chain=3, chain0=1, sweep0=2, n_burn=1, n_keep=2, seed=SEED, H_fc=2, fc_rows=3, H_irf=4, prior=PRIOR, ref=th)
    ini = GC._inits(th, 3)
    a = lib.gibbs(X, ini, **kw)
    b = lib.gibbs(X, ini, constr=_no_rows(r), **kw)
    for n in a:
        np.testing.assert_array_equal(a[n], b[n], err_msg=n)


def check_unrestricted_series(lib, X, th, p, constr):
    """After one sweep from the same theta, the unrestricted series, A and Q of a restricted call are dfm_gibbs' bits."""
    ini = GC._inits(th, 2)
    kw = dict(p=p, n_chain=2, chain0=4, sweep0=9, n_burn=0, n_keep=1, seed=SEED, H_fc=1, fc_rows=2, prior=PRIOR,
              outputs=("Lam", "R", "A", "Q", "F", "X"))
    a = lib.gibbs(X, ini, **kw)
    b = lib.gibbs(X, ini, constr=constr, **kw)
    free = np.setdiff1d(np.arange(X.shape[1]), constr[0])
    np.testing.assert_array_equal(a["Lam"][:, :, free], b["Lam"][:, :, free])
    np.testing.assert_array_equal(a["R"][:, :, free], b["R"][:, :, free])
    for n in ("A", "Q", "F", "X", "loglik"):
        np.testing.assert_array_equal(a[n], b[n], err_msg=n)
    assert not np.array_equal(a["Lam"][:, :, 0], b["Lam"][:, :, 0])


def check_chain_split(lib, X, th, p, constr, n_big=300):
    """Calls of different n_chain and chain0 give the same bits for the same chain ids (n_big spans two sub-batches)."""
    base = GC._inits(th, n_big)
    kw = dict(p=p, sweep0=2, n_burn=1, n_keep=1, seed=SEED, H_fc=1, fc_rows=2, prior=PRIOR, constr=constr, outputs=("Lam", "R", "Q"))
    sub = lambda c0, n: {m: base[m][c0:c0 + n] for m in base}
    big = lib.gibbs(X, sub(0, n_big), n_chain=n_big, chain0=0, **kw)
    head = lib.gibbs(X, sub(0, 20), n_chain=20, chain0=0, **kw)
    tail = lib.gibbs(X, sub(250, n_big - 250), n_chain=n_big - 250, chain0=250, **kw)
    for m in big:
        np.testing.assert_array_equal(head[m], big[m][:20], err_msg=m)
        np.testing.assert_array_equal(tail[m], big[m][250:], err_msg=m)


def check_args(lib, X, th, p, constr):
    r = th["Lam"].shape[1]
    idx, H, h = constr

    def code(c, **kw):
        try:
            args = dict(p=p, n_chain=2, n_keep=1, prior=PRIOR, seed=SEED, constr=c, outputs=("Lam", "R")); args.update(kw)
            return int(lib.gibbs(X, th, **args)["status"].max())
        except DFMError as e:
            return -e.code

    N = X.shape[1]
    assert code((np.array([N], np.int32), H[:1], h[:1])) == -1                  # index outside [0, N)
    assert code((np.array([-1], np.int32), H[:1], h[:1])) == -1
    assert code((idx, np.where(np.arange(H.size).reshape(H.shape) == 4, np.nan, H), h)) == -1
    assert code((idx, H, np.where(np.arange(len(h)) == 3, np.inf, h))) == -1
    assert code((np.zeros(r + 1, np.int32), np.ones((r + 1, r)), np.ones(r + 1))) == -1   # more than r rows on one series
    assert code((idx, None, h)) == -1
    assert code(constr, H_irf=3, ref=th, outputs=("Lam", "irf")) == -1             # no impulse responses with rows
    assert code((np.array([2, 2], np.int32), np.array([[1.0, 0, 0], [2.0, 0, 0]]), np.array([0.1, 0.2]))) == 3   # dependent rows
    assert code(constr) == 0                                                      # the handle stays usable


def models(th, p, B=5):
    """B models around th: model 1 a NaN A and Q (a failed chain), model 3 a Q that is not positive definite."""
    rng = np.random.default_rng(5)
    r = th["Q"].shape[0]
    Lam = np.stack([th["Lam"] * (1 + 0.1 * b) for b in range(B)])
    R = np.stack([th["R"] * (1 + 0.05 * b) for b in range(B)])
    A = np.stack([th["A"] * (1 - 0.05 * b) for b in range(B)])
    Q = np.stack([th["Q"] + 0.01 * b * np.eye(r) for b in range(B)])
    A[1] = np.nan; Q[1] = np.nan
    Q[3] = np.diag(np.r_[1.0, -0.5, np.ones(r - 2)])
    Lam[2, 6] = np.nan                                                            # one more series out of model 2
    scale = 0.5 + rng.random(th["Lam"].shape[0])
    return Lam, R, A, Q, scale


def check_series_responses(lib, th, p, alloc, H=7):
    """dfm_series_responses against the spec (1e-12) for n_shock = 1, 2, r, with host and device memory (device bits = host)."""
    Lam, R, A, Q, scale = models(th, p)
    B, N, r = Lam.shape
    for ns in (1, 2, r):
        got = lib.series_responses(Lam, R, A, Q, H, n_shock=ns, scale=scale)
        assert list(got["status"]) == [0, 3, 0, 3, 0]
        for b in range(B):
            rr, rf, st = IO.responses(Lam[b], R[b], A[b], Q[b], p, H, ns, scale)
            assert st == got["status"][b]
            for g, e in ((got["resp"][b], rr), (got["fevd"][b], rf)):
                assert (np.isnan(g) == np.isnan(e)).all(), b
                if st == 0:
                    assert np.nanmax(np.abs(g - e)) <= 1e-12 * max(1.0, np.nanmax(np.abs(e))), (b, np.nanmax(np.abs(g - e)))
        assert np.isnan(got["resp"][1]).all() and np.isnan(got["fevd"][3]).all()
        assert np.isnan(got["resp"][:, 4]).all() and np.isnan(got["fevd"][2, 6]).all()
        ins = {n: alloc(a_) for n, a_ in dict(Lam=to_cm(Lam), R=np.ascontiguousarray(R), A=to_cm(A), Q=to_cm(Q)).items()}
        sc = alloc(np.ascontiguousarray(scale))
        o = {n: alloc(np.zeros(B * N * H * ns)) for n in ("resp", "fevd")}
        st = alloc(np.zeros(B, np.int32))
        lib.series_responses_raw({n: ins[n][0] for n in ins}, N, r, p, B, H, ns, sc[0], MEM_DEVICE, resp=o["resp"][0],
                                 fevd=o["fevd"][0], status=st[0])
        lib.sync()
        for n in ("resp", "fevd"):
            np.testing.assert_array_equal(o[n][1]().reshape(B, ns, H, N).transpose(0, 3, 2, 1), got[n], err_msg=n)
        np.testing.assert_array_equal(st[1](), got["status"])
    one = lib.series_responses(Lam[0], R[0], A[0], Q[0], H, outputs=("fevd",))
    inm = ~np.isnan(one["fevd"][:, 0, 0])
    tot = one["fevd"].sum(2) + IO.idiosyncratic_share(Lam[0], R[0], A[0], Q[0], p, H)
    np.testing.assert_allclose(tot[inm], 1.0, rtol=0, atol=1e-13)
    try:
        lib.series_responses(Lam, R, A, Q, H, n_shock=r + 1)
    except DFMError as e:
        assert e.code == 1
    else:
        raise AssertionError("n_shock > r accepted")
