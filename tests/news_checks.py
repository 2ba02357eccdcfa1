"""Parity checks of dfm_news against the NumPy spec tests/news_oracle.py.  Each function takes a `Library` (CUDA on an H100,
or the host-emulation build of the same kernel source).  Bars: old / new estimates, news, weights and contributions to
1e-9 (standardized units); the identity sum_j w_j I_j = new - old to 1e-12 relative to the news."""
import numpy as np

from oracle.dgp import simulate_panel
from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, to_cm
from forecast_checks import _params, block_missing_panel
from news_oracle import news as news_spec

TOL = 1e-9


def compare(got, ref, tol=TOL):
    for n in ("old_est", "new_est", "news", "weight", "contrib"):
        g, e = got[n], ref[{"old_est": "old", "new_est": "new"}.get(n, n)]
        assert (np.isnan(g) == np.isnan(e)).all(), n
        ok = ~np.isnan(e)
        assert np.max(np.abs(g[ok] - e[ok]), initial=0.0) <= tol * max(1.0, np.max(np.abs(e[ok]), initial=0.0)), \
            (n, np.max(np.abs(g[ok] - e[ok]), initial=0.0))
    c = np.nan_to_num(got["contrib"]).sum((0, 1))
    fin = ~np.isnan(got["new_est"])
    np.testing.assert_allclose((got["new_est"] - got["old_est"])[fin], c[fin], rtol=0,
                               atol=1e-12 * max(1.0, np.nanmax(np.abs(got["news"]), initial=0.0)) * got["news"].size)


def vintages(N=24, r=3, T=70, p=1, miss=0.0, rep=9, exclude=(), holes=(), release=0.3, news_rows=2, seed=5):
    """A standardized panel (the new vintage) and PCA-started parameters; the old vintage hides a share `release` of the
    series in each of the last news_rows rows."""
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    for t0, t1, i in holes:
        X[t0:t1, i] = np.nan
    Lam, Rv, A, Q = _params(X, r, p)
    for i in exclude:
        Lam[i] = np.nan
    rng = np.random.default_rng(seed)
    Xo = X.copy()
    for t in range(T - news_rows, T):
        hide = rng.random(N) < release
        Xo[t, hide] = np.nan
    return Xo, X, Lam, Rv, A, Q


def default_targets(N, T, H):
    return [(0, T - 1), (N - 1, T - 2), (1, T - 5)] + [(2, T + h) for h in range(H)]


def check_news(lib, N=24, r=3, T=70, p=1, miss=0.0, H=0, rep=9, exclude=(), holes=(), news_rows=2, targets=None, release=0.3):
    Xo, Xn, Lam, Rv, A, Q = vintages(N, r, T, p, miss, rep, exclude, holes, release, news_rows)
    targets = default_targets(N, T, H) if targets is None else targets
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=p, H=H, targets=targets, news_rows=news_rows)
    assert got["status"] == 0
    ref = news_spec(Xo, Xn, Lam, Rv, A, Q, None, p, H, targets, news_rows)
    compare(got, ref)
    return (Xo, Xn, Lam, Rv, A, Q), got


def check_block_missing(lib, H):
    """Block-missing series and a ragged edge (forecast_checks.block_missing_panel), p = 2, released in the last 3 rows."""
    X = block_missing_panel()
    T, N = X.shape
    Lam, Rv, A, Q = _params(X, 2, 2)
    Xo = X.copy(); Xo[T - 3:, ::3] = np.nan; Xo[T - 1, 1::3] = np.nan
    targets = [(0, T - 1), (4, T - 2)] + [(1, T + h) for h in range(H)]
    got = lib.news(Xo, X, Lam, Rv, A, Q, p=2, H=H, targets=targets, news_rows=3)
    assert got["status"] == 0
    compare(got, news_spec(Xo, X, Lam, Rv, A, Q, None, 2, H, targets, 3))


def check_special_targets(lib):
    """A released target (weight 1 on its own cell), a target observed in the old vintage (revision 0), a target out of the
    model (NaN), and a forecast target."""
    Xo, Xn, Lam, Rv, A, Q = vintages(N=20, r=2, T=50, p=2, exclude=(5,), release=0.0)
    T = Xo.shape[0]
    Xo[T - 1, [3, 5, 7]] = np.nan
    targets = [(3, T - 1), (4, T - 1), (5, T - 1), (6, T + 1)]
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=2, H=2, targets=targets, news_rows=1)
    assert got["status"] == 0
    compare(got, news_spec(Xo, Xn, Lam, Rv, A, Q, None, 2, 2, targets, 1))
    assert got["weight"][0, 3, 0] == 1.0 and np.count_nonzero(got["weight"][:, :, 0]) == 1
    assert (got["weight"][:, :, 1] == 0.0).all() and got["new_est"][1] == got["old_est"][1] == Xo[T - 1, 4]
    assert np.isnan(got["old_est"][2]) and np.isnan(got["new_est"][2])
    assert np.isnan(got["news"][0, 5])                                           # a new cell out of the model is not news
    assert np.count_nonzero(got["weight"][:, :, 3]) == 2


def check_no_news(lib):
    Xo, _, Lam, Rv, A, Q = vintages(N=16, r=2, T=40, p=1, miss=0.1)
    T = Xo.shape[0]
    got = lib.news(Xo, Xo.copy(), Lam, Rv, A, Q, p=1, H=1, targets=[(0, T - 1), (3, T)], news_rows=2)
    assert got["status"] == 0
    assert np.isnan(got["news"]).all() and (got["weight"] == 0.0).all() and (got["contrib"] == 0.0).all()
    np.testing.assert_array_equal(got["new_est"], got["old_est"])


def _batch(B=5, N=20, r=2, T=48, p=2, H=2, news_rows=2):
    Xos, Xns, Ls, Rs, As, Qs = [], [], [], [], [], []
    for j in range(B):
        Xo, Xn, Lam, Rv, A, Q = vintages(N, r, T, p, 0.05, rep=30 + j, news_rows=news_rows, seed=j)
        Xos.append(Xo); Xns.append(Xn); Ls.append(Lam); Rs.append(Rv); As.append(A); Qs.append(Q)
    return [np.stack(v) for v in (Xos, Xns, Ls, Rs, As, Qs)]


def check_batch_equals_single(lib):
    Xo, Xn, Lam, Rv, A, Q = _batch()
    T, N = Xo.shape[1:]
    tg = default_targets(N, T, 2)
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=2, H=2, targets=tg, news_rows=2)
    assert (got["status"] == 0).all()
    for j in range(Xo.shape[0]):
        one = lib.news(Xo[j], Xn[j], Lam[j], Rv[j], A[j], Q[j], p=2, H=2, targets=tg, news_rows=2)
        ref = news_spec(Xo[j], Xn[j], Lam[j], Rv[j], A[j], Q[j], None, 2, 2, tg, 2)
        compare({n: got[n][j] for n in ("old_est", "new_est", "news", "weight", "contrib")}, ref)
        for n in ("old_est", "new_est", "news", "weight", "contrib"):
            np.testing.assert_allclose(one[n], got[n][j], rtol=1e-10, atol=1e-12, err_msg=n)


def check_inconsistent_pair(lib):
    """One pair of a batch with an old cell changed, one with a new cell above the window: DFM_ERR_ARG and NaN for those
    pairs, the other pairs bitwise unchanged."""
    Xo, Xn, Lam, Rv, A, Q = _batch()
    T, N = Xo.shape[1:]
    tg = default_targets(N, T, 2)
    good = lib.news(Xo, Xn, Lam, Rv, A, Q, p=2, H=2, targets=tg, news_rows=2)
    Xn2 = Xn.copy(); Xo2 = Xo.copy()
    Xn2[1, 3, 0] += 0.5                                                          # an old cell changed
    Xo2[3, T - 5, 2] = np.nan                                                    # a new cell above the window
    bad = lib.news(Xo2, Xn2, Lam, Rv, A, Q, p=2, H=2, targets=tg, news_rows=2)
    assert list(bad["status"]) == [0, 1, 0, 1, 0]
    for j in (1, 3):
        for n in ("old_est", "new_est", "news", "weight", "contrib"):
            assert np.isnan(bad[n][j]).all(), n
    for j in (0, 2, 4):
        for n in ("old_est", "new_est", "news", "weight", "contrib"):
            np.testing.assert_array_equal(bad[n][j], good[n][j])


def check_mem_device(lib, alloc):
    """mem = DEVICE gives what mem = HOST gives (and finds a new cell above the window on the device).  alloc(array) ->
    (address, to_numpy()) of a device buffer."""
    Xo, Xn, Lam, Rv, A, Q = _batch(B=3)
    B, T, N = Xo.shape; r = Lam.shape[2]; nr, H = 2, 2
    tg = default_targets(N, T, H); nq = len(tg)
    Xo[2, 10, 4] = np.nan                                                        # pair 2: a new cell above the window
    host = lib.news(Xo, Xn, Lam, Rv, A, Q, p=2, H=H, targets=tg, news_rows=nr)
    assert list(host["status"]) == [0, 0, 1]
    ins = {n: alloc(a_) for n, a_ in dict(Xo=to_cm(Xo), Xn=to_cm(Xn), Lam=to_cm(Lam), R=np.ascontiguousarray(Rv), A=to_cm(A),
                                          Q=to_cm(Q)).items()}
    size = dict(old_est=nq, new_est=nq, news=nr * N, weight=nr * N * nq, contrib=nr * N * nq)
    outs = {n: alloc(np.zeros(B * s)) for n, s in size.items()}
    st = alloc(np.full(B, -1, np.int32))
    lib.news_raw(ins["Xo"][0], ins["Xn"][0], T, N, r, 2, H, B, nr, tg, {n: ins[n][0] for n in ("Lam", "R", "A", "Q")},
                 {**{n: v[0] for n, v in outs.items()}, "status": st[0]}, MEM_DEVICE)
    lib.sync()
    assert list(st[1]()) == [0, 0, 1]
    np.testing.assert_array_equal(outs["old_est"][1]().reshape(B, nq), host["old_est"])
    np.testing.assert_array_equal(outs["new_est"][1]().reshape(B, nq), host["new_est"])
    np.testing.assert_array_equal(outs["news"][1]().reshape(B, N, nr).transpose(0, 2, 1), host["news"])
    for n in ("weight", "contrib"):
        np.testing.assert_array_equal(outs[n][1]().reshape(B, nq, N, nr).transpose(0, 3, 2, 1), host[n])


def check_largest_w(lib):
    """W r = 128 (64 periods at r = 2): the W r-sized matrices of k_news_cov live in global scratch."""
    Xo, Xn, Lam, Rv, A, Q = vintages(N=12, r=2, T=30, miss=0.05)
    N = Xo.shape[1]
    tg = [(t % N, t) for t in range(0, 28)] + [(t % N, t) for t in range(30, 64)]
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=1, H=34, targets=tg, news_rows=2)
    assert got["status"] == 0
    compare(got, news_spec(Xo, Xn, Lam, Rv, A, Q, None, 1, 34, tg, 2))


def check_failed_estep(lib):
    """R_i <= 0 fails the E-step: status 3 and NaN outputs."""
    Xo, Xn, Lam, Rv, A, Q = vintages(N=12, r=2, T=30)
    Rv = Rv.copy(); Rv[4] = -1.0
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=1, H=1, targets=[(0, 29)], news_rows=2)
    assert got["status"] == 3
    for n in ("old_est", "new_est", "news", "weight", "contrib"):
        assert np.isnan(got[n]).all(), n


def check_args(lib):
    Xo, Xn, Lam, Rv, A, Q = vintages(N=12, r=2, T=30)
    T, N, r = 30, 12, 2

    def code(**kw):
        args = dict(p=1, H=0, targets=[(0, T - 1)], news_rows=2); args.update(kw)
        X0 = args.pop("Xo", Xo); X1 = args.pop("Xn", Xn); Lm = args.pop("Lam", Lam); A_ = args.pop("A", A); Q_ = args.pop("Q", Q)
        try:
            lib.news(X0, X1, Lm, Rv, A_, Q_, **args)
        except DFMError as e:
            return e.code
        return 0

    assert code() == 0
    assert code(targets=[]) == 1                                                 # n_target = 0
    assert code(targets=[(0, T)]) == 1                                           # period >= T + H
    assert code(targets=[(0, T)], H=1) == 0
    assert code(targets=[(N, T - 1)]) == 1                                       # series >= N
    assert code(targets=[(-1, T - 1)]) == 1
    assert code(news_rows=0) == 1
    assert code(news_rows=T + 1) == 1
    assert code(targets=[(0, t) for t in range(0, 65)]) == 1                     # n_target > 64
    edge = [(t % N, t) for t in range(0, 28)] + [(t % N, t) for t in range(30, 64)]      # 62 periods outside the window
    assert code(targets=edge, H=34) == 0                                         # W r = (62 + 2) 2 = 128
    assert code(targets=edge + [(0, 64)], H=35) == 6                             # W r = 130
    assert code(targets=[(0, t) for t in range(30, 70)], H=40, news_rows=T) == 6  # W r = (30 + 40) 2
    assert code(H=-1) == 1
    assert code(p=25, A=np.zeros((2, 50))) == 6                                  # k = 50 > 48
    B = 65536
    bufs = dict(Xo=to_cm(Xo), Xn=to_cm(Xn), Lam=to_cm(Lam), R=np.ascontiguousarray(Rv), A=to_cm(A), Q=to_cm(Q))
    try:
        lib.news_raw(bufs["Xo"].ctypes.data, bufs["Xn"].ctypes.data, T, N, r, 1, 0, B, 2, [(0, T - 1)],
                     {n: bufs[n].ctypes.data for n in ("Lam", "R", "A", "Q")}, {}, MEM_HOST)
        raise AssertionError("batch > 65535 accepted")
    except DFMError as e:
        assert e.code == 6
    for missing in bufs:
        addr = {n: (0 if n == missing else bufs[n].ctypes.data) for n in bufs}
        try:
            lib.news_raw(addr["Xo"], addr["Xn"], T, N, r, 1, 0, 1, 2, [(0, T - 1)], {n: addr[n] for n in ("Lam", "R", "A", "Q")}, {},
                         MEM_HOST)
            raise AssertionError("null %s accepted" % missing)
        except DFMError as e:
            assert e.code == 1
