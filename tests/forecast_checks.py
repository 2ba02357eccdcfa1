"""Parity checks of dfm_kalman_smooth (smoothing / nowcasting / forecasting at fixed parameters) against the NumPy spec
tests/forecast_oracle.py.  Each function takes a `Library` (CUDA on an H100, or the host-emulation build of the same
kernel source).  Bars: F RMSE < 1e-8; PF, common, xhat, xvar to rtol 1e-7 / atol 1e-10; log-likelihood rtol 1e-10."""
import numpy as np

from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel
from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST
from forecast_oracle import smooth_forecast
from parity_checks import ll_atol, rmse


def _params(X, r, p):
    F0 = R.pca_score(np.nan_to_num(X), r)
    return K.init_from_factors(X, F0, p)


def compare(got, ref, ll_rtol=1e-10, ll_atol=0.0):
    assert rmse(got["F"], ref["F"]) < 1e-8, rmse(got["F"], ref["F"])
    np.testing.assert_allclose(got["PF"], ref["PF"], rtol=1e-7, atol=1e-10)
    for n in ("common", "xhat", "xvar"):
        assert (np.isnan(got[n]) == np.isnan(ref[n])).all(), n
        np.testing.assert_allclose(got[n], ref[n], rtol=1e-7, atol=1e-10, err_msg=n)
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=ll_rtol, atol=ll_atol)


def check_observed_cells(X, got):
    """xhat is the data bitwise where a cell is observed, and xvar is exactly 0 there; every other cell of a series in the
    model (the forecast rows included) has a finite value and a positive variance."""
    T = X.shape[0]
    inmodel = ~np.isnan(got["common"][0])
    obs = ~np.isnan(X) & inmodel[None, :]
    assert np.array_equal(got["xhat"][:T][obs], X[obs])
    assert (got["xvar"][:T][obs] == 0.0).all()
    unobs = np.vstack([~obs, np.ones((got["xhat"].shape[0] - T, X.shape[1]), bool)]) & inmodel[None, :]
    assert np.isfinite(got["xhat"][unobs]).all() and (got["xvar"][unobs] > 0.0).all()


def check_kalman_smooth(lib, N=24, r=3, T=70, p=1, miss=0.0, H=0, rep=9, exclude=(), holes=(), ll_cell_tol=0.0):
    """holes and ll_cell_tol as in parity_checks.check_em."""
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    for t0, t1, i in holes:
        X[t0:t1, i] = np.nan
    Lam, Rv, A, Q = _params(X, r, p)
    for i in exclude:
        Lam[i] = np.nan
    ref = smooth_forecast(X, Lam, Rv, A, Q, None, p, H)
    got = lib.kalman_smooth(X, Lam, Rv, A, Q, p=p, H=H)
    assert got["status"] == 0
    compare(got, ref, ll_atol=ll_atol(X, ll_cell_tol))
    check_observed_cells(X, got)
    for i in exclude:
        assert np.isnan(got["common"][:, i]).all() and np.isnan(got["xhat"][:, i]).all() and np.isnan(got["xvar"][:, i]).all()
    return X, (Lam, Rv, A, Q), got


def block_missing_panel():
    """The shapes of parity_checks.check_em_block_missing, plus a ragged edge: two series end early, one starts late."""
    X, _ = simulate_panel(20, 2, 260, rep=3)
    X[:60, 3] = np.nan; X[200:, 7] = np.nan; X[100:140, 11] = np.nan
    X[-3:, 5] = np.nan; X[-1:, 14] = np.nan
    return X


def check_kalman_smooth_block_missing(lib, H):
    X = block_missing_panel()
    Lam, Rv, A, Q = _params(X, 2, 2)
    ref = smooth_forecast(X, Lam, Rv, A, Q, None, 2, H)
    got = lib.kalman_smooth(X, Lam, Rv, A, Q, p=2, H=H)
    assert got["status"] == 0
    compare(got, ref)
    check_observed_cells(X, got)


def check_kalman_smooth_vs_em(lib, N=24, r=3, T=70, p=2, miss=0.1, H=4):
    """The log-likelihood is the one dfm_em_kalman reports for the parameters entering its first iteration, and the in-sample
    smoothed factors are that E-step's."""
    X, _ = simulate_panel(N, r, T, rep=4, missing_frac=miss)
    Lam, Rv, A, Q = _params(X, r, p)
    em = lib.em_kalman(X, Lam, Rv, A, Q, p=p, max_iter=1, path=1)
    for h_ in (0, H):
        got = lib.kalman_smooth(X, Lam, Rv, A, Q, p=p, H=h_)
        np.testing.assert_allclose(got["loglik"], em["loglik"][0], rtol=1e-12)
        np.testing.assert_allclose(got["F"][:T], em["F"], rtol=1e-10, atol=1e-10)


def check_kalman_smooth_batch(lib, N=16, r=2, T=40, p=2):
    """A batch with different missing patterns gives the results of one call per panel.  (All panels of one call share H;
    panels whose own data end early carry their own NaN tail inside T.)"""
    B, H = 3, 5
    Xb = np.stack([simulate_panel(N, r, T, rep=50 + b, missing_frac=0.08 * b)[0] for b in range(B)])
    Xb[1, -6:, :] = np.nan                              # panel 1: a longer all-missing tail
    Xb[2, -2:, 3:9] = np.nan                            # panel 2: a ragged edge
    ps = [_params(Xb[b], r, p) for b in range(B)]
    Lam, Rv, A, Q = (np.stack([q[j] for q in ps]) for j in range(4))
    got = lib.kalman_smooth(Xb, Lam, Rv, A, Q, p=p, H=H)
    assert (got["status"] == 0).all()
    for b in range(B):
        one = lib.kalman_smooth(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=p, H=H)
        for n in ("F", "PF", "common", "xhat", "xvar"):
            np.testing.assert_allclose(got[n][b], one[n], rtol=1e-12, atol=1e-14, err_msg=n)
        np.testing.assert_allclose(got["loglik"][b], one["loglik"], rtol=1e-13)
        ref = smooth_forecast(Xb[b], Lam[b], Rv[b], A[b], Q[b], None, p, H)
        compare({n: got[n][b] for n in ("F", "PF", "common", "xhat", "xvar")} | {"loglik": got["loglik"][b]}, ref)


def check_kalman_smooth_mem_device(lib, alloc, N=18, r=2, T=50, p=1, H=3, B=2):
    """mem = DEVICE gives what mem = HOST gives.  alloc(n_doubles) -> (address, to_numpy()) of a device buffer; the inputs
    are uploaded through the same allocator."""
    Xb = np.stack([simulate_panel(N, r, T, rep=70 + b, missing_frac=0.05)[0] for b in range(B)])
    ps = [_params(Xb[b], r, p) for b in range(B)]
    Lam, Rv, A, Q = (np.stack([q[j] for q in ps]) for j in range(4))
    host = lib.kalman_smooth(Xb, Lam, Rv, A, Q, p=p, H=H)
    from dynamic_factor_models_b200._lib import to_cm, from_cm
    ins = {n: alloc(a_) for n, a_ in dict(X=to_cm(Xb), Lam=to_cm(Lam), R=np.ascontiguousarray(Rv), A=to_cm(A), Q=to_cm(Q)).items()}
    Tp = T + H
    sizes = dict(F=B * Tp * r, PF=B * Tp * r * r, common=B * Tp * N, xhat=B * Tp * N, xvar=B * Tp * N, loglik=B)
    outs = {n: alloc(np.zeros(s)) for n, s in sizes.items()}
    st = alloc(np.zeros(B, np.int32))
    lib.kalman_smooth_raw(ins["X"][0], T, N, r, p, H, B, {n: ins[n][0] for n in ("Lam", "R", "A", "Q")},
                          {**{n: v[0] for n, v in outs.items()}, "status": st[0]}, MEM_DEVICE)
    lib.sync()
    assert (st[1]() == 0).all()
    dev = {n: v[1]() for n, v in outs.items()}
    np.testing.assert_array_equal(from_cm(dev["F"], Tp, r, B), host["F"])
    np.testing.assert_array_equal(dev["PF"].reshape(B, Tp, r, r), host["PF"])
    for n in ("common", "xhat", "xvar"):
        np.testing.assert_array_equal(from_cm(dev[n], Tp, N, B), host[n])
    np.testing.assert_array_equal(dev["loglik"], host["loglik"])


def check_kalman_smooth_args(lib):
    X, _ = simulate_panel(12, 2, 30, rep=1)
    Lam, Rv, A, Q = _params(X, 2, 1)

    def code(**kw):
        try:
            args = dict(p=1, H=0); args.update(kw)
            A_ = args.pop("A", A)
            lib.kalman_smooth(X, Lam, Rv, A_, Q, **args)
        except DFMError as e:
            return e.code
        return 0

    assert code(H=-1) == 1
    # k = r p = 2 * 25 = 50 > 48: the general path's limit
    assert code(p=25, A=np.zeros((2, 50))) == 6
    assert code(H=2) == 0
    T, N, r = X.shape[0], X.shape[1], 2
    for missing in ("X", "Lam", "R", "A", "Q"):
        ins = dict(X=X, Lam=Lam, R=Rv, A=A, Q=Q)
        from dynamic_factor_models_b200._lib import to_cm
        bufs = {n: (to_cm(v) if v.ndim > 1 else np.ascontiguousarray(v)) for n, v in ins.items()}
        addr = {n: (0 if n == missing else bufs[n].ctypes.data) for n in bufs}
        try:
            lib.kalman_smooth_raw(addr["X"], T, N, r, 1, 0, 1, {n: addr[n] for n in ("Lam", "R", "A", "Q")}, {}, MEM_HOST)
            raise AssertionError("null %s accepted" % missing)
        except DFMError as e:
            assert e.code == 1


def check_closed_forms(ref, A, Q, p, T, H):
    """Forecasts: f_{T+h} = [M^h z_{T|T}]_{1:r};  P_{T+h} = M P_{T+h-1} M' + Q~ (the smoothed = filtered moments there)."""
    r = A.shape[0]; k = r * p
    M = K.companion(A, r, p); Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    z = ref["zs"][T - 1]; P = ref["Ps"][T - 1]
    for h_ in range(1, H + 1):
        z = M @ z; P = M @ P @ M.T + Qt
        np.testing.assert_allclose(ref["zs"][T - 1 + h_], z, rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(ref["Ps"][T - 1 + h_], P, rtol=1e-12, atol=1e-13)
