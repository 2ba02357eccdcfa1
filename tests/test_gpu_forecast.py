"""GPU tests (-m gpu, H100) of dfm_kalman_smooth: smoothing, nowcasting and forecasting at fixed parameters against the
NumPy spec (tests/forecast_oracle.py), on synthetic panels, the C1 panel (hom_fac_1) and a full-size C2 batch."""
import numpy as np
import pytest

import forecast_checks as FC
import parity_checks as P
from forecast_oracle import smooth_forecast

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from dynamic_factor_models_b200 import Library
    L = Library()
    assert L.path.endswith("libdfm_b200.so")
    yield L
    L.close()


def _torch_alloc(keep):
    import torch

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    return alloc


def test_balanced_p1(lib): FC.check_kalman_smooth(lib, p=1, miss=0.0, H=0)
def test_balanced_p1_forecast(lib): FC.check_kalman_smooth(lib, p=1, miss=0.0, H=6)
def test_p2_missing(lib): FC.check_kalman_smooth(lib, p=2, miss=0.12, H=3)
@pytest.mark.parametrize("H", [0, 1, 8])
def test_block_missing_ragged_edge(lib, H): FC.check_kalman_smooth_block_missing(lib, H)
def test_excluded_series(lib): FC.check_kalman_smooth(lib, p=2, miss=0.05, H=4, exclude=(2, 7))
def test_long_balanced_frozen_runs(lib): FC.check_kalman_smooth(lib, N=30, r=3, T=300, p=2, miss=0.0, H=8)
def test_matches_em_first_iteration(lib): FC.check_kalman_smooth_vs_em(lib)
def test_batch_equals_single_calls(lib): FC.check_kalman_smooth_batch(lib)
def test_argument_errors(lib): FC.check_kalman_smooth_args(lib)


def test_mem_device_equals_host(lib):
    keep = []
    FC.check_kalman_smooth_mem_device(lib, _torch_alloc(keep))


def test_few_panels_cluster_path(lib):
    """One long panel: k_em_filter_smooth runs as a thread-block cluster per panel, with frozen runs in the scan."""
    FC.check_kalman_smooth(lib, N=160, r=12, T=700, p=1, miss=0.0, H=8, rep=5)


def test_c1_nowcast(lib, panels):
    """C1: Parametric (r = 8, p = 4, k = 32) on the hom_fac_1 panel, then 8-quarter forecasts and the nowcast of the ragged
    edge in data units, against the spec on the same standardized block and parameters."""
    import dynamic_factor_models_b200 as D
    m = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 8)
    D.estimate(m, D.Parametric(max_iter=5, tol=0.0), lib=lib)
    H = 8
    fc = D.forecast(m, H, lib=lib)
    i0, i1 = m.initperiod, m.lastperiod
    X = m.data[:, fc["series"]][i0 - 1:i1]
    Tw, ns = X.shape
    assert fc["xhat"].shape == (Tw + H, ns) and fc["factor"].shape == (Tw + H, 8)
    mu = np.nanmean(X, 0); sd = np.nanstd(X, 0)
    Xs = (X - mu) / sd
    out = np.isnan(m.lambda_est[:, 0]); Xs[:, out] = np.nan
    Lam = np.where(out[:, None], np.nan, m.em["Lam"])
    ref = smooth_forecast(Xs, Lam, m.em["R"], m.em["A"], m.em["Q"], m.em["P0"], 4, H)
    np.testing.assert_allclose(fc["loglik"], ref["loglik"], rtol=1e-10)
    assert P.rmse(fc["factor"], ref["F"]) < 1e-8
    np.testing.assert_allclose(fc["xhat"], mu + sd * ref["xhat"], rtol=1e-7, atol=1e-10 * np.nanmax(np.abs(X)))
    np.testing.assert_allclose(fc["xvar"], sd ** 2 * ref["xvar"], rtol=1e-7, atol=1e-10)
    inm = ~out
    # the last quarter's missing series are nowcast, every series in the model is forecast 8 quarters ahead
    last_missing = np.isnan(X[-1]) & inm
    assert last_missing.sum() >= 10
    assert np.isfinite(fc["xhat"][Tw - 1, last_missing]).all() and (fc["xvar"][Tw - 1, last_missing] > 0).all()
    assert np.isfinite(fc["xhat"][Tw:, inm]).all() and (fc["xvar"][Tw:, inm] > 0).all()
    obs = ~np.isnan(X) & inm[None, :]
    assert (fc["xvar"][:Tw][obs] == 0.0).all()
    np.testing.assert_allclose(fc["xhat"][:Tw][obs], X[obs], rtol=1e-13)          # the data, through the standardisation round trip


def test_c2_full_batch(lib):
    """C2 shape (N = 200, r = 8, T = 500), 16 panels, H = 8: the spec on two sampled panels."""
    B, N, r, T, H = 16, 200, 8, 500, 8
    Xb = lib.simulate_panels(0, B, N, r, T, 20260922)
    F0 = lib.estimate_factor(Xb, r, max_iter=1)["F"]
    Lam, Rv, A, Q = lib.em_init_from_factors(Xb, F0, 1)
    got = lib.kalman_smooth(Xb, Lam, Rv, A, Q, p=1, H=H)
    assert (got["status"] == 0).all()
    for b in (0, 11):
        ref = smooth_forecast(Xb[b], Lam[b], Rv[b], A[b], Q[b], None, 1, H)
        FC.compare({n: got[n][b] for n in ("F", "PF", "common", "xhat", "xvar")} | {"loglik": got["loglik"][b]}, ref)
