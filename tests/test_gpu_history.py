"""GPU tests (-m gpu, H100) of the historical decompositions (dfm_historical_decomposition): the checks of
tests/test_emu_history.py on the CUDA build, and Stock & Watson's Figure 7 model (the oil series pinned to e_1) through
api.historical_decomposition and api.identified_history."""
import copy

import numpy as np
import pytest

import history_checks as HC
import identified_oracle as IO
from test_gpu_identified import figure7

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


@pytest.fixture
def alloc():
    import torch
    keep = []

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2, 4])
@pytest.mark.parametrize("r", [1, 8, 12])
def test_matches_spec(lib, r, p):
    lib.profile(True)
    HC.check_against_spec(lib, r, p)
    ks = set(lib.profile_report()); lib.profile(False)
    assert {"k_sr_prep", "k_hd_paths"} <= ks and any(k.startswith("k_hd_series") for k in ks), sorted(ks)


def test_k49_refused(lib): HC.check_k49_refused(lib)
def test_failed_models_and_nan_series(lib): HC.check_failed_models_and_nan_series(lib)
def test_device_equals_host(lib, alloc): HC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): HC.check_chunks(lib, alloc)
def test_argument_errors(lib): HC.check_args(lib)


def _rotated(g, Km):
    """g with its EM estimates rotated by f -> K f (P0 of the stacked state by blockdiag(K, .., K))."""
    e = g.em
    r = e["Q"].shape[0]; p = e["A"].shape[1] // r
    Lam, A, Q = IO.rotate(e["Lam"], e["A"], e["Q"], Km, p)
    Kz = np.kron(np.eye(p), Km)
    g2 = copy.copy(g)
    g2.em = dict(e, Lam=Lam, A=A, Q=Q, P0=Kz @ e["P0"] @ Kz.T)
    return g2


def test_figure7_identified_history(lib, panels):
    import dynamic_factor_models_b200 as D
    g, inm = figure7(lib, panels)
    assert len(inm) >= 3, inm
    q = (5, 16, 50, 84, 95)
    hd = D.historical_decomposition(g, lib=lib)
    T, r = hd["shocks"].shape
    assert hd["t0"] == g.initperiod + 3 and hd["contrib"].shape == (len(hd["series"]), T, r)
    X = g.data[:, hd["series"]][g.initperiod - 1:g.lastperiod]
    xmean = lib.standardize(X)[1]
    obs = ~np.isnan(hd["resid"])
    assert obs.sum() > 0.5 * X.size
    tot = xmean[:, None] + hd["base"] + hd["contrib"].sum(-1) + hd["resid"]
    np.testing.assert_allclose(tot[obs], X.T[obs], rtol=1e-10, atol=1e-10 * np.nanmax(np.abs(X)))
    # (both samplers lose chains on this model after 150-230 sweeps: their A draws are not restricted to be stationary;
    # DESIGN.md 4.12)
    out = D.identified_history(g, shocks=1, n_chain=4, n_burn=40, n_keep=80, seed=7, q=q, return_draws=True, lib=lib)
    assert (out["status"] == 0).all(), out["status"]
    ok = np.isfinite(hd["base"][:, 0])
    s = np.nanmax(np.abs(hd["contrib"]))
    np.testing.assert_allclose(out["contrib"][ok, :, 0], hd["contrib"][ok, :, 0], rtol=0, atol=1e-13 * s)
    np.testing.assert_allclose(out["base"][ok], hd["base"][ok], rtol=0, atol=1e-13 * np.nanmax(np.abs(hd["base"])))
    np.testing.assert_allclose(out["rest"][ok], hd["contrib"][ok, :, 1:].sum(-1), rtol=0, atol=1e-12 * s)
    for nm, tail in (("contrib", (len(ok), T, 1)), ("rest", (len(ok), T)), ("base", (len(ok), T)), ("shocks", (T, 1))):
        bd, dr = out[nm + "_bands"], out[nm + "_draws"]
        assert bd.shape == (len(q),) + tail and dr.shape == (4, 80) + tail, nm
        sel = (slice(None), ok) if nm != "shocks" else (slice(None), slice(4, None))   # (eps_t is NaN for t < p = 4)
        assert (np.diff(bd[sel], axis=0) >= 0).all(), nm
        ref = np.percentile(dr.reshape((-1,) + tail), q, axis=0)
        np.testing.assert_allclose(bd[sel], ref[sel], rtol=1e-13, atol=1e-14 * np.nanmax(np.abs(ref)), err_msg=nm)
    t0r = out["t0"] - g.initperiod
    assert np.isfinite(out["rhat"]["loglik"]) and np.isfinite(out["rhat"]["contrib"][ok, t0r + 1:]).all()
    for i in inm:                                         # an oil series' shock-1 part moves with the shock
        assert np.abs(out["contrib_draws"][:, :, i, t0r + 1:, 0]).max() > 0
    Kf = np.eye(r) + 0.3 * np.random.default_rng(3).standard_normal((r, r)); Kf[0] = np.r_[1.0, np.zeros(r - 1)]
    hr = D.historical_decomposition(_rotated(g, Kf), lib=lib)
    np.testing.assert_allclose(hr["contrib"][ok, :, 0], hd["contrib"][ok, :, 0], rtol=0, atol=1e-10 * s)
    np.testing.assert_allclose(hr["base"][ok], hd["base"][ok], rtol=0, atol=1e-10 * np.nanmax(np.abs(hd["base"])))
    with pytest.raises(ValueError):
        D.identified_history(g, shocks=2, lib=lib)        # factor 2 is not named
