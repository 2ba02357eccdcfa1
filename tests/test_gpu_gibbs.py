"""GPU tests (-m gpu, H100) of the Gibbs sampler (dfm_gibbs): the checks of tests/test_emu_gibbs.py on the CUDA build, a C2-shaped
model and the hom_fac_1 Parametric model against the NumPy spec (tests/gibbs_oracle.py), and api.gibbs' bands and split-R^."""
import numpy as np
import pytest

import gibbs_checks as GC
import gibbs_oracle as O
import parity_checks as P

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


@pytest.fixture(scope="module")
def model():
    return GC.model()


@pytest.fixture(scope="module")
def c2(lib):
    """A C2-shaped balanced model (N = 200, r = 8, T = 500, p = 1): theta^ after 20 EM iterations on the device."""
    N, r, T = 200, 8, 500
    X = lib.simulate_panels(0, 1, N, r, T, 20260922)[0]
    F0 = lib.estimate_factor(X, r, max_iter=1)["F"]
    Lam, R, A, Q = lib.em_init_from_factors(X, F0, 1)
    em = lib.em_kalman(X, Lam, R, A, Q, p=1, max_iter=20, want_PF=False)
    return X, dict(Lam=em["Lam"], R=em["R"], A=em["A"], Q=em["Q"], P0=em["P0"])


def _c1(lib, panels):
    import dynamic_factor_models_b200 as D
    m = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 8)
    D.estimate(m, D.Parametric(max_iter=5, tol=0.0), lib=lib)
    return m


def test_chains_p2_missing_ragged_excluded(lib, model): GC.check_chains(lib, *model, p=2, n_burn=2, n_keep=3)
def test_chains_balanced_p1(lib):
    X, th = GC.model(N=14, r=3, T=40, p=1, miss=0.0, exclude=(), ragged=0)
    GC.check_chains(lib, X, th, 1, n_burn=1, n_keep=2, thin=2, H_fc=0, fc_rows=3)
def test_factor_step_is_the_simulation_smoother(lib, model): GC.check_factor_step(lib, *model, p=2)
def test_continuation(lib, model): GC.check_continuation(lib, *model, p=2)
def test_chain_split_invariance(lib, model): GC.check_chain_split(lib, *model, p=2)
def test_failed_chain(lib, model): GC.check_failed_chain(lib, *model, p=2)
def test_argument_errors(lib, model): GC.check_args(lib, *model, p=2)


def test_c2_matches_oracle(lib, c2):
    """C2-shaped model, 2 chains, 3 sweeps (all kept), against the spec chains."""
    X, th = c2
    GC.check_chains(lib, X, th, 1, n_chain=2, n_burn=0, n_keep=3, H_fc=0, fc_rows=0, H_irf=6, chain0=0, sweep0=0)


def test_c1_matches_oracle(lib, panels):
    """hom_fac_1 Parametric model (r = 8, p = 4, 5.7 % missing), 1 chain, 3 sweeps with forecasts, against the spec chain."""
    from dynamic_factor_models_b200.api import _state_space_block
    m = _c1(lib, panels)
    b = _state_space_block(m, 4, lib, "test")
    th = dict(Lam=b["Lam"], R=m.em["R"], A=m.em["A"], Q=m.em["Q"], P0=m.em["P0"])
    GC.check_chains(lib, b["Xs"], th, 4, n_chain=1, n_burn=1, n_keep=2, H_fc=4, fc_rows=6, H_irf=5, chain0=2, sweep0=1)


def test_api_gibbs_bands_and_rhat(lib, panels):
    """api.gibbs: ordered bands equal to numpy.percentile over the draws, finite split-R^, the loglik trace's R^ as the NumPy
    definition."""
    import dynamic_factor_models_b200 as D
    m = _c1(lib, panels)
    q = (5, 16, 50, 84, 95)
    out = D.gibbs(m, n_chain=4, n_burn=20, n_keep=30, H_irf=8, H_fc=3, fc_rows=5, seed=3, q=q, lib=lib)
    assert (out["status"] == 0).all()
    ib, xb = out["irf_bands"], out["x_bands"]
    assert ib.shape == (5, 8, 8, 8) and xb.shape == (5, 5, out["x"].shape[3])
    irf = out["irf"].reshape((-1,) + out["irf"].shape[2:])
    x = out["x"].reshape((-1,) + out["x"].shape[2:])
    ok = ~np.isnan(irf).any(axis=(1, 2, 3))
    assert ok.all()
    assert (np.diff(ib, axis=0) >= 0).all()
    inm = ~np.isnan(xb[0])
    assert (np.diff(xb, axis=0)[:, inm] >= 0).all()
    np.testing.assert_allclose(ib, np.percentile(irf, q, axis=0), rtol=1e-13, atol=1e-14)
    np.testing.assert_allclose(xb[:, inm], np.percentile(x, q, axis=0)[:, inm], rtol=1e-13, atol=1e-12)
    rh = out["rhat"]
    assert np.isfinite(rh["loglik"]) and np.isfinite(rh["R"][~np.isnan(out["R"][0, 0])]).all()
    kept = 20 + np.arange(30)
    assert abs(rh["loglik"] - O.split_rhat(out["loglik"][:, kept])) < 1e-12
    assert len(out["periods"]) == 5 and out["periods"][-1] == m.lastperiod + 3
    with pytest.raises(ValueError):
        D.gibbs(m, n_chain=200, n_keep=100, lib=lib)


def test_c2_rhat_after_burn_in(lib, c2):
    """4 chains on the C2 model, 500 burn-in sweeps and 200 kept: split-R^ of the loglik trace is finite (its value is reported
    in DESIGN.md 4.11; the loglik starts at the EM mode and moves to the posterior's typical set during the burn-in)."""
    X, th = c2
    got = lib.gibbs(X, th, p=1, n_chain=4, n_burn=500, n_keep=200, seed=11, prior=GC.PRIOR, outputs=("R",))
    assert (got["status"] == 0).all()
    rh = O.split_rhat(got["loglik"][:, 500:])
    print(f"C2 split-Rhat(loglik) after 500 burn-in sweeps, 4 chains x 200 kept: {rh:.4f}; "
          f"max split-Rhat(R_i): {np.nanmax(O.split_rhat(got['R'])):.4f}")
    assert np.isfinite(rh)
