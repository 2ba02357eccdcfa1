"""GPU tests (-m gpu, H100) of dfm_simulation_smoother: draws against the NumPy spec (tests/simsmooth_oracle.py) draw for
draw on synthetic panels, the C1 model (hom_fac_1 at its Parametric estimates) and a long panel whose E-step runs as a
thread-block cluster; the moments of 4096 draws of a C2-shaped model against dfm_kalman_smooth's posterior mean and variance."""
import numpy as np
import pytest

import parity_checks as P
import simsmooth_checks as SC
from simsmooth_oracle import simulation_smoother

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


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("miss", [0.0, 0.15])
@pytest.mark.parametrize("H", [0, 3])
def test_draws_match_spec(lib, p, miss, H): SC.check_sim(lib, p=p, miss=miss, H=H)
def test_period_with_fewer_than_r_series(lib): SC.check_sim(lib, r=3, p=2, miss=0.05, H=2, few_obs=(10, 11, 40))
def test_excluded_series(lib): SC.check_sim(lib, p=2, miss=0.05, H=4, exclude=(2, 7))
@pytest.mark.parametrize("H", [0, 8])
def test_block_missing_ragged_edge(lib, H): SC.check_block_missing(lib, H)
def test_long_balanced_frozen_runs(lib): SC.check_sim(lib, N=30, r=3, T=300, p=2, miss=0.0, H=8, n_draw=3)
def test_draws_not_a_multiple_of_the_tile(lib): SC.check_sim(lib, N=10, r=2, T=40, p=1, miss=0.1, H=2, n_draw=37, draw0=1000,
                                                             check_ids=(0, 15, 16, 36))
def test_shard_invariance(lib): SC.check_shard_invariance(lib)
def test_failed_estep(lib): SC.check_failed_estep(lib)
def test_argument_errors(lib): SC.check_args(lib)


def test_mem_device_equals_host(lib):
    keep = []
    SC.check_mem_device(lib, _torch_alloc(keep))


def test_few_panels_cluster_path(lib):
    """One long panel: k_em_filter_smooth runs as a thread-block cluster, with frozen runs in the scan."""
    SC.check_sim(lib, N=160, r=12, T=700, p=1, miss=0.0, H=8, rep=5, n_draw=40, check_ids=(0, 17, 39))


def test_c1_posterior_draws(lib, panels):
    """C1: Parametric (r = 8, p = 4, k = 32) on hom_fac_1, then posterior_draws with H = 8, against the spec on the same
    standardized block and parameters for a few draw ids."""
    import dynamic_factor_models_b200 as D
    m = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 8)
    D.estimate(m, D.Parametric(max_iter=5, tol=0.0), lib=lib)
    H, seed, draw0, n = 8, 77, 3, 40
    dr = D.posterior_draws(m, H, n, seed, draw0=draw0, lib=lib)
    i0, i1 = m.initperiod, m.lastperiod
    X = m.data[:, dr["series"]][i0 - 1:i1]
    Tw, ns = X.shape
    assert dr["x"].shape == (n, Tw + H, ns) and dr["factor"].shape == (n, Tw + H, 8)
    mu = np.nanmean(X, 0); sd = np.nanstd(X, 0)
    Xs = (X - mu) / sd
    out = np.isnan(m.lambda_est[:, 0]); Xs[:, out] = np.nan
    Lam = np.where(out[:, None], np.nan, m.em["Lam"])
    pos = [0, 1, 22, 39]
    refF, refX = simulation_smoother(Xs, Lam, m.em["R"], m.em["A"], m.em["Q"], m.em["P0"], 4, H, seed, [draw0 + j for j in pos])
    assert np.max(np.abs(dr["factor"][pos] - refF)) <= 1e-9
    got_std = (dr["x"][pos] - mu) / sd
    assert (np.isnan(got_std) == np.isnan(refX)).all()
    ok = ~np.isnan(refX)
    assert np.max(np.abs(got_std[ok] - refX[ok])) <= 1e-9
    obs = ~np.isnan(X) & ~out[None, :]
    for j in pos:
        np.testing.assert_allclose(dr["x"][j, :Tw][obs], X[obs], rtol=1e-13)        # the data, through the standardisation
    bands = D.forecast_bands(m, H, [5.0, 50.0, 95.0], 400, seed, lib=lib)
    assert bands["bands"].shape == (3, Tw + H, ns)
    lo, med, hi = bands["bands"]
    inm = ~out
    assert (lo[Tw:, inm] < med[Tw:, inm]).all() and (med[Tw:, inm] < hi[Tw:, inm]).all()


def test_c2_moments_match_kalman_smooth(lib):
    """C2 shape (N = 200, r = 8, T = 500), H = 8, 4096 draws: the sample mean of the factor draws is dfm_kalman_smooth's F
    within 5 Monte-Carlo standard errors, the sample variance its PF diagonal within 5 standard errors of a variance."""
    N, r, T, H, n = 200, 8, 500, 8, 4096
    X = lib.simulate_panels(0, 1, N, r, T, 20260922)[0]
    F0 = lib.estimate_factor(X, r, max_iter=1)["F"]
    Lam, Rv, A, Q = lib.em_init_from_factors(X, F0, 1)
    ks = lib.kalman_smooth(X, Lam, Rv, A, Q, p=1, H=H, outputs=("F", "PF"))
    got = lib.simulation_smoother(X, Lam, Rv, A, Q, p=1, H=H, n_draw=n, seed=5, outputs=("F",))
    assert got["status"] == 0 and ks["status"] == 0
    v = np.einsum("taa->ta", ks["PF"])
    mean = got["F"].mean(0); var = got["F"].var(0, ddof=1)
    assert (np.abs(mean - ks["F"]) <= 5 * np.sqrt(v / n)).all(), np.max(np.abs(mean - ks["F"]) / np.sqrt(v / n))
    assert (np.abs(var - v) <= 5 * v * np.sqrt(2.0 / (n - 1))).all(), np.max(np.abs(var - v) / (v * np.sqrt(2.0 / (n - 1))))
