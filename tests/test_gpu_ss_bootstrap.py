"""GPU tests (-m gpu, H100) of the parametric bootstrap of a fitted state-space model: dfm_ss_simulate_panels against the NumPy
spec (tests/ss_bootstrap_oracle.py), shard and memory invariance, dfm_ss_bootstrap against the spec pipeline (spec panel ->
oracle EM from theta^ -> align -> IRF) on a C2-shaped model (fused EM path) and on the hom_fac_1 Parametric model (general path),
sub-batching, alignment failures, and api.parametric_bootstrap / parametric_irf."""
import numpy as np
import pytest

import parity_checks as P
import ss_bootstrap_checks as BC
import ss_bootstrap_oracle as O

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
    return BC.fitted(N=14, r=3, T=40, p=2, miss=0.1, exclude=(4,), ragged=3)


@pytest.fixture(scope="module")
def c2(lib):
    """A C2-shaped balanced model (N = 200, r = 8, T = 500, p = 1): theta^ after 20 EM iterations on the device."""
    N, r, T = 200, 8, 500
    X = lib.simulate_panels(0, 1, N, r, T, 20260922)[0]
    F0 = lib.estimate_factor(X, r, max_iter=1)["F"]
    Lam, R, A, Q = lib.em_init_from_factors(X, F0, 1)
    em = lib.em_kalman(X, Lam, R, A, Q, p=1, max_iter=20, want_PF=False)
    return X, dict(Lam=em["Lam"], R=em["R"], A=em["A"], Q=em["Q"], P0=em["P0"])


def _torch_alloc(keep):
    import torch

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2, 3])
def test_simulate_matches_spec(lib, p): BC.check_simulate(lib, r=3, p=p, miss=0.1)
def test_simulate_missing_ragged_excluded(lib): BC.check_simulate(lib, N=70, r=5, T=45, p=2, miss=0.2, exclude=(1, 66), ragged=4,
                                                                  n_rep=35, check=(0, 15, 16, 31, 32, 34))
def test_simulate_balanced_r9(lib): BC.check_simulate(lib, N=20, r=9, T=36, p=1, miss=0.0, n_rep=17, check=(0, 16))
def test_simulate_c2(lib, c2): BC.check_simulate(lib, X=c2[0], th=c2[1], p=1, n_rep=40, check=(0, 39))
def test_shard_invariance(lib, model): BC.check_shard_invariance(lib, *model, p=2, n_rep=21, world=8)
def test_mem_device_equals_host(lib, model):
    keep = []
    BC.check_mem_device(lib, _torch_alloc(keep), *model, p=2)


def test_bootstrap_small_general_path(lib, model): BC.check_bootstrap(lib, *model, p=2, n_rep=3, H_fc=2, fc_rows=6, par_tol=1e-9,
                                                                      ll_rtol=1e-11, fc_tol=1e-9)
def test_bootstrap_shards(lib, model): BC.check_bootstrap_shards(lib, *model, p=2)
def test_failed_replicate(lib, model): BC.check_failed_replicate(lib, *model, p=2)
def test_argument_errors(lib, model): BC.check_args(lib, *model, p=2)


def test_c2_fused_path_matches_oracle(lib, c2):
    """C2-shaped balanced model, 5 replicates, 20 EM iterations on the fused path (k_em_fused2 in the profile): replicates 0 and
    4 against the oracle pipeline -- parameters and IRFs to 1e-8, log-likelihood to 1e-9 relative."""
    X, th = c2
    lib.profile(True)
    got = BC.check_bootstrap(lib, X, th, 1, n_rep=5, rep0=7, max_iter=20, H_irf=12, H_fc=0, fc_rows=0, check=(0, 4), par_tol=1e-8,
                             ll_rtol=1e-9)
    prof = lib.profile_report(); lib.profile(False)
    assert any(n.startswith("k_em_fused2") for n in prof) and "k_em_filter_smooth" not in prof, sorted(prof)
    assert (got["status"] == 0).all()


def test_sub_batches_general_path(lib, model):
    """General path (p = 2, missing data, a series out of the model, the forecast E-step): calls of 20, 50 and 300 replicates --
    batches whose own plans of k_em_filter_smooth would differ (clusters of 8 CTAs, 2, none) -- give the same bits for the same
    replication ids."""
    BC.check_sub_batches(lib, *model, p=2)


def test_sub_batches_c2(lib, c2):
    """The same on the fused path (C2 shape, 5 EM iterations) with the forecast E-step of the general path."""
    BC.check_sub_batches(lib, *c2, p=1, max_iter=5)


def test_failed_alignment(lib, model): BC.check_failed_alignment(lib, *model, p=2)
def test_simulate_r48_shared_memory(lib): BC.check_simulate(lib, N=60, r=48, T=60, p=1, miss=0.0, n_rep=9, check=(0, 8))


def _c1(lib, panels):
    import dynamic_factor_models_b200 as D
    m = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 8)
    D.estimate(m, D.Parametric(max_iter=5, tol=0.0), lib=lib)
    return m


def test_c1_general_path_matches_oracle(lib, panels):
    """hom_fac_1 Parametric model (r = 8, p = 4, missing data): parametric_bootstrap with 3 replicates, 3 EM iterations each,
    against the oracle pipeline for replicates 0 and 2, and parametric_irf against the oracle IRF of m.em."""
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200.api import _state_space_block
    m = _c1(lib, panels)
    H_irf, H_fc, fr, seed = 10, 4, 6, 31
    out = D.parametric_bootstrap(m, 3, H_irf=H_irf, H_fc=H_fc, fc_rows=fr, seed=seed, max_iter=3, tol=0.0, lib=lib)
    b = _state_space_block(m, H_fc, lib, "test")
    th = dict(Lam=b["Lam"], R=m.em["R"], A=m.em["A"], Q=m.em["Q"], P0=m.em["P0"])
    raw = dict(Lam=out["Lam"], R=out["R"], A=out["A"], Q=out["Q"], irf=out["irf"], loglik=out["loglik"], iters=out["iters"],
               status=out["status"], xhat=(out["xhat"] - b["xmean"]) / b["xstd"], xvar=out["xvar"] / b["xstd"] ** 2)
    for j in (0, 2):
        ref = O.replicate(b["Xs"], th, 4, seed, j, 3, 0.0, H_irf, H_fc, fr)
        BC.compare_replicate(raw, j, ref, 1e-8, 1e-9, fc_tol=1e-8)
    np.testing.assert_allclose(out["irf_point"], O.irf(m.em["A"], m.em["Q"], 4, H_irf).transpose(2, 1, 0), atol=1e-12)
    np.testing.assert_allclose(D.parametric_irf(m, H_irf, lib=lib), out["irf_point"], atol=0)


def test_parametric_bootstrap_bands(lib, panels):
    """Bands are ordered, the device percentiles are numpy.percentile's, total_var is its definition."""
    import dynamic_factor_models_b200 as D
    m = _c1(lib, panels)
    q = (5, 16, 50, 84, 95)
    out = D.parametric_bootstrap(m, 40, H_irf=8, H_fc=3, fc_rows=5, seed=3, q=q, max_iter=3, tol=0.0, lib=lib)
    ok = out["status"] == 0
    assert ok.sum() >= 38
    ib, xb = out["irf_bands"], out["xhat_bands"]
    assert ib.shape == (5, 8, 8, 8) and xb.shape == (5, 5, out["xhat"].shape[2])
    assert (np.diff(ib, axis=0) >= 0).all()
    inm = ~np.isnan(xb[0])
    assert (np.diff(xb, axis=0)[:, inm] >= 0).all()
    np.testing.assert_allclose(ib, np.percentile(out["irf"][ok], q, axis=0), rtol=1e-13, atol=1e-14)
    np.testing.assert_allclose(xb[:, inm], np.percentile(out["xhat"][ok], q, axis=0)[:, inm], rtol=1e-13, atol=1e-12)
    tv = out["xvar"][ok].mean(0) + out["xhat"][ok].var(0)
    np.testing.assert_allclose(out["total_var"][inm], tv[inm], rtol=1e-13)
    assert (out["total_var"][inm] >= out["xvar"][ok].mean(0)[inm]).all()
    assert len(out["periods"]) == 5 and out["periods"][-1] == m.lastperiod + 3
