"""GPU tests (-m gpu, H100) of the state-space EM under linear restrictions on the loadings (dfm_em_kalman_constrained): the
shared checks of em_constr_checks.py on the CUDA build, the kernels each call launches, a few-panel call (thread-block cluster
filter) against a many-panel call, and Stock & Watson's Figure 7 model (oil prices load one-for-one on factor 1) through
api.estimate(Parametric(), lam_constr_em=...) against the spec."""
import numpy as np
import pytest

import em_constr_checks as CC
import em_constr_oracle as O
import parity_checks as P
from oracle import dfm_ref as R

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


def _kernels(lib, fn):
    lib.profile(True)
    out = fn()
    prof = lib.profile_report(); lib.profile(False)
    return out, set(prof)


def test_missing_p2_mstep_series(lib):
    _, ks = _kernels(lib, lambda: CC.check_vs_spec(lib, N=14, r=3, T=60, p=2, miss=0.08, iters=5))
    assert "k_em_mstep_series" in ks and not any(k.startswith("k_emb_mstep") for k in ks), sorted(ks)


def test_missing_p1_excluded_series(lib): CC.check_vs_spec(lib, N=14, r=3, T=50, p=1, miss=0.05, iters=4, exclude=(1, 3))


def test_balanced_r8_p1_emb(lib):
    """Balanced r = 8, p = 1, even T: without restrictions this shape runs k_em_fused2; with them, the general path with
    k_emb_mstep_constr."""
    _, ks = _kernels(lib, lambda: CC.check_vs_spec(lib, N=40, r=8, T=60, p=1, iters=4))
    assert "k_emb_mstep_constr<NCB>" in ks and "k_em_filter_smooth" in ks, sorted(ks)
    assert not any(k.startswith("k_em_fused") for k in ks) and "k_emb_mstep<NCB>" not in ks, sorted(ks)


def test_balanced_r34_mstep_series(lib):
    _, ks = _kernels(lib, lambda: CC.check_vs_spec(lib, N=80, r=34, T=60, p=1, iters=2, rep=6))
    assert "k_em_mstep_series" in ks and not any(k.startswith("k_emb_mstep") for k in ks), sorted(ks)


def test_batch_equals_single_calls(lib): CC.check_batch(lib)
def test_zero_rows_bit_identical_fused_shape(lib): CC.check_zero_rows_bit_identical(lib, N=24, r=3, T=40, p=1)
def test_zero_rows_bit_identical_general(lib): CC.check_zero_rows_bit_identical(lib, N=16, r=3, T=40, p=2, miss=0.05)
def test_argument_errors(lib): CC.check_args(lib)
def test_dependent_rows_status_3(lib): CC.check_dependent_rows(lib)
def test_dependent_rows_status_3_balanced(lib): CC.check_dependent_rows(lib, N=40, r=3, T=60, p=1)


def test_mem_device_equals_host(lib):
    keep = []
    CC.check_mem_device(lib, _torch_alloc(keep))


def test_few_panels_match_many_panels(lib):
    """One panel (the filter runs as a thread-block cluster per panel) against the same panel inside a batch of 300 (one CTA
    per panel): 1e-10."""
    for miss in (0.06, 0.0):
        X, th = CC.panel(30, 4, 80, 2, miss, rep=31)
        cons = CC.named_and_general(4, 30, np.random.default_rng(31))
        one = lib.em_kalman(X, *th, p=2, max_iter=4, constr=cons)
        B = 300
        many = lib.em_kalman(np.stack([X] * B), *(np.stack([t] * B) for t in th), p=2, max_iter=4, constr=cons)
        for n in ("Lam", "R", "A", "Q", "F", "loglik"):
            for b in (0, B - 1):
                np.testing.assert_allclose(many[n][b], one[n], rtol=1e-10, atol=1e-12, err_msg=n)


OIL = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]


def test_figure7_through_estimate(lib, panels):
    """Figure 7 (Stock_Watson.ipynb:1326-1344): 1985Q1-2014Q4, r = 8, p = 4, the oil series' loadings restricted to e_1 in
    the ALS steps and the EM.  Both sides start from the oracle's PCA scores (as check_constraint).  The oil series'
    standardized loadings are e_1 / xstd (1e-12), the log-likelihood path is the spec's from the same start (1e-10 relative)
    and monotone from iteration 1, and forecast / series_irf run at the restricted fit."""
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200 import api
    data, incl = panels["all_bpdata"], panels["all_inclcode"]
    names = [str(s) for s in panels["all_names"]]
    calds = [tuple(x) for x in panels["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    r, p, iters = 8, 4, 6
    Rm = np.eye(r); rv = np.r_[1.0, np.zeros(r - 1)]
    used = [n for n, c in zip(names, incl) if c == 1]
    g = P.gpu_model(data, incl, r, i0, i1)
    gf = D.construct_constraint(OIL, used, Rm, rv); gfl = D.construct_constraint(OIL, names, Rm, rv)
    xs, _ = R.standardize_data(data[:, incl == 1][i0 - 1:i1])
    f0 = R.pca_score(R.drop_missing_col(xs)[0], r)
    D.estimate_factor(g, lam_constr=gf, lib=lib, f_init=f0)
    D.estimate_factor_loading(g, lam_constr=gfl, lib=lib)
    D.estimate_var(g.factor_var_model, lib=lib)
    F0 = g.factor[i0 - 1:i1].copy()
    api._estimate_parametric(g, D.Parametric(max_iter=iters, tol=0.0), lib, lam_constr_em=gf)
    e = g.em
    assert e["status"] == 0 and e["iters"] == iters
    # the spec from the device's start
    Xs, _, xstd = lib.standardize(data[:, incl == 1][i0 - 1:i1])
    Xs = np.where(np.isnan(g.lambda_est[:, :1].T), np.nan, Xs)
    th = lib.em_init_from_factors(Xs, F0, p)
    cons = e["lam_constr"]
    np.testing.assert_array_equal(cons[2], np.asarray(gf.r, float) / xstd[gf.indices])
    ref = O.em_kalman(Xs, *th, p=p, max_iter=iters, constr=cons)
    np.testing.assert_allclose(e["loglik"], ref["loglik"], rtol=1e-10)
    ll = e["loglik"][1:]
    assert (np.diff(ll) >= -1e-9 * np.abs(ll[:-1])).all(), np.diff(ll)
    assert P.rmse(e["F"], ref["F"]) < 1e-7
    oil = [used.index(n) for n in OIL]
    inm = [i for i in oil if not np.isnan(e["Lam"][i, 0])]
    assert len(inm) >= 3, inm
    for i in inm:
        np.testing.assert_allclose(e["Lam"][i], rv / xstd[i], rtol=0, atol=1e-12 / xstd[i])
    fc = D.forecast(g, 4, lib=lib)
    assert np.isfinite(fc["xhat"][:, inm]).all() and fc["xhat"].shape == (i1 - i0 + 5, len(used))
    si = D.series_irf(g, 8, lib=lib)
    assert si.shape == (len(used), 8, r)
    irf = D.parametric_irf(g, 8, lib=lib)
    for i in inm:                     # data-unit response of an oil series to shock 1 = factor 1's own response
        np.testing.assert_allclose(si[i, :, 0], irf[0, :, 0], rtol=1e-10, atol=1e-12)
    with pytest.raises(ValueError):
        D.parametric_bootstrap(g, 2, lib=lib)
