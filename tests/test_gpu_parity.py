"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C ABI vs the
oracle, on the reference's own panel (hom_fac_1, committed fixture), seeded synthetic panels,
edge cases, and size-independent properties at BASELINE.json's full sizes."""
import numpy as np
import pytest

import parity_checks as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from dynamic_factor_models_b200 import Library
    L = Library()            # in-tree CUDA build; raises if missing (no fallback)
    assert L.path.endswith("libdfm_b200.so")
    yield L
    L.close()


def test_standardize(lib): P.check_standardize(lib)
def test_pca(lib): P.check_pca(lib)
def test_estimate_factor_same_init(lib): P.check_estimate_factor_same_init(lib)
def test_estimate_factor_c1(lib, panels): P.check_estimate_factor_c1(lib, panels)
def test_estimate_factor_c1_r1(lib, panels): P.check_estimate_factor_c1(lib, panels, r=1)
def test_constraint(lib, panels): P.check_constraint(lib, panels)
def test_full_nonparametric_c1(lib, panels): P.check_full_nonparametric_c1(lib, panels)
def test_var_irf(lib): P.check_var_irf(lib)
def test_simulate_panels(lib): P.check_simulate_panels(lib)
def test_simulate_panels_c2_shape(lib): P.check_simulate_panels(lib, N=200, r=8, T=500, B=2, rep0=1249)
def test_simulate_panels_statistics(lib): P.check_simulate_panels_statistics(lib)
def test_bootstrap_panels(lib, panels): P.check_bootstrap_panels(lib, panels)
def test_percentiles(lib): P.check_percentiles(lib)
def test_percentiles_1000(lib): P.check_percentiles(lib, n=1000, d=1536)
def test_var_missing_rows(lib): P.check_var_missing_rows(lib)
def test_fit_correlation(lib, panels): P.check_fit_correlation(lib, panels)
def test_instability_edges(lib): P.check_instability_edges(lib)
def test_instability_r4(lib, panels): P.check_instability(lib, panels, r=4, series=list(range(0, 207, 9)))
def test_instability_r8(lib, panels): P.check_instability(lib, panels, r=8, series=list(range(3, 207, 17)))
def test_em_p1_balanced(lib): P.check_em(lib, p=1, miss=0.0, path=1)
def test_em_p2_missing(lib): P.check_em(lib, p=2, miss=0.12, path=1)
def test_em_p1_missing(lib): P.check_em(lib, p=1, miss=0.1, path=1, rep=10)
def test_em_auto_path(lib): P.check_em(lib, N=40, r=8, T=90, p=1, miss=0.0, path=0, iters=5)
def test_em_convergence_rule(lib): P.check_em_convergence_rule(lib, path=1)
def test_em_p2_long_balanced_frozen(lib): P.check_em(lib, N=30, r=3, T=300, p=2, miss=0.0, iters=3, path=1)
def test_em_r12_balanced_frozen(lib): P.check_em(lib, N=60, r=12, T=240, p=1, miss=0.0, iters=3, path=1)
def test_em_block_missing_frozen(lib): P.check_em_block_missing(lib)
def test_em_r12_long_run(lib): P.check_em(lib, N=50, r=12, T=420, p=1, miss=0.0, iters=3, path=1)      # run scan: 2 row blocks of the state
def test_em_p4_balanced_long_run(lib): P.check_em(lib, N=40, r=8, T=330, p=4, miss=0.0, iters=2, path=1)   # companion state k = 32
def test_em_r20_balanced(lib): P.check_em(lib, N=120, r=20, T=300, p=1, miss=0.0, iters=2, path=1)       # three DMMA column blocks
def test_em_r28_balanced(lib): P.check_em(lib, N=90, r=28, T=300, p=1, miss=0.0, iters=2, path=1)        # four column blocks, 51 KB M-step tile
def test_em_batch(lib): P.check_em_batch(lib, path=1)
def test_als_batch(lib): P.check_als_batch(lib)
def test_als_balanced_fused(lib): P.check_als_balanced(lib)
def test_als_balanced_fused_r8(lib): P.check_als_balanced(lib, N=48, r=8, T=120, B=2)
def test_parametric_c1(lib, panels): P.check_parametric_c1(lib, panels, iters=3)
def test_nile_published_general(lib): P.check_nile_published(lib, path=1)
def test_nile_published_fused(lib): P.check_nile_published(lib, path=2)
def test_nile_published_fused2(lib): P.check_nile_published(lib, path=3)


def test_table2B_through_gpu(lib, panels, notebook_tables):
    """Golden Table 2B (Stock_Watson.ipynb:616-629) reproduced by the CUDA path, r = 1..10."""
    import dynamic_factor_models_b200 as D
    gold = np.array(notebook_tables["table2B"])
    for r in range(1, 11):
        g = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], r)
        D.estimate_factor(g, computeR2=False, lib=lib)
        assert abs((1 - g.fes.ssr / g.fes.tss) - gold[r - 1, 1]) < 6e-4
        assert abs(D.bai_ng_criterion(g) - gold[r - 1, 3]) < 6e-4


def test_table2A_through_gpu(lib, panels, notebook_tables):
    """Golden Table 2A (Stock_Watson.ipynb:569-577; Real panel, N = 58 estimation series, r = 1..5): trace R2, marginal
    R2, Bai-Ng ICp2 and the Ahn-Horenstein eigenvalue ratio, all from the CUDA path."""
    import dynamic_factor_models_b200 as D
    gold = np.array(notebook_tables["table2A"])
    tr, bn = [], []
    for r in range(1, 7):
        g = P.gpu_model(panels["real_bpdata"], panels["real_inclcode"], r)
        D.estimate_factor(g, computeR2=False, lib=lib)
        tr.append(1 - g.fes.ssr / g.fes.tss); bn.append(D.bai_ng_criterion(g))
    tr = np.array(tr); marg = np.diff(np.concatenate([[0], tr])); ah = marg[:-1] / marg[1:]
    got = np.column_stack([np.arange(1, 6), tr[:5], marg[:5], bn[:5], ah[:5]])
    np.testing.assert_allclose(got, gold, atol=6e-4)


def test_table2C_amengual_watson_through_gpu(lib, panels, notebook_tables):
    """Golden Table 2C (Stock_Watson.ipynb:669-683): Amengual-Watson ICp for 1..10 static x 1..10 dynamic factors --
    estimate_factor_numbers (dfm_functions.ipynb:698-768) on the device: 10 static fits, 10 residualising regressions
    (dfm_estimate_loading_ex returns the residuals) and 55 ALS fits of the residual panels."""
    import dynamic_factor_models_b200 as D
    gold = np.array(notebook_tables["table2C"])[:, 1:]
    g = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 1)
    out = D.estimate_factor_numbers(g, 10, lib=lib)
    got = out["aw_icp"]
    mask = ~np.isnan(gold)
    assert (np.isnan(got) == np.isnan(gold)).all()
    np.testing.assert_allclose(got[mask], gold[mask], atol=6e-4)
    gold2b = np.array(notebook_tables["table2B"])
    np.testing.assert_allclose(out["bn_icp"], gold2b[:, 3], atol=6e-4)


def test_c2_full_size_vs_oracle(lib):
    """BASELINE config C2 (N=200, r=8, T=500): 3 EM iterations vs the oracle + EM invariants."""
    P.check_em(lib, N=200, r=8, T=500, p=1, miss=0.0, iters=3, path=0, rep=0)


def test_c2_full_size_properties(lib):
    """Size-independent properties at full C2 size over a batch: monotone log-likelihood, batch
    independence (a panel's result does not depend on its neighbours), permutation equivariance."""
    from oracle.dgp import simulate_batch
    from oracle import dfm_ref as R, kalman_em as K
    B, N, r, T = 6, 200, 8, 500
    Xb = simulate_batch(B, N, r, T, rep0=100)
    inits = [K.init_from_factors(Xb[b], R.pca_score(Xb[b], r), 1) for b in range(B)]
    Lam = np.stack([i[0] for i in inits]); Rv = np.stack([i[1] for i in inits])
    A = np.stack([i[2] for i in inits]); Q = np.stack([i[3] for i in inits])
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=20)
    ll = got["loglik"]
    assert (np.diff(ll, axis=1) > -1e-9 * np.abs(ll[:, :-1])).all()
    perm = np.array([3, 0, 5, 1, 4, 2])
    got2 = lib.em_kalman(Xb[perm], Lam[perm], Rv[perm], A[perm], Q[perm], p=1, max_iter=20)
    np.testing.assert_allclose(got2["F"], got["F"][perm], rtol=1e-12, atol=1e-13)
    # series-permutation equivariance: reordering series leaves factors unchanged (to rounding)
    sp = np.random.default_rng(0).permutation(N)
    got3 = lib.em_kalman(Xb[0][:, sp], Lam[0][sp], Rv[0][sp], A[0], Q[0], p=1, max_iter=20)
    assert P.rmse(got3["F"], got["F"][0]) < 1e-9
    np.testing.assert_allclose(got3["Lam"], got["Lam"][0][sp], rtol=1e-7, atol=1e-9)


# ---- fused per-panel EM kernel (DMMA contractions, steady-state covariance chain), path=2
def test_fused_em_r3(lib): P.check_em(lib, p=1, miss=0.0, path=2)
def test_fused_em_r8(lib): P.check_em(lib, N=40, r=8, T=90, p=1, miss=0.0, path=2, iters=5)
def test_fused_em_r1(lib): P.check_em(lib, N=12, r=1, T=50, p=1, miss=0.0, path=2, iters=4)
def test_fused_em_r5_ragged(lib): P.check_em(lib, N=37, r=5, T=101, p=1, miss=0.0, path=2, iters=4)   # N % 4 != 0, T % 8 != 0
def test_fused_em_convergence_rule(lib): P.check_em_convergence_rule(lib, path=2)
def test_fused_em_batch(lib): P.check_em_batch_balanced(lib, B=7, path=2)
def test_fused_matches_general_c2(lib):
    """fused vs general path on a full-size C2 panel, 10 iterations."""
    from oracle.dgp import simulate_panel
    from oracle import dfm_ref as R, kalman_em as K
    X, _ = simulate_panel(200, 8, 500, rep=3)
    Lam, Rv, A, Q = K.init_from_factors(X, R.pca_score(X, 8), 1)
    g1 = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=10, path=1)
    g2 = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=10, path=2)
    np.testing.assert_allclose(g2["loglik"], g1["loglik"], rtol=1e-11)
    assert P.rmse(g2["F"], g1["F"]) < 1e-9
    np.testing.assert_allclose(g2["PF"], g1["PF"], rtol=1e-7, atol=1e-11)
    np.testing.assert_allclose(g2["Lam"], g1["Lam"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(g2["A"], g1["A"], rtol=1e-6, atol=1e-9)
def test_fused_rejects_missing(lib):
    from dynamic_factor_models_b200 import DFMError
    with pytest.raises(DFMError):
        P.check_em(lib, p=1, miss=0.1, path=2)
    P.check_em(lib, p=1, miss=0.1, path=0)


# ---- TMA-fed fused kernel (cp.async.bulk ring + mbarriers + DMMA), path=3
def test_fused2_em_r3(lib): P.check_em(lib, p=1, miss=0.0, path=3)
def test_fused2_em_r8(lib): P.check_em(lib, N=40, r=8, T=90, p=1, miss=0.0, path=3, iters=5)
def test_fused2_em_r1(lib): P.check_em(lib, N=12, r=1, T=50, p=1, miss=0.0, path=3, iters=4)
def test_fused2_em_r5_ragged(lib): P.check_em(lib, N=37, r=5, T=102, p=1, miss=0.0, path=3, iters=4)   # N % 8 != 0, one short period chunk
def test_fused2_em_long(lib): P.check_em(lib, N=24, r=4, T=300, p=1, miss=0.0, path=3, iters=3)        # several ring wraps, 2 period chunks
def test_fused2_em_ragged_long(lib): P.check_em(lib, N=45, r=8, T=278, p=1, miss=0.0, path=3, iters=3)   # tail chunk 106 periods (len % 4 == 2), N % 8 == 5
def test_fused2_em_exact_chunks(lib): P.check_em(lib, N=16, r=8, T=264, p=1, miss=0.0, path=3, iters=3)   # a full chunk + a 92-period tail (T = 2 x 132 fitted the former box)
def test_fused2_em_convergence_rule(lib): P.check_em_convergence_rule(lib, path=3)
def test_fused2_em_batch(lib): P.check_em_batch_balanced(lib, B=7, path=3)
def test_fused2_matches_general_c2(lib):
    from oracle.dgp import simulate_panel
    from oracle import dfm_ref as R, kalman_em as K
    X, _ = simulate_panel(200, 8, 500, rep=3)
    Lam, Rv, A, Q = K.init_from_factors(X, R.pca_score(X, 8), 1)
    g1 = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=10, path=1)
    g2 = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=10, path=3)
    np.testing.assert_allclose(g2["loglik"], g1["loglik"], rtol=1e-11)
    assert P.rmse(g2["F"], g1["F"]) < 1e-9
    np.testing.assert_allclose(g2["PF"], g1["PF"], rtol=1e-7, atol=1e-11)
    np.testing.assert_allclose(g2["Lam"], g1["Lam"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(g2["A"], g1["A"], rtol=1e-6, atol=1e-9)
def test_fused2_odd_T_falls_back(lib):
    from dynamic_factor_models_b200 import DFMError
    with pytest.raises(DFMError):
        P.check_em(lib, N=20, r=3, T=71, p=1, path=3)
    P.check_em(lib, N=20, r=3, T=71, p=1, path=0)


def test_pca_subspace(lib): P.check_pca(lib, r=5, sizes=((150, 90), (80, 130), (300, 200)))


def test_c3_full_size(lib):
    """BASELINE config C3 (N=2000, r=20, T=2000): PCA by subspace iteration vs LAPACK SVD, one ALS sweep
    and ten EM iterations of the general path (frozen-step logic: ~25 explicit covariance steps of 2000) vs the oracle's C port."""
    from oracle.dgp import simulate_panel
    from oracle.c import kem
    from oracle import dfm_ref as R, kalman_em as K
    N, r, T = 2000, 20, 2000
    X, _ = simulate_panel(N, r, T, rep=0)
    ref = R.pca_score(X, r)
    got = lib.pca_score(X, r)
    got, _ = P.sign_align(got, ref)
    assert P.rmse(got, ref) < 1e-8 * np.abs(ref).max()
    out = lib.estimate_factor(X, r, max_iter=1, compute_r2=False, F_init=ref)
    assert out["stats"]["status"] in (0, 4)
    Lam, Rv, A, Q = lib.em_init_from_factors(X, out["F"], 1)
    em = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=10, want_PF=False)
    cref = kem.em_kalman_batch(X[None], Lam[None], Rv[None], A[None], Q[None], p=1, max_iter=10)
    np.testing.assert_allclose(em["loglik"], cref["loglik"][0], rtol=1e-9)
    assert P.rmse(em["F"], cref["F"][0]) < 1e-8


def _many_small_panels(B, N=16, r=2, T=40):
    from oracle import dfm_ref as R, kalman_em as K
    from oracle.dgp import simulate_panel
    Xb = np.stack([simulate_panel(N, r, T, rep=500 + b)[0] for b in range(B)])
    base = [K.init_from_factors(Xb[b], R.pca_score(Xb[b], r), 1) for b in range(8)]
    rng = np.random.default_rng(1)
    pick = rng.integers(0, 8, B)
    # cheap, valid (not optimal) starting points: parameters of one of 8 fitted panels
    return Xb, np.stack([base[i][0] for i in pick]), np.stack([base[i][1] for i in pick]), np.stack([base[i][2] for i in pick]), np.stack([base[i][3] for i in pick])


def test_pipelined_host_path_matches_monolithic(lib):
    """Host buffers + batch larger than the fused kernel's capacity -> streaming path (one launch that starts
    before the upload, chunks signalled by stream-ordered flag copies, P0 computed in the kernel); must equal
    the upload-then-compute path bit for bit, and a few panels are checked against the oracle."""
    import os
    from oracle import kalman_em as K
    Xb, Lam, Rv, A, Q = _many_small_panels(1500)
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=4)
    os.environ["DFM_NO_PIPELINE"] = "1"
    try:
        ref = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=4)
    finally:
        del os.environ["DFM_NO_PIPELINE"]
    for k in ("F", "Lam", "R", "A", "Q", "loglik", "PF", "P0"):
        np.testing.assert_array_equal(got[k], ref[k])
    assert (got["status"] == 0).all() and (got["iters"] == 4).all()
    for b in (0, 777, 1499):
        o = K.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], p=1, max_iter=4)
        assert P.rmse(got["F"][b], o["F"]) < 1e-8
        np.testing.assert_allclose(got["loglik"][b], o["loglik"], rtol=1e-10)


def test_pipelined_host_path_with_missing_data_falls_back(lib):
    import os
    Xb, Lam, Rv, A, Q = _many_small_panels(1300)
    Xb[1234, 5:9, 3] = np.nan
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=3)
    os.environ["DFM_NO_PIPELINE"] = "1"
    try:
        ref = lib.em_kalman(Xb, Lam, Rv, A, Q, p=1, max_iter=3)
    finally:
        del os.environ["DFM_NO_PIPELINE"]
    for k in ("F", "Lam", "loglik"):
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-12, atol=1e-13)


def test_table4a_through_gpu(lib, panels, notebook_tables):
    """Golden Table 4(a) (Stock_Watson.ipynb): rejection rates of the Chow / QLR tests, r = 4 and 8, factors AND test
    statistics from the GPU path (dfm_estimate_factor -> dfm_instability)."""
    from scipy.stats import chi2
    import dynamic_factor_models_b200 as D
    qlr_thresh = {4: 4 * np.array([5.12, 4.09, 3.59]), 8: 8 * np.array([3.57, 2.98, 2.69])}
    for r, key in ((4, "chow_qlr_r4"), (8, "chow_qlr_r8")):
        m = D.DFMModel(panels["all_bpdata"], panels["all_inclcode"], 20, 40, 3, 224, 0, r, 1e-8, 4, 4)
        D.estimate_factor(m, computeR2=False, lib=lib)
        chow, qlr = D.instability_tests(m, 104, lib=lib)
        ok = ~np.isnan(chow)
        got = [[np.mean(chow[ok] > chi2.ppf(lv, r)), np.mean(qlr[ok] > th)] for lv, th in zip((0.99, 0.95, 0.9), qlr_thresh[r])]
        np.testing.assert_allclose(np.array(got), np.array(notebook_tables["table4"][key]), atol=1e-6)
        # lower half: quantiles of cor(yhat_full, yhat_pre) and cor(yhat_full, yhat_post), factors re-estimated on the sub-samples
        alts = [D.DFMModel(panels["all_bpdata"], panels["all_inclcode"], 20, 40, i0, i1, 0, r, 1e-8, 4, 4) for i0, i1 in ((3, 104), (105, 224))]
        cors = []
        for ma in alts:
            D.estimate_factor(ma, computeR2=False, lib=lib)
            c = D.fitted_value_correlations(m, ma, 104, lib=lib)
            cors.append(np.quantile(c[~np.isnan(c)], [0.05, 0.25, 0.50, 0.75, 0.95]))
        np.testing.assert_allclose(np.array(cors), np.array(notebook_tables["table4"]["cor_r%d" % r]), atol=2e-6)


def test_cluster_sizes_agree(lib): P.check_cluster_sizes(lib)
