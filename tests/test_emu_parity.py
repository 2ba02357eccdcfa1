"""CPU-only: run the parity checks against the HOST-EMULATION build of the kernel source
(tests/emu/libdfm_emu.so = the same .cu/.cuh files compiled by g++ with one logical thread per
block).  This validates kernel index/algebra logic and the C-ABI host orchestration without a GPU;
the real CUDA parity tests are tests/test_gpu_parity.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import parity_checks as P  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def test_standardize(lib): P.check_standardize(lib)
def test_pca(lib): P.check_pca(lib)
def test_pca_subspace(lib): P.check_pca(lib, r=5, sizes=((150, 90), (80, 130)))     # min(T,N) > 64 -> subspace iteration
def test_estimate_factor_same_init(lib): P.check_estimate_factor_same_init(lib)
def test_estimate_factor_c1(lib, panels): P.check_estimate_factor_c1(lib, panels)
def test_constraint(lib, panels): P.check_constraint(lib, panels)
def test_full_nonparametric_c1(lib, panels): P.check_full_nonparametric_c1(lib, panels)
def test_var_irf(lib): P.check_var_irf(lib)
def test_simulate_panels(lib): P.check_simulate_panels(lib)
def test_simulate_panels_statistics(lib): P.check_simulate_panels_statistics(lib)
def test_bootstrap_panels(lib, panels): P.check_bootstrap_panels(lib, panels)
def test_percentiles(lib): P.check_percentiles(lib)
def test_var_missing_rows(lib): P.check_var_missing_rows(lib)
def test_cluster_sizes_call_shape(lib): P.check_cluster_sizes(lib, N=40, r=4, T=120)      # (no clusters under emulation: checks the call path)
def test_fit_correlation(lib, panels): P.check_fit_correlation(lib, panels)
def test_instability_edges(lib): P.check_instability_edges(lib)
def test_instability_few_series(lib, panels): P.check_instability(lib, panels, r=4, series=[5, 60])
def test_em_p1_balanced(lib): P.check_em(lib, p=1, miss=0.0)
def test_em_p2_missing(lib): P.check_em(lib, p=2, miss=0.12)
def test_em_convergence_rule(lib): P.check_em_convergence_rule(lib)
def test_em_p2_long_balanced_frozen(lib): P.check_em(lib, N=30, r=3, T=300, p=2, miss=0.0, iters=3, path=1)
def test_em_block_missing_frozen(lib): P.check_em_block_missing(lib)
def test_em_r12_long_run(lib): P.check_em(lib, N=50, r=12, T=420, p=1, miss=0.0, iters=3, path=1)      # run scan: 2 row blocks of the state
def test_em_p4_balanced_long_run(lib): P.check_em(lib, N=40, r=8, T=330, p=4, miss=0.0, iters=2, path=1)   # companion state k = 32
def test_em_r20_balanced(lib): P.check_em(lib, N=120, r=20, T=300, p=1, miss=0.0, iters=2, path=1)       # three DMMA column blocks
def test_em_r28_balanced(lib): P.check_em(lib, N=90, r=28, T=300, p=1, miss=0.0, iters=2, path=1)        # four column blocks, 51 KB M-step tile
def test_em_batch(lib): P.check_em_batch(lib)
def test_als_batch(lib): P.check_als_batch(lib)
def test_als_balanced_fused(lib): P.check_als_balanced(lib)
def test_als_balanced_fused_r8(lib): P.check_als_balanced(lib, N=48, r=8, T=120, B=2)
def test_parametric_c1(lib, panels): P.check_parametric_c1(lib, panels, iters=2)
def test_nile_published_general(lib): P.check_nile_published(lib, path=1)
def test_nile_published_fused(lib): P.check_nile_published(lib, path=2)
def test_nile_published_fused2(lib): P.check_nile_published(lib, path=3)


# ---- fused per-panel EM kernel (path=2): same source under emulation (DMMA loops have a plain twin)
def test_fused_em_r3(lib): P.check_em(lib, p=1, miss=0.0, path=2)
def test_fused_em_r8(lib): P.check_em(lib, N=40, r=8, T=90, p=1, miss=0.0, path=2, iters=5)
def test_fused_em_r1(lib): P.check_em(lib, N=12, r=1, T=50, p=1, miss=0.0, path=2, iters=4)
def test_fused_em_convergence_rule(lib): P.check_em_convergence_rule(lib, path=2)
def test_fused_em_batch(lib): P.check_em_batch_balanced(lib, path=2)
def test_fused_rejects_missing(lib):
    import numpy as np
    from dynamic_factor_models_b200 import DFMError
    with pytest.raises(DFMError):
        P.check_em(lib, p=1, miss=0.1, path=2)
    P.check_em(lib, p=1, miss=0.1, path=0)       # auto falls back to the general path


# ---- TMA-fed fused kernel (path=3): emulation exercises its serial logic + 32-group scan + ring-scratch indexing
def test_fused2_em_r3(lib): P.check_em(lib, p=1, miss=0.0, path=3)
def test_fused2_em_r8(lib): P.check_em(lib, N=40, r=8, T=90, p=1, miss=0.0, path=3, iters=5)
def test_fused2_em_r1(lib): P.check_em(lib, N=12, r=1, T=50, p=1, miss=0.0, path=3, iters=4)
def test_fused2_em_convergence_rule(lib): P.check_em_convergence_rule(lib, path=3)
def test_fused2_em_batch(lib): P.check_em_batch_balanced(lib, path=3)


@pytest.mark.parametrize("vset", ["A", "B"])
def test_table5_through_kernel_source(lib, panels, notebook_tables, vset):
    """Golden Table 5 (Stock_Watson.ipynb:1250-1261) reproduced through the PRODUCT code path (kernel source under
    host emulation): estimate!() on the C1 panel, a small VAR on observed series with leading missing values,
    canonical correlations of levels and of VAR residuals.  Same check as tests/test_oracle_golden.py does for the
    oracle."""
    import dynamic_factor_models_b200 as D
    from test_oracle_golden import TABLE5_VARS, _canonical_correlations
    names = [str(n) for n in panels["all_names"]]
    g = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 8)
    D.estimate(g, lib=lib)
    cols = [names.index(v) for v in TABLE5_VARS[vset]]
    X = panels["all_bpdata"][:, cols]
    fv = g.factor_var_model
    v = D.VARModel(X, fv.nlag, fv.withconst, fv.initperiod, fv.lastperiod)
    D.estimate_var(v, lib=lib)
    gold = notebook_tables["table5"][vset]
    ok = ~np.isnan(np.column_stack([X, g.factor])).any(1)
    np.testing.assert_allclose(_canonical_correlations(X[ok], g.factor[ok]), gold["level"], rtol=5e-5, atol=5e-7)
    ok = ~np.isnan(np.column_stack([v.resid, fv.resid])).any(1)
    np.testing.assert_allclose(_canonical_correlations(v.resid[ok], fv.resid[ok]), gold["resid"], rtol=5e-5, atol=5e-7)


@pytest.mark.parametrize("N,r,T", [(19, 5, 62), (33, 2, 44), (27, 7, 150), (50, 6, 36)])
def test_fused2_em_ragged_shapes(lib, N, r, T):
    """Shapes that are not multiples of the 8-series / 172-period stage geometry or of the scan chunking, and the
    template instantiations the other tests do not touch (r = 2, 5, 6, 7)."""
    P.check_em(lib, N=N, r=r, T=T, p=1, miss=0.0, path=3, iters=4)


def test_amengual_watson_table2C_corner(lib, panels, notebook_tables):
    """estimate_factor_numbers through the C ABI (device residuals from dfm_estimate_loading_ex): the 3 x 3 corner of
    golden Table 2C (Stock_Watson.ipynb:669-683); the full table runs in the -m gpu tier."""
    import dynamic_factor_models_b200 as D
    g = P.gpu_model(panels["all_bpdata"], panels["all_inclcode"], 1)
    out = D.estimate_factor_numbers(g, 3, lib=lib)
    gold = np.array(notebook_tables["table2C"])[:3, 1:4]
    mask = ~np.isnan(gold)
    assert (np.isnan(out["aw_icp"]) == np.isnan(gold)).all()
    np.testing.assert_allclose(out["aw_icp"][mask], gold[mask], atol=6e-4)
