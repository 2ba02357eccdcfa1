"""CPU-only: dfm_em_kalman_constrained (restricted measurement M-step in k_em_mstep_series and k_emb_mstep_constr) through the
HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the spec (tests/em_constr_oracle.py).  The CUDA
build runs the same checks in tests/test_gpu_em_constr.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import em_constr_checks as CC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def _host_alloc(keep):
    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


def test_missing_p2_mstep_series(lib): CC.check_vs_spec(lib, N=14, r=3, T=60, p=2, miss=0.08, iters=5)
def test_missing_p1_excluded_series(lib): CC.check_vs_spec(lib, N=14, r=3, T=50, p=1, miss=0.05, iters=4, exclude=(1, 3))
def test_balanced_r8_p1_emb(lib):
    """Balanced r = 8, p = 1, even T: the shape the fused kernels take without restrictions; with them, k_emb_mstep_constr."""
    CC.check_vs_spec(lib, N=40, r=8, T=60, p=1, iters=4)
def test_balanced_r34_mstep_series(lib):
    """r = 34 > 32: the multi-CTA contraction kernels are off, the balanced panel takes k_em_mstep_series (r = 40 exceeds the
    filter's shared memory at p = 1 on the general path, so 34 is the largest r class the test can reach with a margin)."""
    CC.check_vs_spec(lib, N=80, r=34, T=60, p=1, iters=2, rep=6)
def test_batch_equals_single_calls(lib): CC.check_batch(lib)
def test_zero_rows_bit_identical_fused_shape(lib): CC.check_zero_rows_bit_identical(lib, N=24, r=3, T=40, p=1)
def test_zero_rows_bit_identical_general(lib): CC.check_zero_rows_bit_identical(lib, N=16, r=3, T=40, p=2, miss=0.05)
def test_argument_errors(lib): CC.check_args(lib)
def test_dependent_rows_status_3(lib): CC.check_dependent_rows(lib)
def test_dependent_rows_status_3_missing(lib): CC.check_dependent_rows(lib, miss=0.05)
def test_mem_device_equals_host(lib):
    keep = []
    CC.check_mem_device(lib, _host_alloc(keep))


def test_estimate_lam_constr_em(lib):
    """api.estimate(Parametric(), lam_constr_em=...): r is divided by the block's xstd, the EM runs restricted (the named series
    load e_1 / xstd), m.em keeps the restriction, series_irf is xstd_i lam_i' irf, and parametric_bootstrap refuses the model."""
    import dynamic_factor_models_b200 as D
    from oracle.dgp import simulate_panel
    X, _ = simulate_panel(12, 2, 80, rep=3, missing_frac=0.03, standardize=False)
    X = X * np.linspace(0.5, 3.0, 12) + 1.0
    r = 2
    m = D.DFMModel(X, np.ones(12, int), 20, 40, 1, 80, 0, r, 1e-8, 2, 2)
    cons = D.construct_constraint(["a", "b"], ["a", "b"] + [str(i) for i in range(10)], np.eye(r), np.r_[1.0, 0.0])
    D.estimate(m, D.Parametric(max_iter=4, tol=0.0), lam_constr_em=cons, lib=lib)
    _, _, xstd = lib.standardize(X)
    assert m.em["status"] == 0
    np.testing.assert_array_equal(m.em["lam_constr"][2], np.asarray(cons.r) / xstd[cons.indices])
    for i in (0, 1):
        np.testing.assert_allclose(m.em["Lam"][i], np.r_[1.0, 0.0] / xstd[i], rtol=0, atol=1e-12 / xstd[i])
    si = D.series_irf(m, 5, lib=lib)
    irf = D.parametric_irf(m, 5, lib=lib)
    np.testing.assert_allclose(si, xstd[:, None, None] * np.einsum("ia,ahj->ihj", m.em["Lam"], irf), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(si[0, :, 0], irf[0, :, 0], rtol=1e-12)
    with pytest.raises(ValueError):
        D.parametric_bootstrap(m, 2, lib=lib)
    m2 = D.DFMModel(X, np.ones(12, int), 20, 40, 1, 80, 0, r, 1e-8, 2, 2)
    D.estimate(m2, D.Parametric(max_iter=4, tol=0.0), lib=lib)
    assert "lam_constr" not in m2.em
