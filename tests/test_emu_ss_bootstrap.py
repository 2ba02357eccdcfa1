"""CPU-only: dfm_ss_simulate_panels and dfm_ss_bootstrap (k_ss_simulate, k_ss_sim_project, k_ss_align) through the
HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec, replicate for replicate.  The CUDA
build runs the same checks in tests/test_gpu_ss_bootstrap.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import ss_bootstrap_checks as BC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.fixture(scope="module")
def model():
    return BC.fitted(N=14, r=3, T=40, p=2, miss=0.1, exclude=(4,), ragged=3)


def _host_alloc(keep):
    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2, 3])
def test_simulate_matches_spec(lib, p): BC.check_simulate(lib, r=3, p=p, miss=0.1)
def test_simulate_missing_ragged_excluded(lib): BC.check_simulate(lib, N=70, r=5, T=45, p=2, miss=0.2, exclude=(1, 66), ragged=4,
                                                                  n_rep=35, check=(0, 15, 16, 31, 32, 34))
def test_simulate_balanced_r9(lib): BC.check_simulate(lib, N=20, r=9, T=36, p=1, miss=0.0, n_rep=17, check=(0, 16))
def test_shard_invariance(lib, model): BC.check_shard_invariance(lib, *model, p=2)
def test_mem_device_equals_host(lib, model):
    keep = []
    BC.check_mem_device(lib, _host_alloc(keep), *model, p=2)


def test_bootstrap_p2_missing_ragged_excluded(lib, model): BC.check_bootstrap(lib, *model, p=2, n_rep=3, H_fc=2, fc_rows=6)
def test_bootstrap_r5_p1_missing(lib):
    X, th = BC.fitted(N=18, r=5, T=30, p=1, miss=0.05)
    BC.check_bootstrap(lib, X, th, 1, n_rep=2, max_iter=2, H_irf=3, H_fc=0, fc_rows=3)
def test_bootstrap_balanced_fused(lib):
    """A balanced p = 1 model with even T, the shape of dfm_em_kalman's fused path (the emulation build has no launch profiler:
    tests/test_gpu_ss_bootstrap.py asserts the path from the profile on the GPU)."""
    X, th = BC.fitted(N=16, r=2, T=24, p=1, miss=0.0)
    BC.check_bootstrap(lib, X, th, 1, n_rep=2, max_iter=3, H_irf=4, H_fc=2, fc_rows=2)
def test_bootstrap_shards(lib, model): BC.check_bootstrap_shards(lib, *model, p=2)
def test_sub_batches_bit_identical(lib, model): BC.check_sub_batches(lib, *model, p=2, max_iter=2)
def test_failed_alignment(lib, model): BC.check_failed_alignment(lib, *model, p=2)
def test_simulate_r48_shared_memory(lib):
    """r = 48, p = 1: the largest state the simulator takes (the Cholesky kernel's shared memory within the default 48 KB)."""
    BC.check_simulate(lib, N=60, r=48, T=60, p=1, miss=0.0, n_rep=9, check=(0, 8))


def test_replicate_driver(lib, model):
    """replicate.ss_bootstrap (one rank): the records and IRFs of one dfm_ss_bootstrap call on the model's block, rearranged."""
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200 import replicate
    from dynamic_factor_models_b200.api import _state_space_block
    X, th = model
    T, N = X.shape
    m = D.DFMModel(X, np.ones(N, int), 10, 10, 1, T, 0, 3, 1e-8, 2, 2)
    m.lambda_est = th["Lam"]
    m.em = dict(th)
    irfs, bands, rec = replicate.ss_bootstrap(lib, m, 3, H_irf=4, H_fc=1, fc_rows=2, max_iter=2, seed=BC.SEED)
    b = _state_space_block(m, 1, lib, "test")
    got = lib.ss_bootstrap(b["Xs"], b["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=2, n_rep=3, seed=BC.SEED, H_irf=4, H_fc=1, fc_rows=2,
                           max_iter=2)
    np.testing.assert_array_equal(irfs, got["irf"])
    nirf = 3 * 4 * 3
    np.testing.assert_array_equal(rec[:, nirf], got["loglik"])
    np.testing.assert_array_equal(rec[:, nirf + 1], got["iters"])
    np.testing.assert_array_equal(rec[:, nirf + 2], got["status"])
    np.testing.assert_array_equal(rec[:, nirf + 3:], got["xhat"].reshape(3, -1))
    assert set(bands) == set(replicate.BAND_PERCENTILES) and bands[50].shape == (3, 4, 3)
    np.testing.assert_allclose(bands[50], np.percentile(got["irf"], 50, axis=0), rtol=1e-13, atol=1e-15)
def test_failed_replicate(lib, model): BC.check_failed_replicate(lib, *model, p=2)
def test_argument_errors(lib, model): BC.check_args(lib, *model, p=2)
