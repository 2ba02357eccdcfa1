"""CPU-only: dfm_kalman_smooth (smoothing / nowcasting / forecasting at fixed parameters) through the HOST-EMULATION
build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec.  The CUDA build runs the same checks in
tests/test_gpu_forecast.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import forecast_checks as FC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def _host_alloc(keep):
    """Emulation 'device' memory is host memory: a numpy buffer stands in for a device allocation."""
    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
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
    FC.check_kalman_smooth_mem_device(lib, _host_alloc(keep))
