"""CPU-only: dfm_historical_decomposition (k_sr_prep, k_hd_paths, k_hd_series) through the HOST-EMULATION build of the kernel
source (tests/emu/libdfm_emu.so) against the NumPy spec tests/history_oracle.py.  The CUDA build runs the same checks in
tests/test_gpu_history.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import history_checks as HC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.fixture
def alloc():
    keep = []

    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2, 4])
@pytest.mark.parametrize("r", [1, 8, 12])
def test_matches_spec(lib, r, p): HC.check_against_spec(lib, r, p)
def test_k49_refused(lib): HC.check_k49_refused(lib)
def test_failed_models_and_nan_series(lib): HC.check_failed_models_and_nan_series(lib)
def test_device_equals_host(lib, alloc): HC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): HC.check_chunks(lib, alloc)
def test_argument_errors(lib): HC.check_args(lib)
