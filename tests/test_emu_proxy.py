"""CPU-only: dfm_proxy_identification (k_sr_prep, k_irf, k_iv_prep, k_iv_boot, k_iv_rot, k_series_resp) through the HOST-EMULATION
build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec tests/proxy_oracle.py.  The CUDA build runs the same
checks in tests/test_gpu_proxy.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import proxy_checks as PC  # noqa: E402
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
@pytest.mark.parametrize("r", [1, 3, 5, 8, 10, 12])
def test_matches_spec(lib, r, p): PC.check_against_spec(lib, r, p)
def test_failed_models(lib): PC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): PC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): PC.check_chunks(lib, alloc)
def test_bounds(lib): PC.check_bounds(lib)
def test_argument_errors(lib): PC.check_args(lib)
