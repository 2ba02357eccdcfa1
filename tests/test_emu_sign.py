"""CPU-only: dfm_sign_restrictions (k_sr_prep, k_irf, k_sign_prep, k_sign_cand, k_sign_pick, k_sign_rot, k_series_resp) through
the HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec tests/sign_oracle.py.  The CUDA
build runs the same checks in tests/test_gpu_sign.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import sign_checks as SC  # noqa: E402
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
@pytest.mark.parametrize("r", [1, 3, 8, 12])
def test_matches_spec(lib, r, p): SC.check_against_spec(lib, r, p)
def test_failed_models(lib): SC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): SC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): SC.check_chunks(lib, alloc)
def test_partial_tiles(lib): SC.check_partial_tiles(lib)
def test_bounds(lib): SC.check_bounds(lib)
def test_argument_errors(lib): SC.check_args(lib)
