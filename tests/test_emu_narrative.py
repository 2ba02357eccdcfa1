"""CPU-only: dfm_narrative_sign_restrictions (k_narr_prep, k_narr_cand, k_narr_rot, k_narr_omega, k_narr_weight with the reused
sign kernels) and dfm_percentiles_weighted through the HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so)
against the NumPy spec tests/narrative_oracle.py.  The CUDA build runs the same checks in tests/test_gpu_narrative.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import narrative_checks as NC  # noqa: E402
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
def test_matches_spec(lib, r, p): NC.check_against_spec(lib, r, p)
def test_no_narrative_rows(lib): NC.check_no_narrative_rows(lib)
def test_kind0_probability(lib): NC.check_kind0_probability(lib)
def test_weighted_percentiles(lib): NC.check_weighted_percentiles(lib)
def test_failed_models(lib): NC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): NC.check_device_equals_host(lib, alloc)
def test_chunks(lib): NC.check_chunks(lib)
def test_bounds(lib): NC.check_bounds(lib)
def test_argument_errors(lib): NC.check_args(lib)
