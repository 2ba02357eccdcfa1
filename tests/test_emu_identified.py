"""CPU-only: dfm_gibbs_constrained (k_gibbs_draw_constr) and dfm_series_responses (k_sr_prep, k_irf, k_series_resp) through the
HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec tests/identified_oracle.py.  The CUDA
build runs the same checks in tests/test_gpu_identified.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import gibbs_checks as GC  # noqa: E402
import identified_checks as IC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.fixture(scope="module")
def model():
    return GC.model()


@pytest.fixture
def alloc():
    keep = []

    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


def test_chains_match_spec(lib, model): IC.check_chains(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_no_rows_is_gibbs(lib, model): IC.check_no_rows_is_gibbs(lib, *model, p=2)
def test_unrestricted_series_unchanged(lib, model): IC.check_unrestricted_series(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_chain_split_invariance(lib, model): IC.check_chain_split(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_argument_errors_and_dependent_rows(lib, model): IC.check_args(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_series_responses_match_spec(lib, model, alloc): IC.check_series_responses(lib, model[1], 2, alloc)
