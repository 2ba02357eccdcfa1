"""CPU-only: the cases of tests/em_constr_dispatch_checks.py (dfm_em_kalman_constrained at the sizes and edges it accepts) on
the HOST-EMULATION build of the kernel source (132 SMs), against the NumPy spec.  The emulation build has no launch profiler,
so the kernel-set assertions run only in tests/test_gpu_em_constr_dispatch.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import em_constr_dispatch_checks as ECD  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402

NSM = 132                              # dfm_handle::nsm of the emulation build


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


@pytest.mark.parametrize("case", ECD.CASES, ids=[c.id for c in ECD.CASES])
def test_em_constr_dispatch(lib, alloc, case):
    case.run(lib, NSM, alloc)
