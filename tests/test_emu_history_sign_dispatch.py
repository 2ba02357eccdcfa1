"""CPU-only: the cases of tests/history_sign_dispatch_checks.py (historical decompositions and sign restrictions at their size
edges) on the HOST-EMULATION build of the kernel source (132 SMs), against the NumPy specs.  The emulation build has no launch
profiler, so the kernel-set assertions run only in tests/test_gpu_history_sign_dispatch.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import history_sign_dispatch_checks as HS  # noqa: E402
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


@pytest.mark.parametrize("case", HS.CASES, ids=[c.id for c in HS.CASES])
def test_history_sign_dispatch(lib, alloc, case):
    case.run(lib, NSM, alloc)
