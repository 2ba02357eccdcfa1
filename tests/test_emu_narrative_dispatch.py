"""CPU-only: the cases of tests/narrative_dispatch_checks.py (narrative sign restrictions and weighted percentiles at their size
edges) on the HOST-EMULATION build of the kernel source (132 SMs), against the NumPy spec.  The emulation build has no launch
profiler, so the kernel-set assertions run only in tests/test_gpu_narrative_dispatch.py (-m gpu), which also runs the cases of
GPU_ONLY (2^20 simulations per kept slot)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import narrative_dispatch_checks as ND  # noqa: E402
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


CASES = [c for c in ND.CASES if c.id not in ND.GPU_ONLY]


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_narrative_dispatch(lib, alloc, case):
    case.run(lib, NSM, alloc)
