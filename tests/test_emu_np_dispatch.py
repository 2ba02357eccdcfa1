"""CPU-only: the non-parametric dispatch cases of tests/np_dispatch_checks.py on the HOST-EMULATION build of the kernel
source, against the oracle.  The emulation build refuses the launches the H100 would refuse (grid, block and shared-memory
limits) but has no launch profiler, so the kernel-set assertions run only in tests/test_gpu_np_dispatch.py (-m gpu)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import np_dispatch_checks as NP  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.mark.parametrize("case", NP.CASES, ids=[c.id for c in NP.CASES])
def test_np_dispatch(lib, case):
    case.run(lib)
