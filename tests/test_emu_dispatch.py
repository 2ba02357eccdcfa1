"""CPU-only: the dispatch cases of tests/dispatch_checks.py on the HOST-EMULATION build of the kernel source, against the
oracle.  This keeps the index and algebra logic of those branches under the CPU tier; the emulation build has no launch
profiler, so the kernel-set assertions run only in tests/test_gpu_dispatch.py (-m gpu)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import dispatch_checks as DC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.mark.parametrize("case", DC.CASES, ids=[c.id for c in DC.CASES])
def test_dispatch(lib, case):
    case.run(lib)
