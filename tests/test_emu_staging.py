"""CPU-only: output staging of the single-call entry points (tests/staging_checks.py) through the HOST-EMULATION build of the
kernel source (tests/emu/libdfm_emu.so): device memory against host memory, outputs left out, and a call in a grown, used
workspace.  The CUDA build runs the same checks in tests/test_gpu_staging.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import staging_checks as S  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


def _new_lib():
    return Library(build_emu.build())


@pytest.fixture(scope="module")
def lib():
    L = _new_lib()
    yield L
    L.close()


@pytest.fixture
def alloc():
    """Emulation 'device' memory is host memory: a numpy buffer stands in for a device allocation."""
    keep = []

    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    yield alloc
    keep.clear()


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_device_equals_host(lib, alloc, name):
    S.check_device_equals_host(lib, S.CASES[name], alloc)


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_optional_outputs(lib, alloc, name):
    S.check_optional_outputs(lib, S.CASES[name], alloc)


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_grown_workspace(lib, alloc, name):
    S.check_grown_workspace(lib, _new_lib, S.CASES[name], alloc)
