"""GPU tests (-m gpu, H100) of the output staging of the single-call entry points (tests/staging_checks.py): device memory
(torch CUDA tensors) against host memory, outputs left out, and a call in a grown, used workspace."""
import numpy as np
import pytest

import staging_checks as S

pytestmark = pytest.mark.gpu


def _new_lib():
    from dynamic_factor_models_b200 import Library
    return Library()


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L = _new_lib()
    assert L.path.endswith("libdfm_b200.so")
    yield L
    L.close()


@pytest.fixture
def alloc():
    import torch
    keep = []

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    yield alloc
    torch.cuda.synchronize()
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
