"""GPU tests (-m gpu, H100) of the narrative sign restrictions and the weighted percentiles at their size edges: every case of
tests/narrative_dispatch_checks.py against the NumPy spec, with the kernels each call launched and did not launch asserted from
the launch profiler."""
import numpy as np
import pytest

import narrative_dispatch_checks as ND

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from dynamic_factor_models_b200 import Library
    L = Library()
    assert L.path.endswith("libdfm_b200.so")
    yield L
    L.close()


@pytest.fixture(scope="module")
def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


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


@pytest.mark.parametrize("case", ND.CASES, ids=[c.id for c in ND.CASES])
def test_narrative_dispatch(lib, nsm, alloc, case):
    log = ND.KernelLog(lib, methods=ND.METHODS)
    case.run(log, nsm, alloc)
    log.check(case.kernels)
