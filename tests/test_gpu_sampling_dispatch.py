"""GPU tests (-m gpu, H100) of the sampling entry points at their size edges: every case of tests/sampling_dispatch_checks.py
against the NumPy specs, with the kernels each call launched and did not launch asserted from the launch profiler."""
import pytest

import sampling_dispatch_checks as SD

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


@pytest.mark.parametrize("case", SD.CASES, ids=[c.id for c in SD.CASES])
def test_sampling_dispatch(lib, nsm, case):
    log = SD.KernelLog(lib, methods=SD.METHODS)
    case.run(log, nsm)
    log.check(case.kernels)
