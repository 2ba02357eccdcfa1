"""GPU tests (-m gpu, H100) of the non-parametric dispatch branches: every case of tests/np_dispatch_checks.py against the
oracle, with the kernels each call launched and did not launch asserted from the launch profiler."""
import pytest

import dispatch_checks as DC
import np_dispatch_checks as NP

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


@pytest.mark.parametrize("case", NP.CASES, ids=[c.id for c in NP.CASES])
def test_np_dispatch(lib, case):
    log = DC.KernelLog(lib, methods=NP.METHODS)
    case.run(log)
    log.check(case.kernels)
