"""GPU tests (-m gpu, H100) of the fused EM kernels in the regimes of their covariance chain (tests/fused_chain_checks.py):
every case against the oracle with the kernel each call launched asserted from the launch profiler, the stage geometry
of k_em_fused2 / k_als_fused2 at the 172-period box, and batches with more panels than resident CTAs that mix fast,
slow and never-frozen chains on the same CTA."""
import pytest

import dispatch_checks as DC
import fused_chain_checks as FC

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


@pytest.mark.parametrize("case", FC.CASES, ids=[c.id for c in FC.CASES])
def test_fused_chain(lib, case):
    log = DC.KernelLog(lib)
    FC.run_case(log, case)
    log.check(FC.KERNELS[case.path])


@pytest.mark.parametrize("geom", FC.GEOM_EM, ids=["T%s_N%d_r%d" % g for g in FC.GEOM_EM])
def test_geometry_em(lib, geom):
    log = DC.KernelLog(lib)
    FC.check_geom_em(log, *geom)
    log.check(FC.F2)


@pytest.mark.parametrize("geom", FC.GEOM_ALS, ids=["T%s_N%d_r%d" % g for g in FC.GEOM_ALS])
def test_geometry_als(lib, geom):
    log = DC.KernelLog(lib)
    FC.check_geom_als(log, *geom)
    log.check(FC.ALS_KERNELS)


def test_past_tmax(lib):
    log = DC.KernelLog(lib)
    FC.check_past_tmax(log)
    log.check(FC.F1)


def test_mixed_batch_fused2(lib, nsm):
    # k_em_fused2: __launch_bounds__(256, 2) and more than a third of the SM's shared memory per CTA: two CTAs per SM
    smem = FC.fused2_smem_bytes(FC.MIX["T"], FC.MIX["N"], FC.MIX["r"])
    assert 2 * (smem + 1024) <= 228 * 1024 < 3 * (smem + 1024)
    log = DC.KernelLog(lib)
    FC.check_mixed_batch(log, 3, 2 * nsm)
    log.check(FC.F2)


def test_mixed_batch_fused(lib, nsm):
    per_sm = FC.fused_resident_per_sm(FC.MIX["T"], FC.MIX["N"], FC.MIX["r"])
    assert per_sm == FC.G["F1_MINB"]
    log = DC.KernelLog(lib)
    FC.check_mixed_batch(log, 2, per_sm * nsm)
    log.check(FC.F1)
