"""CPU-only: the cases of tests/sampling_dispatch_checks.py on the HOST-EMULATION build of the kernel source (132 SMs), against
the NumPy specs.  The emulation build has no launch profiler, so the kernel-set assertions run only in
tests/test_gpu_sampling_dispatch.py (-m gpu)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import sampling_dispatch_checks as SD  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402

NSM = 132                              # dfm_handle::nsm of the emulation build


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.mark.parametrize("case", SD.CASES, ids=[c.id for c in SD.CASES])
def test_sampling_dispatch(lib, case):
    case.run(lib, NSM)


def test_gibbs_draw_guard_unreachable():
    """dfm_gibbs' `gibbs_draw_smem > kMaxSmem` refusal would fire only at p = 1, r >= 45, where ss_check has refused already."""
    fires = [(r, p) for r in range(1, 49) for p in range(1, 49) if r * p <= 48 and SD.gibbs_draw_smem(r, p) > SD.KMAX_SMEM]
    assert fires == [(45, 1), (46, 1), (47, 1), (48, 1)]
    for r, p in fires:
        for nsm in (66, 114, 132):
            assert not SD.ss_accepts(nsm, SD.ssb_batch(nsm, 60, 20, r, p), r, p)
    assert SD.ss_accepts(132, 1, 36, 1) and not SD.ss_accepts(132, 1, 37, 1)
