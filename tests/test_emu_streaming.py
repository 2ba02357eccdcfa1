"""CPU-only rehearsal of tests/streaming_checks.py.  The host-emulation build has no streaming host path, so nothing here
tests it; what runs is every case of the table, cut to its first panels, on the emulated k_em_fused2 by the
upload-then-compute path against the oracle.  That shows the inputs are valid (the persistent transition matrices, the
mixed-quality starts and their spread of stopping iterations, the caller's P0, the panel that fails), that k_lyapunov's
P0 solves the Lyapunov equation, and that the oracle side of every GPU check runs.  The streaming path itself is tested
in tests/test_gpu_streaming.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import streaming_checks as S  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def test_batches_exceed_every_resident_grid():
    """The batch of every case is larger than 132 SMs x the CTAs per SM that shared memory and threads allow."""
    for c in S.CASES + S.P0_CASES:
        x = S.build(c, 8)
        T, N = x.X.shape[1:]
        r = x.Lam.shape[-1]
        assert S.FC.fused2_shape_ok(T, N, r) and c.B > 132 * 2 and c.B >= S.stream_batch(T, N, r), c.id
    assert S.stream_batch(346, 40, 8) == 132 * 2 + 37


def test_persistent_radii():
    x = S.build(S.BY_ID["persistent"], 8)
    rho = [np.abs(np.linalg.eigvals(a)).max() for a in x.A]
    np.testing.assert_allclose(rho, [0.98, 0.999] * 4, rtol=1e-12)
    errs = [S.lyapunov_error(x, S.K.lyapunov_doubling(x.A[b], x.Q[b]), b)[0] for b in range(8)]
    assert max(errs[0::2]) < 1e-12 and min(errs[1::2]) > 1e-6           # at 0.999 twelve doublings truncate visibly


@pytest.mark.parametrize("case", S.CASES + S.P0_CASES, ids=[c.id for c in S.CASES + S.P0_CASES])
def test_case_rehearsal(lib, case):
    S.check_rehearsal(lib, case)


@pytest.mark.parametrize("value", (0.0, -0.5))
def test_failed_panel_rehearsal(lib, value):
    S.check_rehearsal_failed_panel(lib, value)
