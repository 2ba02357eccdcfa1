"""CPU-only: the cases of tests/identified_dispatch_checks.py on the HOST-EMULATION build of the kernel source (132 SMs), against
the NumPy specs, and the enumerations showing two shared-memory refusals cannot fire.  The emulation build has no launch
profiler, so the kernel-set assertions run only in tests/test_gpu_identified_dispatch.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import identified_dispatch_checks as ID  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402

NSM = 132                              # dfm_handle::nsm of the emulation build


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.fixture
def alloc():
    keep = []

    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


@pytest.mark.parametrize("case", ID.CASES, ids=[c.id for c in ID.CASES])
def test_identified_dispatch(lib, alloc, case):
    case.run(lib, NSM, alloc)


def test_gibbs_draw_constr_guard_unreachable():
    """dfm_gibbs_constrained's `smDc > kMaxSmem` refusal: over every (r, p) dfm_gibbs accepts (k <= 48, ss_check at the sub-batch
    size, for a few SM counts and panel sizes) the largest k_gibbs_draw_constr plan is 162 640 B at (36, 1), under 225 280 B."""
    acc = {(r, p) for r in range(1, 49) for p in range(1, 49) if r * p <= 48
           for nsm in (66, 114, 132) for T, N in ((60, 20), (200, 1300)) if ID.gibbs_accepts(nsm, T, N, r, p)}
    assert (36, 1) in acc and (37, 1) not in acc and (12, 4) in acc
    worst = max(acc, key=lambda rp: ID.gibbs_draw_constr_smem(*rp))
    assert worst == (36, 1) and ID.gibbs_draw_constr_smem(36, 1) == 162640 <= ID.KMAX_SMEM
    assert ID.gibbs_draw_constr_smem(12, 4) == 84784


def test_series_responses_r_guard_unreachable():
    """dfm_series_responses' "r too large" refusal: (sm0 + r r) 8 over every r <= 64 and n_shock <= r is at most 164 864 B (at
    r = n_shock = 64), under 225 280 B."""
    need = {(r, ns): ID.sr_smem0(r, ns) + r * r * 8 for r in range(1, 65) for ns in range(1, r + 1)}
    worst = max(need, key=need.get)
    assert worst == (64, 64) and need[worst] == 164864 <= ID.KMAX_SMEM
    assert all(ID.sr_accepts(r, ns) for r, ns in need)
