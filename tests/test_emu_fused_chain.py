"""CPU-only: the chain planner of tests/fused_chain_checks.py against the oracle's filter, and every case of its tables on
the HOST-EMULATION build of the fused kernels against the oracle.  The emulation runs the kernels' serial logic (the
explicit/frozen split, ring vs global scratch, the likelihood branches, the scans); the warp-parallel parts and the
kernel-set assertions run in tests/test_gpu_fused_chain.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import fused_chain_checks as FC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def test_geometry():
    """The ring holds 12 / 15 / 22 / 31 / 50 / 88 / 195 / 687 explicit steps for r = 8 .. 1 at the 172-period stage, and
    the two-stage likelihood takes up to 20 (r = 8) and 34 (r = 7) explicit periods."""
    assert [FC.nexs(r) for r in range(8, 0, -1)] == [12, 15, 22, 31, 50, 88, 195, 687]
    for r, top in ((8, 20), (7, 34)):
        fits = [nE for nE in range(1, 200) if 2 * nE * r <= (FC.G["BND"] * r + r * r) - (FC.gparts(r) + 1) * r * r]
        assert max(fits) == top
    assert (FC.GROUPS3, FC.GROUPS2) == (28, 16)


@pytest.mark.parametrize("case", FC.CASES, ids=[c.id for c in FC.CASES])
def test_plan(case):
    """Each case reaches its branches at iteration 0, with the margin, and the oracle's filter freezes where the planner
    says (for the cases that have the margin)."""
    m = FC.plan_case(case)
    if case.model.get("margin", FC.MARGIN) >= FC.MARGIN:
        assert m.plan.margin >= FC.MARGIN
        assert FC.oracle_freeze(m.X, m.Lam, m.R, m.A, m.Q, m.P0) == m.plan.nE
    if case.path == 3:
        assert m.X.shape[0] % 2 == 0


def test_plan_table_covers_backward_branches():
    plans = [FC.plan_case(c).plan for c in FC.CASES]
    assert any(p.frozen and p.tb == -1 for p in plans)                  # smoothed chain not converged by lo
    assert any(p.tb > p.lo for p in plans)                              # closed-form moment sums over [lo, tb)
    assert any(p.levels3 == 5 and p.Lc3 == 1 for p in plans)            # n = 28: all five Kogge-Stone levels, Lc = 1
    assert any(p.frozen and p.n < 42 for p in plans)


@pytest.mark.parametrize("shape", FC.EXISTING_SHAPES, ids=["N%d_r%d_T%d" % s for s in FC.EXISTING_SHAPES])
def test_existing_shapes_freeze_early(shape):
    """The parity tests' fused-path shapes freeze after 5..8 steps at every EM iteration: none of them reaches the
    regimes of CASES, which is why this module exists."""
    assert all(5 <= nE <= 8 for nE in FC.existing_shape_nE(*shape))


def test_mixed_batch_models():
    for m, w in zip(FC.mixed_models(), FC.MIX_WANTS):
        assert FC.WANTS[w][0](m.plan), (w, m.plan[:13])
    assert FC.fused_resident_per_sm(FC.MIX["T"], FC.MIX["N"], FC.MIX["r"]) == FC.G["F1_MINB"]


@pytest.mark.parametrize("case", FC.CASES, ids=[c.id for c in FC.CASES])
def test_fused_chain(lib, case):
    FC.run_case(lib, case)


@pytest.mark.parametrize("geom", FC.GEOM_EM, ids=["T%s_N%d_r%d" % g for g in FC.GEOM_EM])
def test_geometry_em(lib, geom):
    FC.check_geom_em(lib, *geom)


@pytest.mark.parametrize("geom", FC.GEOM_ALS, ids=["T%s_N%d_r%d" % g for g in FC.GEOM_ALS])
def test_geometry_als(lib, geom):
    FC.check_geom_als(lib, *geom)


def test_past_tmax(lib):
    FC.check_past_tmax(lib)
