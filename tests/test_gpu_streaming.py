"""GPU tests (-m gpu, H100) of the streaming host path of dfm_em_kalman: host buffers and more panels than k_em_fused2
keeps resident.  The cases and checks are in tests/streaming_checks.py; every check asserts from the launch counter that
its calls streamed.  Each case is built inside its test and runs once."""
import pytest

import streaming_checks as S

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


def _ids(cases):
    return [c.id for c in cases]


@pytest.mark.parametrize("case", S.CASES, ids=_ids(S.CASES))
def test_equals_monolithic(lib, case):
    S.check_equals_monolithic(lib, case)


@pytest.mark.parametrize("case", S.CASES, ids=_ids(S.CASES))
def test_vs_oracle(lib, case):
    S.check_vs_oracle(lib, case)


_P0 = S.P0_CASES + [S.BY_ID["persistent"], S.BY_ID["caller_p0"]]


@pytest.mark.parametrize("case", _P0, ids=_ids(_P0))
def test_p0(lib, case):
    S.check_p0(lib, case)


def test_batch_edges(lib):
    S.check_batch_edges(lib)


def test_null_outputs(lib):
    S.check_null_outputs(lib)


def test_handle_reuse(lib):
    S.check_handle_reuse(lib)


@pytest.mark.parametrize("where", sorted(S.FALLBACK_PLACEMENTS))
def test_fallback(lib, where):
    S.check_fallback(lib, where)


def test_fallback_refused_on_path3(lib):
    S.check_fallback_refused(lib)


@pytest.mark.parametrize("value", (0.0, -0.5))
def test_failed_panel(lib, value):
    S.check_failed_panel(lib, value)
