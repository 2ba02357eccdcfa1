"""CPU-only: dfm_news through the HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec
tests/news_oracle.py.  The CUDA build runs the same checks in tests/test_gpu_news.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import news_checks as NC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def _host_alloc(keep):
    """Emulation 'device' memory is host memory: a numpy buffer stands in for a device allocation."""
    def alloc(a):
        buf = np.array(a, copy=True)
        keep.append(buf)
        return buf.ctypes.data, (lambda: buf.copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("miss", [0.0, 0.15])
@pytest.mark.parametrize("H", [0, 3])
def test_news_matches_spec(lib, p, miss, H): NC.check_news(lib, p=p, miss=miss, H=H)
def test_excluded_series(lib): NC.check_news(lib, p=2, miss=0.05, H=4, exclude=(0, 7))
@pytest.mark.parametrize("H", [0, 8])
def test_block_missing_ragged_edge(lib, H): NC.check_block_missing(lib, H)
def test_long_balanced_frozen_runs(lib): NC.check_news(lib, N=30, r=3, T=300, p=2, miss=0.0, H=2, news_rows=3,
                                                       targets=[(0, 299), (5, 298), (9, 150), (3, 300), (4, 301)])
def test_many_series_and_window_rows(lib): NC.check_news(lib, N=150, r=2, T=60, p=1, miss=0.05, H=2, news_rows=11,
                                                         targets=[(t % 150, 49 + t) for t in range(13)])
def test_special_targets(lib): NC.check_special_targets(lib)
def test_no_news(lib): NC.check_no_news(lib)
def test_largest_w(lib): NC.check_largest_w(lib)
def test_batch_equals_single(lib): NC.check_batch_equals_single(lib)
def test_inconsistent_pair_in_batch(lib): NC.check_inconsistent_pair(lib)
def test_failed_estep(lib): NC.check_failed_estep(lib)
def test_argument_errors(lib): NC.check_args(lib)


def test_mem_device_equals_host(lib):
    keep = []
    NC.check_mem_device(lib, _host_alloc(keep))
