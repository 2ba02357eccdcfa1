"""CPU-only: dfm_simulation_smoother through the HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against
the NumPy spec, draw for draw.  The CUDA build runs the same checks in tests/test_gpu_simsmooth.py (-m gpu)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import simsmooth_checks as SC  # noqa: E402
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
def test_draws_match_spec(lib, p, miss, H): SC.check_sim(lib, p=p, miss=miss, H=H)
def test_period_with_fewer_than_r_series(lib): SC.check_sim(lib, r=3, p=2, miss=0.05, H=2, few_obs=(10, 11, 40))
def test_excluded_series(lib): SC.check_sim(lib, p=2, miss=0.05, H=4, exclude=(2, 7))
@pytest.mark.parametrize("H", [0, 8])
def test_block_missing_ragged_edge(lib, H): SC.check_block_missing(lib, H)
def test_long_balanced_frozen_runs(lib): SC.check_sim(lib, N=30, r=3, T=300, p=2, miss=0.0, H=8, n_draw=3)
def test_draws_not_a_multiple_of_the_tile(lib): SC.check_sim(lib, N=10, r=2, T=40, p=1, miss=0.1, H=2, n_draw=37, draw0=1000,
                                                             check_ids=(0, 15, 16, 36))
def test_shard_invariance(lib): SC.check_shard_invariance(lib)
def test_failed_estep(lib): SC.check_failed_estep(lib)
def test_argument_errors(lib): SC.check_args(lib)


def test_mem_device_equals_host(lib):
    keep = []
    SC.check_mem_device(lib, _host_alloc(keep))
