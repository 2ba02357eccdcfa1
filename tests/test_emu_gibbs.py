"""CPU-only: dfm_gibbs (k_sim_gains over chains, k_gibbs_paths, k_gibbs_stats, k_gibbs_draw, k_sim_project per chain) through the
HOST-EMULATION build of the kernel source (tests/emu/libdfm_emu.so) against the NumPy spec tests/gibbs_oracle.py, chain for
chain.  The CUDA build runs the same checks in tests/test_gpu_gibbs.py (-m gpu)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import gibbs_checks as GC  # noqa: E402
from dynamic_factor_models_b200 import Library  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


@pytest.fixture(scope="module")
def model():
    return GC.model()


def test_chains_p2_missing_ragged_excluded(lib, model): GC.check_chains(lib, *model, p=2, n_burn=2, n_keep=3)
def test_chains_balanced_p1(lib):
    X, th = GC.model(N=14, r=3, T=40, p=1, miss=0.0, exclude=(), ragged=0)
    GC.check_chains(lib, X, th, 1, n_burn=1, n_keep=2, thin=2, H_fc=0, fc_rows=3)
def test_factor_step_is_the_simulation_smoother(lib, model): GC.check_factor_step(lib, *model, p=2)
def test_continuation(lib, model): GC.check_continuation(lib, *model, p=2)
def test_chain_split_invariance(lib, model): GC.check_chain_split(lib, *model, p=2)
def test_failed_chain(lib, model): GC.check_failed_chain(lib, *model, p=2)
def test_argument_errors(lib, model): GC.check_args(lib, *model, p=2)
