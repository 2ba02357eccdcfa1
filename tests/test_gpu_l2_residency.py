"""GPU tests (-m gpu, H100) of the L2 residency plan of the TMA kernels k_em_fused2 / k_als_fused2: how much of a panel a
CTA keeps in L2 depends on how many CTAs are active in its round, and a cache hint must never change a result.  A batch
of two full rounds plus a tail, with panels that converge at different iterations (so that the rounds drift apart), has
to give every panel bit for bit what the same panel gives alone (one CTA, every series block kept), and the same on a
second call."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, R, T, SEED = 200, 8, 500, 20260922
SAMPLE = (0, 5, 263, 264, 400, -7, -1)          # first and second round, round boundaries, the tail


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
def batch(lib):
    """2 x (resident CTAs) + 7 C2-shaped panels with their starting factors and EM parameters."""
    import torch
    grid = 2 * torch.cuda.get_device_properties(0).multi_processor_count          # two CTAs per SM
    B = 2 * grid + 7
    Xb = lib.simulate_panels(0, B, N, R, T, SEED)
    F0 = lib.estimate_factor(Xb, R, max_iter=1)["F"]
    return Xb, F0, lib.em_init_from_factors(Xb, F0, 1)


def _same(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), f"{what}: {k} differs"


def test_em_batch_equals_single_panels(lib, batch):
    Xb, _, (Lam, Rv, A, Q) = batch
    kw = dict(p=1, max_iter=60, tol=1e-7, want_PF=False)
    got = lib.em_kalman(Xb, Lam, Rv, A, Q, **kw)
    assert (got["status"] == 0).all()
    assert len(np.unique(got["iters"])) > 1                 # panels finish at different iterations: the rounds drift
    _same(got, lib.em_kalman(Xb, Lam, Rv, A, Q, **kw), "repeated batch call")
    for b in SAMPLE:
        one = lib.em_kalman(Xb[b], Lam[b], Rv[b], A[b], Q[b], **kw)
        _same({k: one[k] for k in ("Lam", "R", "A", "Q", "F", "loglik")}, {k: got[k][b] for k in ("Lam", "R", "A", "Q", "F", "loglik")},
              f"panel {b}")
        assert one["iters"] == got["iters"][b] and one["status"] == got["status"][b]


def test_als_batch_equals_single_panels(lib, batch):
    Xb, F0, _ = batch
    kw = dict(tol=1e-10, max_iter=40, compute_r2=False)
    got = lib.estimate_factor(Xb, R, F_init=F0, **kw)
    its = np.array([s["iters"] for s in got["stats"]])
    again = lib.estimate_factor(Xb, R, F_init=F0, **kw)
    _same({k: got[k] for k in ("F", "Lam")}, {k: again[k] for k in ("F", "Lam")}, "repeated batch call")
    for b in SAMPLE:
        one = lib.estimate_factor(Xb[b], R, F_init=F0[b], **kw)
        _same({k: one[k] for k in ("F", "Lam")}, {k: got[k][b] for k in ("F", "Lam")}, f"panel {b}")
        assert one["stats"]["iters"] == its[b] and one["stats"]["ssr"] == got["stats"][b]["ssr"]
