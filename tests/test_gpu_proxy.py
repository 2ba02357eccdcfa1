"""GPU tests (-m gpu, H100) of the proxy (external instrument) identification (dfm_proxy_identification): the checks of
tests/test_emu_proxy.py on the CUDA build, and Stock & Watson's Figure 7 block (plain Parametric() fit, and the oil-named fit) with
a synthetic instrument built from the fit's own smoothed innovations plus seeded noise, unavailable in its first rows."""
import copy

import numpy as np
import pytest

import proxy_checks as PC
import proxy_oracle as PO
from test_gpu_identified import figure7
from test_gpu_sign import figure7_plain

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


@pytest.fixture
def alloc():
    import torch
    keep = []

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    return alloc


@pytest.mark.parametrize("p", [1, 2, 4])
@pytest.mark.parametrize("r", [1, 3, 5, 8, 10, 12])
def test_matches_spec(lib, r, p):
    lib.profile(True)
    PC.check_against_spec(lib, r, p)
    ks = set(lib.profile_report()); lib.profile(False)
    assert {"k_sr_prep", "k_irf", "k_iv_prep", "k_iv_boot", "k_iv_rot", "k_series_resp"} <= ks, sorted(ks)


def test_failed_models(lib): PC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): PC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): PC.check_chunks(lib, alloc)
def test_bounds(lib): PC.check_bounds(lib)
def test_argument_errors(lib): PC.check_args(lib)


@pytest.fixture(scope="module")
def plain(lib, panels):
    return figure7_plain(lib, panels)


def _instrument(g, lib, seed=5, lead=10):
    """omega_0' u_t of the fit's smoothed innovations plus N(0, 0.5^2) noise, NaN in the first `lead` rows."""
    import dynamic_factor_models_b200 as D
    b = D.api._state_space_block(g, 0, lib, "t")
    e = b["em"]
    _, _, F = D.api._history_rows(g, b, None, "t")
    eta = PO.innovations(e["A"], F, b["p"])
    u = np.linalg.solve(np.linalg.cholesky(e["Q"]), np.nan_to_num(eta).T).T
    z = u @ (np.arange(1.0, 9.0) / np.linalg.norm(np.arange(1.0, 9.0))) + 0.5 * np.random.default_rng(seed).standard_normal(len(u))
    z[:lead] = np.nan
    return z, b, F


def _rotated(g, Km):
    """A copy of g with the factors normalised as f -> K f (m.em rotated; the smoothed path follows)."""
    import identified_oracle as IO
    e = g.em
    r = e["Q"].shape[0]; p = e["A"].shape[1] // r
    Lk, Ak, Qk = IO.rotate(e["Lam"], e["A"], e["Q"], Km, p)
    Kb = np.kron(np.eye(p), Km)
    g2 = copy.copy(g)
    g2.em = dict(e, Lam=Lk, A=Ak, Q=Qk, P0=Kb @ e["P0"] @ Kb.T)
    return g2


def test_figure7_proxy(lib, plain, panels):
    import dynamic_factor_models_b200 as D
    g, inm = plain
    H, q, nb = 12, (5, 16, 50, 84, 95), 512
    z, b, F = _instrument(g, lib)
    z2 = z + 0.3 * np.random.default_rng(9).standard_normal(len(z))
    i0 = inm[0]
    o = D.proxy_identified_responses(g, {"a": z, "b": z2}, i0, H, n_boot=nb, block=4, q=4, seed=3, q_bands=q, return_draws=True, lib=lib)
    assert (o["status"] == 0).all() and o["names"] == ["a", "b"]
    e = b["em"]
    Z = np.column_stack([z, z2])
    ref = PO.identify(b["Lam"], e["R"], e["A"], e["Q"], F, Z, b["p"], H, i0, q=4, block=4, n_boot=nb, seed=3, scale=b["xstd"])
    tol = lambda x: 1e-9 * max(1.0, np.nanmax(np.abs(x)))
    for nm, got, exp in (("resp", o["resp"], ref["resp"][:, 0]), ("fevd", o["fevd"], ref["fevd"][:, 0]),
                         ("resp_draws", o["resp_draws"], ref["resp"][:, 1:]), ("fevd_draws", o["fevd_draws"], ref["fevd"][:, 1:])):
        exp = np.moveaxis(exp, 0, -1)
        assert (np.isnan(got) == np.isnan(exp)).all(), nm
        assert np.nanmax(np.abs(got - exp)) <= tol(exp), nm
    for nm, key in (("reliability", "reliability"), ("first_stage_F", "fs_F"), ("first_stage_pi", "fs_pi")):
        np.testing.assert_allclose(o[nm], ref[key], rtol=1e-9, err_msg=nm)
    np.testing.assert_allclose(o["eps"], ref["eps"].T, rtol=1e-9, atol=1e-12)
    np.testing.assert_array_equal(o["resp_unit"][i0, 0], [1.0, 1.0])
    assert o["first_stage_F"].min() > 10 and 0.5 < o["shock_corr"][0, 1] <= 1.0 + 1e-12
    # the bands are numpy's percentiles of the returned records
    fin = np.isfinite(o["resp"][:, 0, 0])
    for nm in ("resp", "resp_unit", "fevd"):
        exp = np.percentile(o[nm + "_draws"][:, fin], q, axis=0)
        np.testing.assert_allclose(o[nm + "_bands"][:, fin], exp, rtol=1e-12, atol=1e-14 * np.abs(exp).max(), err_msg=nm)
    # invariance: the same call on a rotated copy of m.em
    Km = np.eye(8) + 0.3 * np.random.default_rng(4).standard_normal((8, 8))
    o2 = D.proxy_identified_responses(_rotated(g, Km), {"a": z, "b": z2}, i0, H, n_boot=nb, block=4, q=4, seed=3, q_bands=q, lib=lib)
    for nm in ("resp", "resp_unit", "fevd", "eps", "reliability", "first_stage_F", "resp_bands", "fevd_bands"):
        np.testing.assert_allclose(o2[nm], o[nm], rtol=1e-6, atol=1e-9 * np.nanmax(np.abs(o[nm])), err_msg=nm)
    # the Gibbs variant at the GPU test's sizes
    r = D.proxy_restricted_responses(g, z, i0, H, n_chain=4, n_burn=40, n_keep=80, boot_per_draw=1, block=4, seed=7, q_bands=q, lib=lib)
    assert (r["status"] == 0).all() and (r["proxy_status"] == 0).all()
    for nm in ("resp", "resp_unit", "fevd"):
        assert np.isfinite(r[nm + "_bands"][:, fin]).all(), nm
    assert np.isfinite(r["rhat"]["loglik"])
    # the oil-named fit: accepted by the point call, refused by the sampler
    gc, _ = figure7(lib, panels)
    zc, _, _ = _instrument(gc, lib)
    oc = D.proxy_identified_responses(gc, zc, i0, H, n_boot=64, lib=lib)
    assert (oc["status"] == 0).all() and oc["block"] == round(len(zc) ** (1 / 3))
    with pytest.raises(ValueError):
        D.proxy_restricted_responses(gc, zc, i0, H, n_chain=1, n_keep=1, lib=lib)
