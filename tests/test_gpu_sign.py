"""GPU tests (-m gpu, H100) of the shocks identified by sign restrictions (dfm_sign_restrictions): the checks of
tests/test_emu_sign.py on the CUDA build, and Stock & Watson's Figure 7 block fitted with a plain Parametric() (no loading
restriction), shock 1 restricted by the four oil series responding + at h = 0..3, through api.sign_identified_set and
api.sign_restricted_responses."""
import numpy as np
import pytest

import parity_checks as P
import sign_checks as SC
from test_gpu_identified import OIL, figure7

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
@pytest.mark.parametrize("r", [1, 3, 8, 12])
def test_matches_spec(lib, r, p):
    lib.profile(True)
    SC.check_against_spec(lib, r, p)
    ks = set(lib.profile_report()); lib.profile(False)
    assert {"k_sr_prep", "k_irf", "k_sign_prep", "k_sign_cand", "k_sign_pick", "k_sign_rot", "k_series_resp"} <= ks, sorted(ks)


def test_failed_models(lib): SC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): SC.check_device_equals_host(lib, alloc)
def test_chunks(lib, alloc): SC.check_chunks(lib, alloc)
def test_partial_tiles(lib): SC.check_partial_tiles(lib)
def test_bounds(lib): SC.check_bounds(lib)
def test_argument_errors(lib): SC.check_args(lib)


def figure7_plain(lib, panels, iters=20):
    """hom_fac_1, 1985Q1-2014Q4, r = 8, p = 4, Parametric() without restrictions.  Returns (model, oil series in the model)."""
    import dynamic_factor_models_b200 as D
    data, incl = panels["all_bpdata"], panels["all_inclcode"]
    names = [str(s) for s in panels["all_names"]]
    calds = [tuple(x) for x in panels["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    g = P.gpu_model(data, incl, 8, i0, i1)
    D.estimate(g, D.Parametric(max_iter=iters, tol=0.0), lib=lib)
    assert g.em["status"] == 0 and g.em.get("lam_constr") is None
    used = [n for n, c in zip(names, incl) if c == 1]
    oil = [used.index(n) for n in OIL]
    return g, [i for i in oil if not np.isnan(g.lambda_est[i, 0]) and not np.isnan(g.em["R"][i])]


def _satisfied(resp, inm, shock=0, horizons=range(4)):
    """Every oil row positive in every non-NaN draw (resp (..., ns, H, n_shock))."""
    v = np.take(resp[..., shock], inm, axis=-2)[..., list(horizons)]
    ok = ~np.isnan(v).any(axis=(-2, -1))
    return bool((v[ok] > 0).all()), ok


@pytest.fixture(scope="module")
def plain(lib, panels):
    return figure7_plain(lib, panels)


def test_figure7_sign_restrictions(lib, plain, panels):
    import dynamic_factor_models_b200 as D
    g, inm = plain
    assert len(inm) >= 3, inm
    H, q = 12, (5, 16, 50, 84, 95)
    rs = [(i, 1, 1, (0, 3)) for i in inm]
    s = D.sign_identified_set(g, rs, H, n_rot=1 << 20, n_keep=4096, seed=11, q=q, lib=lib)
    assert 0 < s["n_accept"] <= 1 << 20 and s["rows"].shape == (4 * len(inm), 4)
    nk = min(s["n_accept"], 4096)
    assert s["resp"].shape == (nk, len(s["series"]), H, 1) and s["rot"].shape == (nk, 8, 8)
    sat, ok = _satisfied(s["resp"], inm)
    assert sat and ok.all()
    np.testing.assert_allclose(np.einsum("kab,kac->kbc", s["rot"], s["rot"]), np.broadcast_to(np.eye(8), (nk, 8, 8)), atol=1e-13)
    fin = np.isfinite(s["resp"][0, :, 0, 0])
    for nm in ("resp", "fevd"):
        dr = s[nm][:, fin]
        np.testing.assert_allclose(s[nm + "_bands"][:, fin], np.percentile(dr, q, axis=0), rtol=1e-13, atol=1e-14 * np.abs(dr).max())
        np.testing.assert_array_equal(s[nm + "_lo"][fin], dr.min(0))
        np.testing.assert_array_equal(s[nm + "_hi"][fin], dr.max(0))
    # (both samplers lose chains on this model after 150-230 sweeps: their A draws are not restricted to be stationary;
    # DESIGN.md 4.12)
    o = D.sign_restricted_responses(g, rs, H, n_chain=4, n_burn=40, n_keep=80, rot_per_draw=4, seed=7, q=q, lib=lib)
    assert (o["status"] == 0).all(), o["status"]
    dr = o["resp_draws"]
    assert dr.shape == (4, 80, 4, len(s["series"]), H, 1)
    sat, ok = _satisfied(dr, inm)
    assert sat
    np.testing.assert_allclose(1.0 - ok.mean(), 1.0 - o["accept_rate"], rtol=0, atol=1e-15)
    assert o["n_empty"] == int((o["accept"] == 0).sum()) and 0 < o["accept_rate"] <= 1
    for nm in ("resp", "fevd"):
        x = o[nm + "_draws"].reshape((-1,) + o[nm + "_draws"].shape[3:])[:, fin]
        ref = np.nanpercentile(x, q, axis=0)
        np.testing.assert_allclose(o[nm + "_bands"][:, fin], ref, rtol=1e-13, atol=1e-14 * np.nanmax(np.abs(ref)))
    assert np.isfinite(o["rhat"]["loglik"])
    with pytest.raises(ValueError):
        D.sign_identified_set(g, [(inm[0], 2, 1, 0)], H, n_shock=1, lib=lib)           # shock 2 > n_shock
    gc, _ = figure7(lib, panels)
    with pytest.raises(ValueError):
        D.sign_restricted_responses(gc, rs, H, n_chain=1, n_keep=1, lib=lib)           # a lam_constr_em fit


def test_posterior_chain_split(lib, plain):
    """Chains 0-1 in one call and chain 1 alone (chain0 = 1) give chain 1 the same draws, acceptances and bands' inputs."""
    import dynamic_factor_models_b200 as D
    g, inm = plain
    rs = [(i, 1, 1, (0, 3)) for i in inm]
    kw = dict(n_burn=5, n_keep=8, rot_per_draw=4, seed=3, lib=lib)
    both = D.sign_restricted_responses(g, rs, 6, n_chain=2, **kw)
    one = D.sign_restricted_responses(g, rs, 6, n_chain=1, chain0=1, **kw)
    assert (both["status"] == 0).all()
    for nm in ("resp_draws", "fevd_draws", "accept"):
        np.testing.assert_array_equal(one[nm][0], both[nm][1], err_msg=nm)
