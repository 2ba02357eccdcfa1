"""GPU tests (-m gpu, H100) of the Gibbs sampler under restrictions on the loadings (dfm_gibbs_constrained) and of the series
responses / variance decompositions (dfm_series_responses): the checks of tests/test_emu_identified.py on the CUDA build, and
Stock & Watson's Figure 7 model (the oil series pinned to e_1) through api.identified_responses."""
import numpy as np
import pytest

import gibbs_checks as GC
import identified_checks as IC
import parity_checks as P

pytestmark = pytest.mark.gpu

OIL = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]


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
def model():
    return GC.model()


@pytest.fixture
def alloc():
    import torch
    keep = []

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
    return alloc


def test_chains_match_spec(lib, model):
    lib.profile(True)
    IC.check_chains(lib, *model, p=2, constr=IC.constr_for(model[1]))
    ks = set(lib.profile_report()); lib.profile(False)
    assert "k_gibbs_draw_constr" in ks and "k_gibbs_draw" not in ks, sorted(ks)


def test_no_rows_is_gibbs(lib, model): IC.check_no_rows_is_gibbs(lib, *model, p=2)
def test_unrestricted_series_unchanged(lib, model): IC.check_unrestricted_series(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_chain_split_invariance(lib, model): IC.check_chain_split(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_argument_errors_and_dependent_rows(lib, model): IC.check_args(lib, *model, p=2, constr=IC.constr_for(model[1]))
def test_series_responses_match_spec(lib, model, alloc): IC.check_series_responses(lib, model[1], 2, alloc)


def figure7(lib, panels, iters=20):
    """hom_fac_1, 1985Q1-2014Q4, r = 8, p = 4, the oil series' loadings pinned to e_1 in the ALS steps and the EM (as
    test_gpu_em_constr.py's Figure 7 test).  Returns (model, oil series in the model)."""
    import dynamic_factor_models_b200 as D
    data, incl = panels["all_bpdata"], panels["all_inclcode"]
    names = [str(s) for s in panels["all_names"]]
    calds = [tuple(x) for x in panels["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    r = 8
    Rm = np.eye(r); rv = np.r_[1.0, np.zeros(r - 1)]
    used = [n for n, c in zip(names, incl) if c == 1]
    g = P.gpu_model(data, incl, r, i0, i1)
    gf = D.construct_constraint(OIL, used, Rm, rv); gfl = D.construct_constraint(OIL, names, Rm, rv)
    D.estimate(g, D.Parametric(max_iter=iters, tol=0.0), lam_constr_f=gf, lam_constr_fl=gfl, lam_constr_em=gf, lib=lib)
    assert g.em["status"] == 0
    oil = [used.index(n) for n in OIL]
    return g, [i for i in oil if not np.isnan(g.em["Lam"][i, 0])]


def test_figure7_identified_responses(lib, panels):
    import dynamic_factor_models_b200 as D
    g, inm = figure7(lib, panels)
    assert len(inm) >= 3, inm
    H, q = 12, (5, 16, 50, 84, 95)
    # (both samplers lose chains on this model after 150-230 sweeps with this seed: their A draws are not restricted to be
    # stationary; DESIGN.md 4.12)
    out = D.identified_responses(g, H, shocks=1, n_chain=4, n_burn=40, n_keep=80, seed=7, q=q, lib=lib)
    assert (out["status"] == 0).all(), out["status"]
    xstd = lib.standardize(g.data[:, g.inclcode == 1][g.initperiod - 1:g.lastperiod])[2]
    e1 = np.r_[1.0, np.zeros(7)]
    for i in inm:                                         # every kept oil-series draw on its restriction
        np.testing.assert_allclose(out["Lam"][:, :, i], np.broadcast_to(e1 / xstd[i], out["Lam"].shape[:2] + (8,)), rtol=0,
                                   atol=1e-12 / xstd[i])
    si = D.series_irf(g, H, lib=lib)
    ok = ~np.isnan(si[:, 0, 0])
    np.testing.assert_allclose(out["resp"][ok, :, 0], si[ok, :, 0], rtol=1e-12, atol=1e-12 * np.nanmax(np.abs(si)))
    vd = D.variance_decomposition(g, H, lib=lib)
    np.testing.assert_array_equal(out["fevd"][..., 0], vd["fevd"][..., 0])
    for nm in ("resp", "fevd"):
        bd, dr = out[nm + "_bands"], out[nm + "_draws"]
        assert bd.shape == (len(q), len(ok), H, 1) and dr.shape == (4, 80, len(ok), H, 1)
        assert (np.diff(bd[:, ok], axis=0) >= 0).all()
        np.testing.assert_allclose(bd[:, ok], np.percentile(dr.reshape((-1,) + dr.shape[2:]), q, axis=0)[:, ok], rtol=1e-13, atol=1e-14)
    assert np.isfinite(out["rhat"]["loglik"]) and np.isfinite(out["rhat"]["resp"][ok]).all()
    for i in inm:                                         # an oil series' response to shock 1 is factor 1's own, in data units
        assert np.isfinite(out["resp_draws"][:, :, i]).all()
    with pytest.raises(ValueError):
        D.identified_responses(g, H, shocks=2, lib=lib)   # factor 2 is not named
    with pytest.raises(ValueError):
        D.gibbs(g, n_chain=1, n_keep=1, lib=lib)
