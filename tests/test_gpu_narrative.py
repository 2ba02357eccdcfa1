"""GPU tests (-m gpu, H100) of narrative sign restrictions (dfm_narrative_sign_restrictions, dfm_percentiles_weighted): the checks
of tests/test_emu_narrative.py on the CUDA build, and Stock & Watson's Figure 7 block fitted with a plain Parametric(), shock 1
restricted by the oil series responding + at h = 0..3, plus two narrative rows at 1990Q3 (the Gulf War oil shock): shock 1 was
positive, and it was the most important contributor to the first in-model oil series' unexpected change that quarter."""
import numpy as np
import pytest

import narrative_checks as NC
import narrative_oracle as NO
import sign_oracle as SO
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
@pytest.mark.parametrize("r", [1, 3, 8, 12])
def test_matches_spec(lib, r, p):
    lib.profile(True)
    NC.check_against_spec(lib, r, p)
    ks = set(lib.profile_report()); lib.profile(False)
    assert {"k_sr_prep", "k_irf", "k_sign_prep", "k_narr_prep", "k_narr_cand", "k_sign_pick", "k_narr_rot", "k_series_resp",
            "k_narr_omega", "k_narr_weight"} <= ks, sorted(ks)


def test_no_narrative_rows(lib): NC.check_no_narrative_rows(lib)
def test_kind0_probability(lib): NC.check_kind0_probability(lib)
def test_weighted_percentiles(lib): NC.check_weighted_percentiles(lib)
def test_failed_models(lib): NC.check_failed_models(lib)
def test_device_equals_host(lib, alloc): NC.check_device_equals_host(lib, alloc)
def test_chunks(lib): NC.check_chunks(lib)
def test_bounds(lib): NC.check_bounds(lib)
def test_argument_errors(lib): NC.check_args(lib)


@pytest.fixture(scope="module")
def plain(lib, panels):
    return figure7_plain(lib, panels)


def _period(g, panels, year, quarter):
    calds = [tuple(x) for x in panels["calds"]]
    return calds.index((year, quarter)) + 1


def _check_draws(rot, eps, U, oil0, c_of, row):
    """Both narrative rows hold for every kept draw, recomputed from rot, eps and the path's u_t."""
    np.testing.assert_allclose(eps[:, row, :], np.einsum("a,nak->nk", U[row], rot[:, :, :eps.shape[2]]), rtol=1e-10, atol=1e-12)
    assert (eps[:, row, 0] > 0).all()
    for om in rot:
        Hk = NO.contributions(c_of(oil0), om, U, row, 0)
        assert np.abs(Hk[0]) > np.abs(Hk[1:]).max()


def test_figure7_narrative(lib, plain, panels):
    import dynamic_factor_models_b200 as D
    import identified_oracle as IO
    g, inm = plain
    H, q = 12, (5, 16, 50, 84, 95)
    rs = [(i, 1, 1, (0, 3)) for i in inm]
    per = _period(g, panels, 1990, 3)
    narrative = [("shock", 1, per, 1), ("most", 1, inm[0], per, 0)]
    s = D.narrative_identified_set(g, rs, narrative, H, n_rot=1 << 20, n_keep=4096, seed=11, q=q, lib=lib)
    base = D.sign_identified_set(g, rs, H, n_rot=1 << 20, n_keep=16, seed=11, q=q, lib=lib)
    nk = len(s["cand"])
    assert nk > 0, "no draw of 2^20 satisfies the narrative rows on the Figure 7 block"
    assert s["n_accept"] <= base["n_accept"]
    b = D.api._state_space_block(g, 0, lib, "t")
    e = b["em"]
    # every kept id is accepted by the sign rows alone (sign_identified_set's decision, recomputed by the spec), and the kept
    # rotation is that candidate's Omega with column 1 oriented
    rl = [tuple(int(v) for v in rw) for rw in s["rows"]]
    C = SO.row_vectors(b["Lam"], e["A"], e["Q"], b["p"], rl, H)
    Om = SO.omegas(11, 0, s["cand"], 8)
    ok, flip, _ = SO.decide(C, [j for _, _, j, _ in rl], Om)
    assert ok.all()
    np.testing.assert_allclose(s["rot"][:, :, 1:], Om[:, :, 1:], rtol=0, atol=1e-10)       # (Gram-Schmidt against numpy's QR)
    np.testing.assert_allclose(np.abs(s["rot"][:, :, 0]), np.abs(Om[:, :, 0]), rtol=0, atol=1e-10)
    _, _, F = D.api._history_rows(g, b, None, "t")
    U = NO.shocks_u(e["A"], e["Q"], F, b["p"])
    P = IO.psi(e["A"], e["Q"], b["p"], H)
    c_of = lambda i: np.einsum("a,hab->hb", b["Lam"][i], P)
    _check_draws(s["rot"], s["eps"], U, inm[0], c_of, per - g.initperiod)
    w = s["weight"]
    assert np.isfinite(w).sum() == nk - s["n_zero_omega"] and (w[np.isfinite(w)] >= 1).all()
    assert 0 < s["ess"] <= nk
    fin = np.isfinite(s["resp"][0, :, 0, 0])
    for nm in ("resp", "fevd"):
        ref = NO.weighted_percentiles(s[nm][:, fin].reshape(nk, -1), np.where(np.isfinite(w), w, 0.0), q)
        np.testing.assert_array_equal(s[nm + "_bands"][:, fin].reshape(len(q), -1), ref)
        np.testing.assert_array_equal(s[nm + "_lo"][fin], s[nm][:, fin].min(0))
    # history=True from base period 1990Q2: the contribution of shock 1 to the oil series at 1990Q3 is the H_1 of the "most"
    # row (times xstd), positive in every kept draw (the oil series responds + at h = 0 and the shock is +)
    hs = D.narrative_identified_set(g, rs, narrative, H, n_rot=1 << 20, n_keep=256, seed=11, q=q, history=True, t0=per - 1,
                                    return_draws=True, lib=lib)
    hh, row = hs["history"], per - g.initperiod
    assert hh["t0"] == per - 1 and hh["contrib_draws"].shape == (len(hs["cand"]), len(s["series"]), F.shape[0], 1)
    np.testing.assert_array_equal(hs["cand"], s["cand"][:len(hs["cand"])])
    H1 = np.array([NO.contributions(c_of(inm[0]), om, U, row, 0)[0] for om in hs["rot"]]) * b["xstd"][inm[0]]
    np.testing.assert_allclose(hh["contrib_draws"][:, inm[0], row, 0], H1, rtol=1e-9)
    assert (H1 > 0).all() and hh["contrib_bands"][0, inm[0], row, 0] > 0
    wh = np.where(np.isfinite(hs["weight"]), hs["weight"], 0.0)
    ref = NO.weighted_percentiles(hh["contrib_draws"][:, fin].reshape(len(wh), -1), wh, q)
    np.testing.assert_array_equal(hh["contrib_bands"][:, fin].reshape(len(q), -1), ref)
    o = D.narrative_restricted_responses(g, rs, narrative, H, n_chain=4, n_burn=40, n_keep=80, rot_per_draw=4, seed=7, q=q, lib=lib)
    assert (o["status"] == 0).all(), o["status"]
    dr = o["resp_draws"]
    ok = ~np.isnan(dr[..., 0, 0, 0])
    assert ok.any() and (np.isnan(o["weight"]) == ~ok).all()
    oil = np.take(dr[..., 0], inm, axis=-2)[..., :4][ok]
    assert (oil > 0).all()
    wv = o["weight"].reshape(-1)
    wf = np.where(np.isfinite(wv), wv, 0.0)
    for nm in ("resp", "fevd"):
        x = o[nm + "_draws"].reshape((-1,) + o[nm + "_draws"].shape[3:])[:, fin]
        ref = NO.weighted_percentiles(x.reshape(x.shape[0], -1), np.where(np.isnan(wv), 0.0, wf), q)
        np.testing.assert_array_equal(o[nm + "_bands"][:, fin].reshape(len(q), -1), ref)
    gc, _ = figure7(lib, panels)
    with pytest.raises(ValueError):
        D.narrative_restricted_responses(gc, rs, narrative, H, n_chain=1, n_keep=1, lib=lib)     # a lam_constr_em fit
    with pytest.raises(ValueError):
        D.narrative_identified_set(g, rs, [("shock", 1, g.initperiod, 1)], H, lib=lib)           # a period before initperiod + p
