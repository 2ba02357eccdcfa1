"""GPU tests (-m gpu, H100) of dfm_news: the news decomposition against the NumPy spec (tests/news_oracle.py) on synthetic
panels, a release step of the C1 model (hom_fac_1 at its Parametric estimates) through api.news, a 16-pair C2 batch, and
a long panel whose E-step runs as a thread-block cluster."""
import numpy as np
import pytest

import parity_checks as P
import news_checks as NC
from news_oracle import news as news_spec

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


def _torch_alloc(keep):
    import torch

    def alloc(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr(), (lambda: t.cpu().numpy().copy())
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
    NC.check_mem_device(lib, _torch_alloc(keep))


def test_few_panels_cluster_path(lib):
    """One long panel: k_em_filter_smooth runs as a thread-block cluster, with frozen runs in the scan."""
    NC.check_news(lib, N=160, r=12, T=700, p=1, miss=0.0, H=2, rep=5, news_rows=2,
                  targets=[(0, 699), (17, 698), (40, 700), (3, 701), (100, 650)])


def test_c2_batch(lib):
    """16 C2-shaped pairs (N = 200, r = 8, T = 500), ~30 % of the series released in each of the last two rows: every pair's
    new_est is dfm_kalman_smooth's xhat on its new vintage, and two pairs match the spec."""
    B, N, r, T, H, nr = 16, 200, 8, 500, 2, 2
    Xn = lib.simulate_panels(0, B, N, r, T, 20261016)
    F0 = lib.estimate_factor(Xn, r, max_iter=1)["F"]
    Lam, Rv, A, Q = lib.em_init_from_factors(Xn, F0, 1)
    rng = np.random.default_rng(3)
    Xo = Xn.copy()
    Xo[:, T - nr:, :][rng.random((B, nr, N)) < 0.3] = np.nan
    tg = [(q, T - 2 + q) for q in range(4)]
    got = lib.news(Xo, Xn, Lam, Rv, A, Q, p=1, H=H, targets=tg, news_rows=nr)
    assert (got["status"] == 0).all()
    ks = lib.kalman_smooth(Xn, Lam, Rv, A, Q, p=1, H=H, outputs=("xhat",))
    ko = lib.kalman_smooth(Xo, Lam, Rv, A, Q, p=1, H=H, outputs=("xhat",))
    for q, (i, t) in enumerate(tg):
        np.testing.assert_allclose(got["new_est"][:, q], ks["xhat"][:, t, i], rtol=0, atol=1e-9)
        np.testing.assert_allclose(got["old_est"][:, q], ko["xhat"][:, t, i], rtol=0, atol=1e-9)
    for j in (0, 11):
        NC.compare({n: got[n][j] for n in ("old_est", "new_est", "news", "weight", "contrib")},
                   news_spec(Xo[j], Xn[j], Lam[j], Rv[j], A[j], Q[j], None, 1, H, tg, nr))


def test_c1_release_step(lib, panels):
    """C1: Parametric (r = 8, p = 4) on hom_fac_1 with the last two rows of a third of the series hidden, then api.news
    against the full data: targets one series at the last in-sample row and at T+1, H = 2.  Checked against the spec and,
    in data units, against the identity by_series.sum(1) + revision_effect = new - old and dfm_kalman_smooth on the new
    vintage -- also with a few old cells revised."""
    import dynamic_factor_models_b200 as D
    data, incl = panels["all_bpdata"], panels["all_inclcode"]
    i0, i1, H = 3, 224, 2
    cols = np.flatnonzero(incl == 1)
    hidden = cols[::3]
    old = data.copy(); old[i1 - 2:i1, hidden] = np.nan
    m = P.gpu_model(old, incl, 8, i0, i1)
    D.estimate(m, D.Parametric(max_iter=5, tol=0.0), lib=lib)
    out_model = np.isnan(m.lambda_est[:, 0])
    cand = [j for j in range(len(cols)) if not out_model[j] and np.isnan(data[i1 - 1, cols[j]])]
    c = int(cols[cand[0]] if cand else cols[1])
    targets = [(c, i1), (c, i1 + 1)]
    e, r, p = m.em, 8, 4
    Lam = np.where(out_model[:, None], np.nan, e["Lam"])
    Xold = old[:, cols][i0 - 1:i1]; Xnew = data[:, cols][i0 - 1:i1]
    Xs, mu, sd = lib.standardize(Xold)
    Xs[:, out_model] = np.nan

    def std_new(raw):
        xn = np.where(np.isnan(Xs), (raw - mu) / sd, Xs)
        xn[:, out_model] = np.nan
        return xn

    T = Xs.shape[0]; j = int(np.nonzero(cols == c)[0][0])
    for revise in (False, True):
        new_raw = data.copy()
        if revise:                                                              # a few old cells revised
            for cc in cols[1:12:3]:
                new_raw[i1 - 6, cc] += 0.1 * np.nanstd(data[:, cc])
        res = D.news(m, new_raw, targets, H=H, lib=lib)
        Xn_raw = new_raw[:, cols][i0 - 1:i1]
        Xrev = np.where(~np.isnan(Xs) & (Xn_raw != Xold), (Xn_raw - mu) / sd, Xs)
        Xrev[:, out_model] = np.nan
        Xn = np.where(np.isnan(Xrev), std_new(Xn_raw), Xrev)
        Xn[:, out_model] = np.nan
        tot = res["by_series"].sum(1) + res["revision_effect"]
        np.testing.assert_allclose(tot, res["new"] - res["old"], rtol=1e-10, atol=1e-10 * np.abs(res["new"]).max())
        ks = lib.kalman_smooth(Xn, Lam, e["R"], e["A"], e["Q"], p=p, P0=e["P0"], H=H, outputs=("xhat",))
        np.testing.assert_allclose(res["new"], mu[j] + sd[j] * ks["xhat"][[t - i0 for _, t in targets], j], rtol=1e-10)
        fc = D.forecast(m, H, lib=lib)
        np.testing.assert_allclose(res["old"], fc["xhat"][[t - i0 for _, t in targets], j], rtol=1e-10)
        if revise:
            assert np.abs(res["revision_effect"]).max() > 0
        else:
            assert (res["revision_effect"] == 0).all()
        nr = len(res["periods"])
        tg = [(j, t - i0) for _, t in targets]
        ref = news_spec(Xrev, Xn, Lam, e["R"], e["A"], e["Q"], e["P0"], p, H, tg, nr)
        assert ref["status"] == 0
        np.testing.assert_allclose(res["contributions"] / sd[j], np.transpose(ref["contrib"], (2, 0, 1)), rtol=0, atol=1e-9)
        w = np.transpose(ref["weight"], (2, 0, 1)) * sd[j] / sd[None, None, :]
        np.testing.assert_allclose(res["weights"], w, rtol=1e-8, atol=1e-9)
        assert res["news"].shape == (nr, len(cols)) and res["by_series"].shape == (2, len(cols))
        assert nr == 2
