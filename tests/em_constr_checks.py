"""Checks of dfm_em_kalman_constrained (the state-space EM under linear restrictions on the loadings) against the spec
(tests/em_constr_oracle.py), shared by the host-emulation tests (test_emu_em_constr.py) and the GPU tests
(test_gpu_em_constr.py).  Each function takes a `Library`."""
import numpy as np
import pytest

import em_constr_oracle as O
from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
from oracle import dfm_ref as R
from oracle import kalman_em as K
from oracle.dgp import simulate_panel

OUTS = ("Lam", "R", "A", "Q", "P0", "F", "PF", "loglik", "iters", "status")


def panel(N, r, T, p, miss=0.0, rep=5):
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    F0 = R.pca_score(np.nan_to_num(X), r)
    return X, K.init_from_factors(X, F0, p)


def named_and_general(r, N, rng, general=(3,), named=(0, 1)):
    """Series in `named` load e_1' only; two random rows on each series of `general`; one on series N - 2."""
    idx, H, h = [], [], []
    for i in named:
        idx += [i] * r; H.append(np.eye(r)); h.append(np.r_[1.0, np.zeros(r - 1)])
    for i in general:
        idx += [i, i]; H.append(rng.standard_normal((2, r))); h.append(rng.standard_normal(2))
    idx.append(N - 2); H.append(rng.standard_normal((1, r))); h.append(rng.standard_normal(1))
    return np.array(idx), np.vstack(H), np.concatenate(h)


def compare(got, ref, cons, par_tol=1e-8, ll_rtol=1e-10):
    """One panel's results against the spec from the same start: log-likelihood path rtol ll_rtol, Lam, R, A, Q, F within
    par_tol of max |ref| (relative for R), the restriction to 1e-12 and the log-likelihood monotone from iteration 1."""
    np.testing.assert_allclose(got["loglik"], ref["loglik"], rtol=ll_rtol)
    use = ~np.isnan(ref["R"])                                   # (series out of the model keep their R on the device)
    for n in ("A", "Q", "F"):
        np.testing.assert_allclose(got[n], ref[n], rtol=0, atol=par_tol * np.abs(ref[n]).max(), err_msg=n)
    np.testing.assert_allclose(got["Lam"][use], ref["Lam"][use], rtol=0, atol=par_tol * np.abs(ref["Lam"][use]).max())
    np.testing.assert_allclose(got["R"][use], ref["R"][use], rtol=par_tol)
    ll = got["loglik"][1:]
    assert (np.diff(ll) >= -1e-9 * np.abs(ll[:-1])).all(), np.diff(ll)
    for i, (Hi, hi) in O.by_series(cons, got["Lam"].shape[0]).items():
        if not np.isnan(got["Lam"][i, 0]):
            np.testing.assert_allclose(Hi @ got["Lam"][i], hi, rtol=0, atol=1e-12 * max(1.0, np.abs(hi).max()))


def check_vs_spec(lib, N, r, T, p, miss=0.0, iters=4, rep=5, cons=None, exclude=()):
    X, th = panel(N, r, T, p, miss, rep)
    Lam = th[0].copy()
    for i in exclude:                                          # series out of the model: their rows are ignored
        Lam[i] = np.nan
    th = (Lam,) + th[1:]
    cons = cons if cons is not None else named_and_general(r, N, np.random.default_rng(rep))
    ref = O.em_kalman(X, *th, p=p, max_iter=iters, constr=cons)
    got = lib.em_kalman(X, *th, p=p, max_iter=iters, constr=cons)
    assert got["status"] == 0 and got["iters"] == iters
    compare(got, ref, cons)
    for i in exclude:
        assert np.isnan(got["Lam"][i]).all()
    return got


def check_batch(lib, N=16, r=3, T=40, p=2):
    """A batch of 3 panels (one balanced, two with missing data) equals 3 one-panel calls, and the spec."""
    pans = [panel(N, r, T, p, miss, rep) for miss, rep in ((0.0, 21), (0.06, 22), (0.1, 23))]
    cons = named_and_general(r, N, np.random.default_rng(4))
    Xb = np.stack([x for x, _ in pans])
    th = [np.stack([t[j] for _, t in pans]) for j in range(4)]
    got = lib.em_kalman(Xb, *th, p=p, max_iter=3, constr=cons)
    for b in range(3):
        one = lib.em_kalman(Xb[b], *(t[b] for t in th), p=p, max_iter=3, constr=cons)
        for n in ("Lam", "R", "A", "Q", "F", "loglik"):
            np.testing.assert_allclose(got[n][b], one[n], rtol=1e-12, atol=1e-13, err_msg=n)
        ref = O.em_kalman(Xb[b], *(t[b] for t in th), p=p, max_iter=3, constr=cons)
        compare({n: got[n][b] for n in ("Lam", "R", "A", "Q", "F", "loglik")}, ref, cons)


def check_zero_rows_bit_identical(lib, N=24, r=3, T=40, p=1, miss=0.0):
    """n_constr = 0 is dfm_em_kalman, bit for bit (balanced p = 1: the fused path; with missing data: the general path)."""
    X, th = panel(N, r, T, p, miss)
    ref = lib.em_kalman(X, *th, p=p, max_iter=4)
    got = lib.em_kalman(X, *th, p=p, max_iter=4, constr=(np.zeros(0, np.int32), np.zeros((0, r)), np.zeros(0)))
    for n in OUTS:
        np.testing.assert_array_equal(got[n], ref[n], err_msg=n)


def check_args(lib, N=12, r=3, T=30, p=1):
    X, th = panel(N, r, T, p)
    ok = (np.array([0, 0]), np.eye(r)[:2], np.array([1.0, 0.0]))
    bad = [(np.array([N]), np.eye(r)[:1], np.array([1.0])),                       # index outside [0, N)
           (np.array([-1]), np.eye(r)[:1], np.array([1.0])),
           (np.zeros(r + 1, int), np.vstack([np.eye(r), np.ones((1, r))]), np.zeros(r + 1)),   # more than r rows
           (np.array([1]), np.array([[1.0, np.nan, 0.0]]), np.array([1.0])),      # non-finite H
           (np.array([1]), np.eye(r)[:1], np.array([np.inf])),                    # non-finite h
           (None, np.eye(r)[:1], np.array([1.0])), (np.array([1]), None, np.array([1.0])), (np.array([1]), np.eye(r)[:1], None)]
    for c in bad:
        with pytest.raises(DFMError) as ei:
            lib.em_kalman(X, *th, p=p, max_iter=2, constr=c)
        assert ei.value.code == 1, c
    for path in (2, 3):
        with pytest.raises(DFMError) as ei:
            lib.em_kalman(X, *th, p=p, max_iter=2, constr=ok, path=path)
        assert ei.value.code == 6
    assert lib.em_kalman(X, *th, p=p, max_iter=2, constr=ok, path=1)["status"] == 0


def check_dependent_rows(lib, N=14, r=3, T=40, p=1, miss=0.0):
    """Dependent rows on one series (a singular G) give the panel status 3 (DFM_ERR_NOT_PD), as the spec raises."""
    X, th = panel(N, r, T, p, miss)
    cons = (np.array([2, 2]), np.array([[1.0, 0.5, 0.0], [2.0, 1.0, 0.0]]), np.array([1.0, 2.0]))
    with pytest.raises(O.ConstraintSingular):
        O.em_kalman(X, *th, p=p, max_iter=1, constr=cons)
    assert lib.em_kalman(X, *th, p=p, max_iter=3, constr=cons)["status"] == 3


def check_mem_device(lib, alloc, N=14, r=3, T=40, p=2, miss=0.08):
    """DFM_MEM_DEVICE equals DFM_MEM_HOST bit for bit.  alloc(array) -> (address, read-back function)."""
    X, th = panel(N, r, T, p, miss)
    cons = named_and_general(r, N, np.random.default_rng(9))
    ref = lib.em_kalman(X, *th, p=p, max_iter=3, constr=cons)
    k = r * p
    ins = dict(X=to_cm(X), Lam=to_cm(th[0]), R=np.ascontiguousarray(th[1]), A=to_cm(th[2]), Q=to_cm(th[3]))
    size = dict(Lam=N * r, R=N, A=r * k, Q=r * r, P0=k * k, F=T * r, PF=T * r * r, loglik=3)
    dev = {n: alloc(a) for n, a in ins.items()}
    outs = {n: alloc(np.zeros(s)) for n, s in size.items()}
    outs.update(iters=alloc(np.zeros(1, np.int32)), status=alloc(np.zeros(1, np.int32)))
    lib.em_kalman_raw(dev["X"][0], T, N, r, p, 1, 3, 0.0, {n: dev[n][0] for n in ("Lam", "R", "A", "Q")},
                      {n: o[0] for n, o in outs.items()}, MEM_DEVICE, constr=cons)
    lib.sync()
    got = {n: o[1]() for n, o in outs.items()}
    np.testing.assert_array_equal(got["loglik"], ref["loglik"])
    np.testing.assert_array_equal(got["Lam"].reshape(r, N).T, ref["Lam"])
    np.testing.assert_array_equal(got["R"], ref["R"])
    np.testing.assert_array_equal(got["F"].reshape(r, T).T, ref["F"])
    np.testing.assert_array_equal(got["A"].reshape(k, r).T, ref["A"])
    assert int(got["status"][0]) == 0 and int(got["iters"][0]) == 3
