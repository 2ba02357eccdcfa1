"""Parity checks of dfm_simulation_smoother against the NumPy spec tests/simsmooth_oracle.py, draw for draw (the device and
the spec consume the same Philox normals).  Each function takes a `Library` (CUDA on an H100, or the host-emulation build of
the same kernel source).  Bar: max abs difference <= 1e-10 (standardized units)."""
import numpy as np

from oracle.dgp import simulate_panel
from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST, to_cm, from_cm
from forecast_checks import _params
from simsmooth_oracle import simulation_smoother

SEED = 20261016


def compare(got, refF, refX, tol=1e-10):
    assert np.max(np.abs(got["F"] - refF)) <= tol, np.max(np.abs(got["F"] - refF))
    if "X" in got:
        assert (np.isnan(got["X"]) == np.isnan(refX)).all()
        ok = ~np.isnan(refX)
        assert np.max(np.abs(got["X"][ok] - refX[ok]), initial=0.0) <= tol, np.max(np.abs(got["X"][ok] - refX[ok]))


def problem(N=24, r=3, T=70, p=1, miss=0.0, rep=9, exclude=(), holes=(), few_obs=()):
    """A standardized panel and PCA-started parameters; holes = (t0, t1, i) blocks of NaN; few_obs = periods that observe
    only the first r - 1 series (C_t of rank < r)."""
    X, _ = simulate_panel(N, r, T, rep=rep, missing_frac=miss)
    for t0, t1, i in holes:
        X[t0:t1, i] = np.nan
    Lam, Rv, A, Q = _params(X, r, p)
    for t in few_obs:
        X[t, r - 1:] = np.nan
    for i in exclude:
        Lam[i] = np.nan
    return X, Lam, Rv, A, Q


def check_sim(lib, N=24, r=3, T=70, p=1, miss=0.0, H=0, rep=9, exclude=(), holes=(), few_obs=(), n_draw=5, draw0=0, seed=SEED,
              check_ids=None):
    """The draws of one call against the spec, draw for draw (all of them, or the positions in check_ids)."""
    X, Lam, Rv, A, Q = problem(N, r, T, p, miss, rep, exclude, holes, few_obs)
    got = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=n_draw, seed=seed, draw0=draw0)
    assert got["status"] == 0
    assert got["F"].shape == (n_draw, T + H, r) and got["X"].shape == (n_draw, T + H, N)
    pos = list(range(n_draw)) if check_ids is None else list(check_ids)
    refF, refX = simulation_smoother(X, Lam, Rv, A, Q, None, p, H, seed, [draw0 + j for j in pos])
    compare(dict(F=got["F"][pos], X=got["X"][pos]), refF, refX)
    obs = ~np.isnan(X)
    obs[:, list(exclude)] = False
    for j in range(n_draw):
        assert np.array_equal(got["X"][j, :T][obs], X[obs])                      # observed cells: the data, bitwise
        for i in exclude:
            assert np.isnan(got["X"][j, :, i]).all()
    return X, (Lam, Rv, A, Q), got


def check_block_missing(lib, H):
    """Block-missing series and a ragged edge (forecast_checks.block_missing_panel), p = 2."""
    from forecast_checks import block_missing_panel
    X = block_missing_panel()
    Lam, Rv, A, Q = _params(X, 2, 2)
    got = lib.simulation_smoother(X, Lam, Rv, A, Q, p=2, H=H, n_draw=3, seed=SEED, draw0=11)
    assert got["status"] == 0
    compare(got, *simulation_smoother(X, Lam, Rv, A, Q, None, 2, H, SEED, [11, 12, 13]))


def check_shard_invariance(lib, N=20, r=2, T=60, p=2, miss=0.1, H=4):
    """Draws [0, 100) of one call equal [0, 37) + [37, 100) of two calls, bit for bit."""
    X, Lam, Rv, A, Q = problem(N, r, T, p, miss)
    full = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=100, seed=SEED)
    a = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=37, seed=SEED, draw0=0)
    b = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=63, seed=SEED, draw0=37)
    for n in ("F", "X"):
        np.testing.assert_array_equal(full[n], np.concatenate([a[n], b[n]]))
    only_f = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=100, seed=SEED, outputs=("F",))
    np.testing.assert_array_equal(only_f["F"], full["F"])
    other = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=2, seed=SEED + 1)
    assert not np.array_equal(other["F"], full["F"][:2])


def check_mem_device(lib, alloc, N=18, r=2, T=50, p=1, H=3, n_draw=21):
    """mem = DEVICE gives what mem = HOST gives.  alloc(array) -> (address, to_numpy()) of a device buffer."""
    X, Lam, Rv, A, Q = problem(N, r, T, p, 0.05, rep=70)
    host = lib.simulation_smoother(X, Lam, Rv, A, Q, p=p, H=H, n_draw=n_draw, seed=SEED, draw0=5)
    ins = {n: alloc(a_) for n, a_ in dict(X=to_cm(X), Lam=to_cm(Lam), R=np.ascontiguousarray(Rv), A=to_cm(A), Q=to_cm(Q)).items()}
    Tp = T + H
    outs = dict(F=alloc(np.zeros(n_draw * Tp * r)), X=alloc(np.zeros(n_draw * Tp * N)))
    st = alloc(np.full(1, -1, np.int32))
    lib.simulation_smoother_raw(ins["X"][0], T, N, r, p, H, n_draw, 5, SEED, {n: ins[n][0] for n in ("Lam", "R", "A", "Q")},
                                {"F": outs["F"][0], "X": outs["X"][0], "status": st[0]}, MEM_DEVICE)
    lib.sync()
    assert st[1]()[0] == 0
    np.testing.assert_array_equal(from_cm(outs["F"][1](), Tp, r, n_draw), host["F"])
    np.testing.assert_array_equal(from_cm(outs["X"][1](), Tp, N, n_draw), host["X"])


def check_failed_estep(lib):
    """R_i <= 0 fails the E-step: status 3 and NaN draws."""
    X, Lam, Rv, A, Q = problem(12, 2, 30, 1)
    Rv = Rv.copy(); Rv[4] = -1.0
    got = lib.simulation_smoother(X, Lam, Rv, A, Q, p=1, H=2, n_draw=3, seed=SEED)
    assert got["status"] == 3
    assert np.isnan(got["F"]).all() and np.isnan(got["X"]).all()


def check_args(lib):
    X, Lam, Rv, A, Q = problem(12, 2, 30, 1)

    def code(**kw):
        try:
            args = dict(p=1, H=0, n_draw=2); args.update(kw)
            A_ = args.pop("A", A)
            lib.simulation_smoother(X, Lam, Rv, A_, Q, **args)
        except DFMError as e:
            return e.code
        return 0

    assert code(n_draw=0) == 1
    assert code(draw0=-1) == 1
    assert code(H=-1) == 1
    assert code(p=25, A=np.zeros((2, 50))) == 6                   # k = 50 > 48
    assert code(H=2, outputs=("F",)) == 0
    assert code(H=2, outputs=()) == 0
    T, N, r = X.shape[0], X.shape[1], 2
    bufs = dict(X=to_cm(X), Lam=to_cm(Lam), R=np.ascontiguousarray(Rv), A=to_cm(A), Q=to_cm(Q))
    for missing in bufs:
        addr = {n: (0 if n == missing else bufs[n].ctypes.data) for n in bufs}
        try:
            lib.simulation_smoother_raw(addr["X"], T, N, r, 1, 0, 1, 0, SEED, {n: addr[n] for n in ("Lam", "R", "A", "Q")}, {}, MEM_HOST)
            raise AssertionError("null %s accepted" % missing)
        except DFMError as e:
            assert e.code == 1
