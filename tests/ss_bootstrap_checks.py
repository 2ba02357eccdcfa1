"""Parity checks of dfm_ss_simulate_panels / dfm_ss_bootstrap against the NumPy spec tests/ss_bootstrap_oracle.py, replicate for
replicate (the device and the spec consume the same Philox normals).  Each function takes a `Library` (CUDA on an H100, or the
host-emulation build of the same kernel source)."""
import numpy as np

from oracle import kalman_em as K
from dynamic_factor_models_b200 import DFMError
from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm, from_cm
import simsmooth_checks as SC
import ss_bootstrap_oracle as O

SEED = 20261016


def fitted(N=14, r=3, T=40, p=2, miss=0.1, rep=9, exclude=(), ragged=0, em_iters=3):
    """A standardized panel (missing cells, a ragged edge of `ragged` rows on the first half of the series, series out of the
    model) and theta^ = a few oracle EM iterations from the PCA start, with P0."""
    X, Lam, Rv, A, Q = SC.problem(N, r, T, p, miss, rep, exclude=exclude)
    if ragged:
        X[T - ragged:, :N // 2] = np.nan
    k = r * p
    Qt = np.zeros((k, k)); Qt[:r, :r] = Q
    P0 = K.lyapunov_doubling(K.companion(A, r, p), Qt)
    em = K.em_kalman(X, Lam, Rv, A, Q, p=p, P0=P0, max_iter=em_iters)
    Lh = em["Lam"].copy()
    return X, dict(Lam=Lh, R=em["R"], A=em["A"], Q=em["Q"], P0=P0)


def check_simulate(lib, N=14, r=3, T=40, p=2, miss=0.1, exclude=(), ragged=0, n_rep=19, rep0=3, check=None, tol=1e-12, X=None, th=None):
    """Panels of one call against the spec (all replicates, or the positions in `check`): NaN pattern exact, values to tol."""
    if X is None:
        X, th = fitted(N, r, T, p, miss, exclude=exclude, ragged=ragged)
    got = lib.ss_simulate_panels(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, n_rep=n_rep, seed=SEED, rep0=rep0)
    assert got.shape == (n_rep, X.shape[0], X.shape[1])
    for b in (range(n_rep) if check is None else check):
        ref, _ = O.simulate_panel(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p, SEED, rep0 + b)
        assert (np.isnan(ref) == np.isnan(got[b])).all(), b
        ok = ~np.isnan(ref)
        assert np.max(np.abs(ref[ok] - got[b][ok])) <= tol, (b, np.max(np.abs(ref[ok] - got[b][ok])))
    use = O.in_model(th["Lam"], th["R"])
    assert np.isnan(got[:, :, ~use]).all() and np.isnan(got[:, np.isnan(X)]).all()
    return X, th, got


def compare_replicate(got, b, ref, par_tol, ll_rtol, fc_tol=None):
    al = ref["aligned"]
    assert got["status"][b] == 0 and al is not None
    assert got["iters"][b] == ref["iters"]
    for n in ("Lam", "R", "A", "Q"):
        g, r_ = got[n][b], al[n]
        assert (np.isnan(g) == np.isnan(r_)).all(), n
        assert np.nanmax(np.abs(g - r_)) <= par_tol, (n, np.nanmax(np.abs(g - r_)))
    ri = ref["irf"].transpose(2, 1, 0)                      # (shock, h, var) -> (var, h, shock)
    assert np.max(np.abs(got["irf"][b] - ri)) <= par_tol, np.max(np.abs(got["irf"][b] - ri))
    assert abs(got["loglik"][b] - ref["loglik"]) <= ll_rtol * abs(ref["loglik"]), (got["loglik"][b], ref["loglik"])
    if fc_tol is not None:
        for n in ("xhat", "xvar"):
            g, r_ = got[n][b], ref[n]
            assert (np.isnan(g) == np.isnan(r_)).all(), n
            assert np.nanmax(np.abs(g - r_)) <= fc_tol, (n, np.nanmax(np.abs(g - r_)))


def check_bootstrap(lib, X, th, p, n_rep=3, rep0=2, max_iter=3, tol=0.0, H_irf=6, H_fc=2, fc_rows=4, check=None, par_tol=1e-10,
                    ll_rtol=1e-12, fc_tol=1e-10):
    """dfm_ss_bootstrap against the spec pipeline (spec panel -> oracle EM from theta^ -> align -> IRF -> forecasts)."""
    got = lib.ss_bootstrap(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, n_rep=n_rep, seed=SEED, rep0=rep0, H_irf=H_irf,
                           H_fc=H_fc, fc_rows=fc_rows, max_iter=max_iter, tol=tol)
    r = th["Lam"].shape[1]
    assert got["irf"].shape == (n_rep, r, H_irf, r) and got["A"].shape == (n_rep, r, r * p)
    if fc_rows:
        assert got["xhat"].shape == (n_rep, fc_rows, X.shape[1])
    for b in (range(n_rep) if check is None else check):
        ref = O.replicate(X, th, p, SEED, rep0 + b, max_iter, tol, H_irf, H_fc, fc_rows)
        compare_replicate(got, b, ref, par_tol, ll_rtol, fc_tol if fc_rows else None)
    return got


def check_shard_invariance(lib, X, th, p, n_rep=21, world=8):
    """Panels of ids [0, n_rep) from one call equal the concatenation of `world` shards (dfm_shard_range), bit for bit."""
    args = (X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"])
    full = lib.ss_simulate_panels(*args, p=p, n_rep=n_rep, seed=SEED, rep0=0)
    parts = []
    for g in range(world):
        b, e = lib.shard_range(n_rep, g, world)
        if e > b:
            parts.append(lib.ss_simulate_panels(*args, p=p, n_rep=e - b, seed=SEED, rep0=b))
    np.testing.assert_array_equal(full, np.concatenate(parts))
    other = lib.ss_simulate_panels(*args, p=p, n_rep=2, seed=SEED + 1, rep0=0)
    assert not np.array_equal(np.nan_to_num(other), np.nan_to_num(full[:2]))


def check_bootstrap_shards(lib, X, th, p, n_rep=5, max_iter=2):
    """The records of ids [0, n_rep) from one dfm_ss_bootstrap call equal those of two calls on [0, 2) and [2, n_rep)."""
    kw = dict(p=p, seed=SEED, H_irf=5, H_fc=1, fc_rows=3, max_iter=max_iter)
    args = (X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"])
    full = lib.ss_bootstrap(*args, n_rep=n_rep, rep0=0, **kw)
    a = lib.ss_bootstrap(*args, n_rep=2, rep0=0, **kw)
    b = lib.ss_bootstrap(*args, n_rep=n_rep - 2, rep0=2, **kw)
    for n in full:
        np.testing.assert_array_equal(full[n], np.concatenate([a[n], b[n]]), err_msg=n)


def check_sub_batches(lib, X, th, p, n_big=300, max_iter=3, H_fc=2, fc_rows=4):
    """The replicates run in sub-batches of a size fixed by the model's shape and the device (264 for small models on an H100,
    a plan of the general path's kernels that differs from the plans of smaller batches).  A call on ids [0, n_big), which
    spans two sub-batches, gives the bits of a call on [0, 20) and of a call on [250, n_big), whose ids straddle the first
    sub-batch boundary of the big call."""
    kw = dict(p=p, seed=SEED, H_irf=6, H_fc=H_fc, fc_rows=fc_rows, max_iter=max_iter)
    args = (X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"])
    big = lib.ss_bootstrap(*args, n_rep=n_big, rep0=0, **kw)
    head = lib.ss_bootstrap(*args, n_rep=20, rep0=0, **kw)
    tail = lib.ss_bootstrap(*args, n_rep=n_big - 250, rep0=250, **kw)
    for n in big:
        np.testing.assert_array_equal(big[n][:20], head[n], err_msg=n)
        np.testing.assert_array_equal(big[n][250:], tail[n], err_msg=n)
    return big


def check_mem_device(lib, alloc, X, th, p, n_rep=9):
    """dfm_ss_simulate_panels with device memory gives what host memory gives, bit for bit.  alloc(array) -> (address,
    to_numpy()) of a device buffer."""
    T, N = X.shape; r = th["Lam"].shape[1]
    host = lib.ss_simulate_panels(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, n_rep=n_rep, seed=SEED, rep0=4)
    ins = {n: alloc(a_) for n, a_ in dict(X=to_cm(X), Lam=to_cm(th["Lam"]), R=np.ascontiguousarray(th["R"]), A=to_cm(th["A"]),
                                          Q=to_cm(th["Q"]), P0=to_cm(th["P0"])).items()}
    o = alloc(np.zeros(n_rep * T * N))
    lib.ss_simulate_panels_raw(ins["X"][0], T, N, r, p, {n: ins[n][0] for n in ("Lam", "R", "A", "Q", "P0")}, SEED, 4, n_rep, o[0], MEM_DEVICE)
    lib.sync()
    np.testing.assert_array_equal(from_cm(o[1](), T, N, n_rep), host)


def check_failed_replicate(lib, X, th, p):
    """A replicate whose EM fails (R_i <= 0 in theta^ fails the E-step) has a nonzero status and NaN records."""
    th = dict(th); th["R"] = th["R"].copy(); th["R"][1] = -1.0
    got = lib.ss_bootstrap(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, n_rep=2, seed=SEED, H_irf=4, H_fc=1, fc_rows=2,
                           max_iter=2)
    assert (got["status"] != 0).all()
    for n in ("Lam", "A", "Q", "irf", "xhat", "xvar"):
        assert np.isnan(got[n]).all(), n


def check_failed_alignment(lib, X, th, p, max_iter=3):
    """theta^ with a zero loading column: every replicate's X = (Lam*' W Lam*)^-1 Lam*' W Lam^ has a zero column, so the
    alignment fails (the spec's align() returns None) while the EM succeeds: status 3, NaN parameters, IRFs and forecasts, the
    EM's log-likelihood and iteration count as the spec's."""
    th = dict(th); th["Lam"] = th["Lam"].copy(); th["Lam"][:, -1] = 0.0
    got = lib.ss_bootstrap(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, n_rep=2, seed=SEED, rep0=1, H_irf=4, H_fc=1,
                           fc_rows=2, max_iter=max_iter)
    for b in range(2):
        ref = O.replicate(X, th, p, SEED, 1 + b, max_iter, 0.0, 4, 1, 2)
        assert ref["em"]["loglik"].size == max_iter and ref["aligned"] is None
        assert got["status"][b] == 3 and got["iters"][b] == ref["iters"]
        assert abs(got["loglik"][b] - ref["loglik"]) <= 1e-10 * abs(ref["loglik"])
        for n in ("Lam", "R", "A", "Q", "irf", "xhat", "xvar"):
            assert np.isnan(got[n][b]).all(), n


def check_args(lib, X, th, p):
    T, N = X.shape; r = th["Lam"].shape[1]

    def code(**kw):
        try:
            args = dict(p=p, n_rep=2, H_irf=4, H_fc=1, fc_rows=2, max_iter=2); args.update(kw)
            A_ = args.pop("A", th["A"]); P0 = args.pop("P0", th["P0"])
            lib.ss_bootstrap(X, th["Lam"], th["R"], A_, th["Q"], P0, **args)
        except DFMError as e:
            return e.code
        return 0

    assert code(H_irf=0) == 1
    assert code(H_irf=-3) == 1
    assert code(n_rep=0) == 1
    assert code(fc_rows=T + 2) == 1
    assert code(H_fc=-1) == 1
    assert code(max_iter=0) == 1
    assert code(rep0=-1) == 1
    assert code(p=25, A=np.zeros((r, 25 * r)), P0=np.eye(25 * r)) == 6           # k = 25 r > 48
    bufs = dict(X=to_cm(X), Lam=to_cm(th["Lam"]), R=np.ascontiguousarray(th["R"]), A=to_cm(th["A"]), Q=to_cm(th["Q"]),
                P0=to_cm(th["P0"]))
    for missing in bufs:
        addr = {n: (0 if n == missing else bufs[n].ctypes.data) for n in bufs}
        for fn in ("boot", "sim"):
            try:
                prm = {n: addr[n] for n in ("Lam", "R", "A", "Q", "P0")}
                if fn == "boot":
                    lib.ss_bootstrap_raw(addr["X"], T, N, r, p, prm, {}, 0, 1)
                else:
                    lib.ss_simulate_panels_raw(addr["X"], T, N, r, p, prm, SEED, 0, 1, bufs["X"].ctypes.data, 0)
                raise AssertionError("null %s accepted by %s" % (missing, fn))
            except DFMError as e:
                assert e.code == 1
