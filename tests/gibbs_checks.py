"""Parity checks of dfm_gibbs against the NumPy spec tests/gibbs_oracle.py, chain for chain (the device and the spec consume the same
Philox numbers).  Each function takes a `Library` (CUDA on an H100, or the host-emulation build of the same kernel source)."""
import numpy as np

from dynamic_factor_models_b200 import DFMError
import gibbs_oracle as O
import ss_bootstrap_checks as BC
import ss_bootstrap_oracle as SBO

SEED = 20261016
PRIOR = dict(kap_lam=0.01, a_R=3.0, b_R=1.0, kap_A=0.01, nu_Q=5.0, s_Q=1.0)


def model(N=14, r=3, T=40, p=2, miss=0.1, exclude=(4,), ragged=3):
    """A standardized panel and theta^ (with P0) from a few oracle EM iterations (ss_bootstrap_checks.fitted)."""
    return BC.fitted(N=N, r=r, T=T, p=p, miss=miss, exclude=exclude, ragged=ragged)


def _inits(th, n_chain, jitter=0.05):
    """Per-chain initial parameters: theta^ with the loadings scaled by (1 + jitter c) (distinct chains, same model)."""
    L = np.stack([th["Lam"] * (1.0 + jitter * c) for c in range(n_chain)])
    rep = lambda a_: np.stack([a_] * n_chain)
    return dict(Lam=L, R=rep(th["R"]), A=rep(th["A"]), Q=rep(th["Q"]), P0=rep(th["P0"]))


def _chain_init(ini, c):
    return {n: ini[n][c] for n in ini}


def compare_chain(got, c, ref, tol=1e-8):
    assert got["status"][c] == 0
    for n in ("Lam", "R", "A", "Q", "F"):
        g, r_ = got[n][c], ref[n]
        assert (np.isnan(g) == np.isnan(r_)).all(), n
        assert np.nanmax(np.abs(g - r_)) <= tol, (n, np.nanmax(np.abs(g - r_)))
    if "X" in got and got["X"].shape[2]:
        g, r_ = got["X"][c], ref["X"][:, -got["X"].shape[2]:]
        assert (np.isnan(g) == np.isnan(r_)).all()
        assert np.nanmax(np.abs(g - r_)) <= tol, np.nanmax(np.abs(g - r_))
    assert np.max(np.abs(got["loglik"][c] - ref["loglik"]) / np.abs(ref["loglik"])) <= 1e-10


def check_chains(lib, X, th, p, n_chain=2, n_burn=2, n_keep=3, thin=1, H_fc=2, fc_rows=4, chain0=3, sweep0=5, check=None,
                 H_irf=4, tol=1e-8):
    """Every kept draw, the loglik trace and the panel draws of a call against the spec chain."""
    ini = _inits(th, n_chain)
    got = lib.gibbs(X, ini, p=p, n_chain=n_chain, chain0=chain0, sweep0=sweep0, n_burn=n_burn, n_keep=n_keep, thin=thin, seed=SEED,
                    H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, prior=PRIOR, ref=th)
    r = th["Lam"].shape[1]
    assert got["Lam"].shape == (n_chain, n_keep) + th["Lam"].shape and got["loglik"].shape == (n_chain, n_burn + n_keep * thin)
    for c in (range(n_chain) if check is None else check):
        ref = O.chain(X, _chain_init(ini, c), p, PRIOR, SEED, chain0 + c, sweep0, n_burn, n_keep, thin, H=H_fc)
        compare_chain(got, c, ref, tol)
        if H_irf:
            for j in range(n_keep):
                al = SBO.align(th["Lam"], th["R"], ref["Lam"][j], ref["R"][j], ref["A"][j], ref["Q"][j], p)
                ri = SBO.irf(al["A"], al["Q"], p, H_irf).transpose(2, 1, 0)
                assert np.max(np.abs(got["irf"][c, j] - ri)) <= 1e-7 * max(1.0, np.max(np.abs(ri))), j
    use = SBO.in_model(th["Lam"], th["R"])
    assert np.isnan(got["Lam"][:, :, ~use]).all() and np.isnan(got["R"][:, :, ~use]).all()
    assert got["Q"].shape[-2:] == (r, r)
    return got


def check_factor_step(lib, X, th, p, H_fc=2, c=7, sweep0=11):
    """From theta_c, the factor draw of the first sweep equals dfm_simulation_smoother's draw gibbs_id(c, sweep0)."""
    got = lib.gibbs(X, th, p=p, n_chain=1, chain0=c, sweep0=sweep0, n_burn=0, n_keep=1, seed=SEED, H_fc=H_fc, fc_rows=0, prior=PRIOR,
                    outputs=("F",))
    ss = lib.simulation_smoother(X, th["Lam"], th["R"], th["A"], th["Q"], p=p, P0=th["P0"], H=H_fc, n_draw=1, seed=SEED,
                                 draw0=O.gibbs_id(c, sweep0), outputs=("F",))
    assert np.max(np.abs(got["F"][0, 0] - ss["F"][0])) <= 1e-10, np.max(np.abs(got["F"][0, 0] - ss["F"][0]))


def check_continuation(lib, X, th, p, a=2, n_chain=2):
    """One call of 2a kept sweeps equals two calls of a, the second started from the first's last draw, sweep0 advanced."""
    ini = _inits(th, n_chain)
    kw = dict(p=p, n_chain=n_chain, chain0=1, n_burn=0, thin=1, seed=SEED, H_fc=1, fc_rows=2, prior=PRIOR, outputs=("Lam", "R", "A", "Q", "F", "X"))
    full = lib.gibbs(X, ini, n_keep=2 * a, sweep0=3, **kw)
    one = lib.gibbs(X, ini, n_keep=a, sweep0=3, **kw)
    last = {n: one[n][:, -1] for n in ("Lam", "R", "A", "Q")}
    last["P0"] = ini["P0"]
    two = lib.gibbs(X, last, n_keep=a, sweep0=3 + a, **kw)
    for n in ("Lam", "R", "A", "Q", "F", "X"):
        np.testing.assert_array_equal(full[n], np.concatenate([one[n], two[n]], axis=1), err_msg=n)
    np.testing.assert_array_equal(full["loglik"], np.concatenate([one["loglik"], two["loglik"]], axis=1))


def check_chain_split(lib, X, th, p, counts=(20, 50, 300), n_keep=2):
    """Calls with different n_chain and chain0 splits give identical bits for the same chain ids: a call on [0, 300) spans two
    sub-batches (264 chains each for small models on an H100), the others straddle its boundary."""
    base = _inits(th, max(counts) + 30)
    kw = dict(p=p, sweep0=2, n_burn=1, n_keep=n_keep, seed=SEED, H_fc=1, fc_rows=2, prior=PRIOR, outputs=("Lam", "R", "F", "X"))
    sub = lambda c0, n: {m: base[m][c0:c0 + n] for m in base}
    big = lib.gibbs(X, sub(0, counts[-1]), n_chain=counts[-1], chain0=0, **kw)
    for n in counts[:-1]:
        got = lib.gibbs(X, sub(0, n), n_chain=n, chain0=0, **kw)
        for m in got:
            np.testing.assert_array_equal(got[m], big[m][:n], err_msg=m)
    c0 = 250
    got = lib.gibbs(X, sub(c0, 30), n_chain=30, chain0=c0, **kw)
    for m in got:
        np.testing.assert_array_equal(got[m], big[m][c0:c0 + 30], err_msg=m)
    return big


def check_failed_chain(lib, X, th, p):
    """A chain whose E-step fails (R_i <= 0 in its init) has status 3 and NaN records; its neighbours are the chains of a call
    without it."""
    ini = _inits(th, 3)
    bad = {n: ini[n].copy() for n in ini}
    bad["R"][1, 1] = -1.0
    kw = dict(p=p, n_chain=3, n_burn=1, n_keep=2, seed=SEED, H_fc=1, fc_rows=2, prior=PRIOR, H_irf=3, ref=th)
    got = lib.gibbs(X, bad, **kw)
    ok = lib.gibbs(X, ini, **kw)
    assert got["status"][1] == 3 and got["status"][0] == 0 and got["status"][2] == 0
    for n in ("Lam", "R", "A", "Q", "irf", "F", "X", "loglik"):
        assert np.isnan(got[n][1]).all(), n
        for c in (0, 2):
            np.testing.assert_array_equal(got[n][c], ok[n][c], err_msg=n)


def check_args(lib, X, th, p):
    T, N = X.shape; r = th["Lam"].shape[1]

    def code(**kw):
        try:
            args = dict(p=p, n_chain=1, n_keep=1, prior=PRIOR, seed=SEED); args.update(kw)
            init = args.pop("init", th)
            lib.gibbs(X, init, **args)
        except DFMError as e:
            return e.code
        return 0

    assert code(n_keep=0) == 1
    assert code(thin=0) == 1
    assert code(n_burn=-1) == 1
    assert code(chain0=-1) == 1
    assert code(chain0=(1 << 16) - 1, n_chain=2) == 1
    assert code(sweep0=(1 << 24) - 1, n_keep=2) == 1
    assert code(fc_rows=T + 3, H_fc=2) == 1
    assert code(H_fc=-1) == 1
    assert code(H_irf=-1) == 1
    assert code(H_irf=3) == 1                                       # no ref
    for bad in (dict(kap_lam=0.0), dict(a_R=0.5), dict(b_R=-1.0), dict(kap_A=0.0), dict(s_Q=0.0), dict(nu_Q=1.0 - T + r),
                dict(kap_lam=np.nan)):
        pr = dict(PRIOR); pr.update(bad)
        assert code(prior=pr) == 1, bad
    assert code(init=dict(th, P0=np.eye(r * p)), p=p) == 0
    big = dict(Lam=th["Lam"], R=th["R"], A=np.zeros((r, 25 * r)), Q=th["Q"], P0=np.eye(25 * r))
    assert code(init=big, p=25) == 6                               # k = 25 r > 48
    # the handle stays usable
    assert code() == 0
