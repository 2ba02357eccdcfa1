"""Checks of the streaming host path of dfm_em_kalman (em_streaming in dfm_api.cu, DESIGN.md section 4.5): host buffers
and more panels than k_em_fused2 keeps resident at once.  One launch starts before any panel is on the device, a copy
stream uploads 32-panel chunks with a "landed" flag each, the kernel computes P0 and pre-fills its log-likelihood rows
itself, and the host ships 128-panel result chunks while the kernel runs.  None of that exists in the host-emulation
build, so the checks that drive it run on the H100 only (tests/test_gpu_streaming.py); tests/test_emu_streaming.py
rehearses the inputs of CASES and the oracle side of the checks on the emulated kernels.

The reference of a streaming call is the same call with DFM_NO_PIPELINE=1 (upload, then k_lyapunov, k_fill,
k_em_scan_fused and the EM kernel): the same kernel on the same inputs, so every output has to agree bit for bit.  The
oracle and scipy's Lyapunov solver are the independent references.  Every check asserts from the handle's launch counter
that the call it means to test did stream: a streaming call launches the EM kernel, k_unpack_psf when PF is asked for
and k_em_scan_fused when some panel ended with status 3, and nothing else."""
import collections
import contextlib
import os

import numpy as np

from oracle import dfm_ref as R, kalman_em as K
from oracle.dgp import simulate_panel
import fused_chain_checks as FC
import parity_checks as P

OUTPUTS = ("F", "Lam", "R", "A", "Q", "P0", "PF", "loglik", "iters", "status")
SMALL = dict(N=16, r=2, T=40)                    # the shape of the batch-edge, reuse, fallback and failed-panel checks
EMU_PANELS = 24                                  # panels of each case the emulation rehearsal runs


@contextlib.contextmanager
def no_pipeline():
    """The upload-then-compute host path (the library reads the variable at every call)."""
    old = os.environ.get("DFM_NO_PIPELINE")
    os.environ["DFM_NO_PIPELINE"] = "1"
    try:
        yield
    finally:
        if old is None:
            del os.environ["DFM_NO_PIPELINE"]
        else:
            os.environ["DFM_NO_PIPELINE"] = old


def stream_batch(T, N, r):
    """A batch no H100 keeps resident: 37 panels more than 132 SMs hold when only shared memory (228 KB per SM, 1 KB
    reserved per CTA) and the 2048 threads per SM limit the CTAs of k_em_fused2.  Registers can only lower the count."""
    per_sm = min(2048 // FC.G["F2_THREADS"], (228 * 1024) // (FC.fused2_smem_bytes(T, N, r) + 1024))
    return 132 * per_sm + 37


# ------------------------------------------------------------------------------------------------------ the inputs
Inputs = collections.namedtuple("Inputs", "X Lam R A Q P0 opts")


def _fitted_starts(Xb, r, seed, nbase=8):
    """Cheap, valid (not optimal) starts: each panel gets the fitted parameters of one of the first nbase panels."""
    base = [K.init_from_factors(Xb[b], R.pca_score(Xb[b], r), 1) for b in range(nbase)]
    pick = np.random.default_rng(seed).integers(0, nbase, len(Xb))
    return [np.stack([base[i][j] for i in pick]) for j in range(4)]


def dgp_inputs(B, N, r, T, seed, **opts):
    Xb = np.stack([simulate_panel(N, r, T, rep=seed + b)[0] for b in range(B)])
    Lam, Rv, A, Q = _fitted_starts(Xb, r, seed)
    return Inputs(Xb, Lam, Rv, A, Q, None, dict(dict(max_iter=4, tol=0.0), **opts))


def persistent_inputs(B, seed, N=24, r=4, T=120, radii=(0.98, 0.999)):
    """Panels drawn from state-space models whose transition matrix has spectral radius 0.98 (even panels) or 0.999 (odd
    panels), started at the models' own parameters: P0 is far from Q, and at 0.999 twelve doublings have not converged."""
    models = []
    for j in range(8):
        a = np.linspace(radii[j % 2], 0.5, r)
        models.append(FC.model_params(r, N, 40.0, a, np.geomspace(1.0, 0.4, r), seed + j))
    Xb = np.stack([FC.simulate(*models[b % 8], T, seed + 100 + b) for b in range(B)])
    Lam, Rv, A, Q = [np.stack([models[b % 8][j] for b in range(B)]) for j in range(4)]
    return Inputs(Xb, Lam, Rv, A, Q, None, dict(max_iter=4, tol=0.0))


def early_stop_inputs(B, seed, N=16, r=2, T=40):
    """Starts of mixed quality: the fitted parameters of another panel with loadings shrunk towards zero by a factor that
    cycles over the batch, so that the panels meet tol = 1e-4 after different numbers of iterations."""
    x = dgp_inputs(B, N, r, T, seed, max_iter=30, tol=1e-4)
    shrink = np.array([1.0, 0.9, 0.7, 0.5, 0.3, 0.15, 0.05])[np.arange(B) % 7]
    return x._replace(Lam=x.Lam * shrink[:, None, None])


def caller_p0_inputs(B, seed):
    """The r8_two_chunks panels with a P0 of the caller's that is not the Lyapunov solution and differs from panel to panel
    and from seed to seed (what an earlier call left in the workspace is never the right P0), stopping early: the kernel
    then has to pre-fill the log-likelihood rows although it computes no P0."""
    x = dgp_inputs(B, 40, 8, 346, seed, max_iter=12, tol=1e-3)
    scale = 1.5 + np.random.default_rng(seed).uniform(size=B)
    return x._replace(P0=scale[:, None, None] * np.eye(8))


def head(x, n):
    """The first n panels of the inputs."""
    return Inputs(*[None if a is None else a[:n] for a in x[:6]], x.opts)


Case = collections.namedtuple("Case", "id build B")
CASES = [
    # r = 1, N % 8 = 5
    Case("r1_ragged", lambda s, B: dgp_inputs(B, 13, 1, 50, s), stream_batch(50, 13, 1)),
    # odd template, one full period chunk + a 106-period tail chunk, N % 8 = 5
    Case("r5_ragged_long", lambda s, B: dgp_inputs(B, 37, 5, 278, s), stream_batch(278, 37, 5)),
    # the R == 8 branches at a small N, two full period chunks + a 2-period tail
    Case("r8_two_chunks", lambda s, B: dgp_inputs(B, 40, 8, 346, s), stream_batch(346, 40, 8)),
    Case("persistent", lambda s, B: persistent_inputs(B, s), stream_batch(120, 24, 4)),
    Case("early_stop", lambda s, B: early_stop_inputs(B, s), 1500),
    Case("caller_p0", lambda s, B: caller_p0_inputs(B, s), stream_batch(346, 40, 8)),
]
# the in-kernel P0 of every template: one EM iteration, so the call is little more than P0 and one E-step
P0_CASES = [Case("p0_r%d" % r, (lambda r_: lambda s, B: dgp_inputs(B, 16, r_, 40, s, max_iter=1))(r), stream_batch(40, 16, r))
            for r in range(1, 9)]
BY_ID = {c.id: c for c in CASES + P0_CASES}
SEED = 4200


def build(case, B=None, seed=SEED):
    return case.build(seed, case.B if B is None else B)


# ------------------------------------------------------------------------------------------------------ the calls
def run(lib, x, want_PF=True, **kw):
    """em_kalman on the inputs, and the number of kernels the call launched."""
    l0 = lib.launches
    got = lib.em_kalman(x.X, x.Lam, x.R, x.A, x.Q, p=1, P0=x.P0, want_PF=want_PF, **dict(x.opts, **kw))
    return got, lib.launches - l0


def streamed_launches(got, want_PF=True):
    """Kernels of a streaming call that stayed on the fused kernel."""
    return 1 + int(want_PF) + int((np.asarray(got["status"]) == 3).any())


def monolithic_launches(x, want_PF=True):
    """Kernels of an upload-then-compute call of a balanced batch: k_lyapunov (no caller P0), k_fill, k_em_scan_fused, EM."""
    return 3 + int(x.P0 is None) + int(want_PF)


def run_streaming(lib, x, want_PF=True, **kw):
    got, n = run(lib, x, want_PF, **kw)
    assert n == streamed_launches(got, want_PF), "the call did not stream: %d kernel launches" % n
    return got


def run_monolithic(lib, x, want_PF=True, **kw):
    with no_pipeline():
        ref, n = run(lib, x, want_PF, **kw)
    assert n == monolithic_launches(x, want_PF), "upload-then-compute call: %d kernel launches" % n
    return ref


def assert_same(got, ref, what, panels=None):
    """Bit-identical outputs (NaN == NaN), of the panels `panels` (default: all)."""
    assert set(got) == set(ref)
    for k in got:
        a, b = (got[k], ref[k]) if panels is None else (got[k][panels], ref[k][panels])
        if not np.array_equal(a, b, equal_nan=True):
            bad = np.unique(np.nonzero(~((a == b) | ((a != a) & (b != b))))[0])
            raise AssertionError("%s: %s differs in %d panels, first %s" % (what, k, len(bad), bad[:8]))


def panel(res, b):
    return {k: res[k][b] for k in res}


def oracle(x, b):
    o = x.opts
    return K.em_kalman(x.X[b], x.Lam[b], x.R[b], x.A[b], x.Q[b], p=1, P0=None if x.P0 is None else x.P0[b],
                       max_iter=o["max_iter"], tol=o["tol"])


def compare_with_oracle(x, got, b):
    """Panel b of a batched result against the oracle from the same start (the bars of P.check_em), with the oracle's
    stopping iteration and the NaN tail of the log-likelihood row."""
    ref = oracle(x, b)
    g = panel(got, b)
    n = ref["iters"]
    assert g["status"] == 0 and g["iters"] == n, "panel %d: status %d, %d iterations, oracle %d" % (b, g["status"], g["iters"], n)
    assert np.isnan(g["loglik"][n:]).all()
    g["loglik"] = g["loglik"][:n]
    P.compare_em(g, ref, P.ll_atol(x.X[b], 1e-13))


def sample_panels(B, seed=7):
    """The first, the last and three seeded-random panels."""
    return sorted({0, B - 1} | set(int(b) for b in np.random.default_rng(seed).integers(1, B - 1, 3)))


def lyapunov_error(x, P0, b):
    """max |P0 - P| / max |P| against scipy's direct solution of P = A P A' + Q, and the spectral radius of A."""
    from scipy.linalg import solve_discrete_lyapunov
    ref = solve_discrete_lyapunov(x.A[b], x.Q[b])
    return np.abs(P0 - ref).max() / np.abs(ref).max(), np.abs(np.linalg.eigvals(x.A[b])).max()


def assert_lyapunov(x, P0, panels, what):
    """P0 solves the Lyapunov equation to 1e-12 where the radius is at most 0.98; beyond it twelve doublings truncate the
    sum, and the error is printed only."""
    worst = 0.0
    for b in panels:
        err, rho = lyapunov_error(x, P0[b], b)
        if rho <= 0.9801:
            assert err <= 1e-12, "%s: panel %d (radius %.4f): P0 off the Lyapunov solution by %.3g" % (what, b, rho, err)
        else:
            worst = max(worst, err)
    if worst:
        print("%s: truncation error of 12 doublings at radius > 0.98: %.3g (relative)" % (what, worst))


# ------------------------------------------------------------------------------------------------------ the checks
def check_equals_monolithic(lib, case):
    x = build(case)
    got = run_streaming(lib, x)
    ref = run_monolithic(lib, x)
    assert_same(got, ref, case.id)
    assert (got["status"] == 0).all()
    if x.opts["tol"] > 0:
        its = got["iters"]
        assert case.id != "early_stop" or len(np.unique(its)) >= 5, np.unique(its)
        assert its.min() >= 2 and its.max() <= x.opts["max_iter"]
        for b in range(len(its)):
            assert np.isfinite(got["loglik"][b, :its[b]]).all() and np.isnan(got["loglik"][b, its[b]:]).all(), b
    else:
        assert (got["iters"] == x.opts["max_iter"]).all() and np.isfinite(got["loglik"]).all()


def check_vs_oracle(lib, case):
    x = build(case, seed=SEED + 10000)
    got = run_streaming(lib, x)
    for b in sample_panels(len(x.X)):
        compare_with_oracle(x, got, b)


def check_p0(lib, case):
    x = build(case, seed=SEED + 20000)
    got = run_streaming(lib, x)
    ref = run_monolithic(lib, x)
    assert np.array_equal(got["P0"], ref["P0"]), "%s: in-kernel P0 differs from k_lyapunov's" % case.id
    if x.P0 is not None:
        assert np.array_equal(got["P0"], x.P0)                    # the caller's, not the Lyapunov solution
        for b in sample_panels(len(x.X)):
            compare_with_oracle(x, got, b)
        return
    assert_lyapunov(x, got["P0"], range(len(x.X)), case.id)
    for b in sample_panels(len(x.X)):
        np.testing.assert_allclose(got["P0"][b], K.lyapunov_doubling(x.A[b], x.Q[b]), rtol=1e-13, atol=0)


def check_rehearsal(lib, case, B=EMU_PANELS):
    """The first B panels of a case on k_em_fused2 without streaming (the host-emulation build cannot stream): every panel
    against the oracle, P0 against the Lyapunov solution, and the spread of the stopping iterations."""
    x = build(case, B)
    got, _ = run(lib, x, path=3)
    for b in range(B):
        compare_with_oracle(x, got, b)
    if x.P0 is None:
        assert_lyapunov(x, got["P0"], range(B), case.id)
    else:
        assert np.array_equal(got["P0"], x.P0)
    if x.opts["tol"] > 0:
        assert (got["iters"] < x.opts["max_iter"]).sum() > B // 2         # panels stop early: their rows keep a NaN tail
        assert case.id != "early_stop" or len(np.unique(got["iters"])) >= 5, np.unique(got["iters"])


def check_rehearsal_failed_panel(lib, value, B=EMU_PANELS, bad=(11,)):
    """The failed-panel inputs on k_em_fused2 without streaming: status 3 for the bad panel, its neighbours untouched."""
    x = failed_panel_inputs(B, value, bad)
    got, _ = run(lib, x, path=3)
    assert got["status"][bad[0]] == 3 and (np.delete(got["status"], bad) == 0).all(), got["status"]
    for b in (bad[0] - 1, bad[0] + 1):
        compare_with_oracle(x, got, b)


def find_resident(lib, x):
    """The largest batch the library runs upload-then-compute: bisection on the launch count of one-iteration calls."""
    def streams(B):
        got, n = run(lib, head(x, B), want_PF=False, max_iter=1)
        assert n in (streamed_launches(got, False), monolithic_launches(x, False)), n
        return n == streamed_launches(got, False)
    lo, hi = 1, len(x.X)                                            # lo does not stream, hi does
    assert not streams(lo) and streams(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (lo, mid) if streams(mid) else (mid, hi)
    return lo


def check_batch_edges(lib, B=1500):
    """Prefixes of one batch: the smallest batch that streams (one panel in a second round), batches that end inside an
    upload chunk (32 panels) and a return chunk (128), one that ends on both (1280), one whose last upload chunk holds one
    panel (1281).  A panel's results must not depend on the chunk or round it fell in."""
    x = dgp_inputs(B, seed=SEED, **SMALL)
    resident = find_resident(lib, x)
    assert resident + 33 < 1279, resident
    ref = run_monolithic(lib, x)
    for n in (resident + 1, resident + 33, 1279, 1280, 1281, B):
        got = run_streaming(lib, head(x, n))
        assert_same(got, {k: ref[k][:n] for k in ref}, "prefix of %d panels (resident %d)" % (n, resident))


def raw_call(lib, x, names):
    """dfm_em_kalman through the C structs with only the outputs `names` requested (the others NULL); the buffers start
    as a sentinel so that an output the library skipped shows."""
    from dynamic_factor_models_b200._lib import MEM_HOST, to_cm
    B, T, N = x.X.shape
    r, mi = x.Lam.shape[-1], x.opts["max_iter"]
    bufs = dict(X=to_cm(x.X), Lam=to_cm(x.Lam), R=np.ascontiguousarray(x.R), A=to_cm(x.A), Q=to_cm(x.Q))
    size = dict(F=T * r, Lam=N * r, R=N, A=r * r, Q=r * r, P0=r * r, PF=T * r * r, loglik=mi, iters=1, status=1)
    out = {k: np.full(B * size[k], -77, dtype=np.int32 if k in ("iters", "status") else np.float64) for k in names}
    l0 = lib.launches
    lib.em_kalman_raw(bufs["X"].ctypes.data, T, N, r, 1, B, mi, x.opts["tol"], {k: bufs[k].ctypes.data for k in ("Lam", "R", "A", "Q")},
                      {k: a.ctypes.data for k, a in out.items()}, MEM_HOST)
    assert lib.launches - l0 == 1 + int("PF" in names), "the raw call did not stream"
    return out


def flat(res, k):
    """An output of Library.em_kalman in the library's own layout (column-major panels)."""
    from dynamic_factor_models_b200._lib import to_cm
    a = res[k]
    return (to_cm(a) if k in ("F", "Lam", "A", "Q", "P0") else np.ascontiguousarray(a)).ravel()


def check_null_outputs(lib, B=1500):
    x = early_stop_inputs(B, SEED)
    full = run_streaming(lib, x)
    for names in (("loglik", "status"), tuple(k for k in OUTPUTS if k != "PF")):
        out = raw_call(lib, x, names)
        for k in names:
            assert np.array_equal(out[k], flat(full, k), equal_nan=True), "outputs %s: %s differs from the full call" % (names, k)


def device_general_call(lib, x, sync):
    """A DFM_MEM_DEVICE call of the general path (path 1) on torch tensors; without `sync` it returns with its work in
    flight.  Returns the output tensors."""
    import torch
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    B, T, N = x.X.shape
    r, mi = x.Lam.shape[-1], x.opts["max_iter"]
    dev = {k: torch.from_numpy(v).cuda() for k, v in dict(X=to_cm(x.X), Lam=to_cm(x.Lam), R=np.ascontiguousarray(x.R), A=to_cm(x.A),
                                                         Q=to_cm(x.Q)).items()}
    size = dict(F=T * r, Lam=N * r, R=N, A=r * r, Q=r * r, P0=r * r, loglik=mi)
    out = {k: torch.zeros(B * n, dtype=torch.float64, device="cuda") for k, n in size.items()}
    out.update({k: torch.zeros(B, dtype=torch.int32, device="cuda") for k in ("iters", "status")})
    torch.cuda.synchronize()
    lib.em_kalman_raw(dev["X"].data_ptr(), T, N, r, 1, B, mi, 0.0, {k: dev[k].data_ptr() for k in ("Lam", "R", "A", "Q")},
                      {k: a.data_ptr() for k, a in out.items()}, MEM_DEVICE, path=1)
    if sync:
        lib.sync()
    return out, dev


def check_handle_reuse(lib, B=1700):
    """One handle through a large, a smaller and a larger streaming call (the completion flags grow; only the flags of the
    call's own panels are reset), then a streaming call issued while a device-resident call is still in flight on the
    handle's stream (the copy streams must wait for it before they touch the shared workspace).  Each result equals the
    same call on another handle."""
    from dynamic_factor_models_b200 import Library
    x = dgp_inputs(B, seed=SEED + 1, **SMALL)
    small = find_resident(lib, x) + 36
    assert small < 1500
    second = Library()
    try:
        for n in (1500, small, B):
            assert_same(run_streaming(second, head(x, n)), run_streaming(lib, head(x, n)), "call %d of the reused handle" % n)
        xd = head(x, 1500)._replace(opts=dict(max_iter=10, tol=0.0))
        dout, keep = device_general_call(second, xd, sync=False)
        got = run_streaming(second, head(x, 1500))
        second.sync()
        assert_same(got, run_streaming(lib, head(x, 1500)), "streaming call behind a device-resident call")
        dref, keep2 = device_general_call(lib, xd, sync=True)
        for k in dout:                                                # ... and that call's own results are intact
            assert np.array_equal(dout[k].cpu().numpy(), dref[k].cpu().numpy(), equal_nan=True), "device-resident call: %s" % k
        del keep, keep2
    finally:
        second.close()


FALLBACK_PLACEMENTS = {"first": (0,), "last": (-1,), "many": (0, 31, 32, 640, -1), "excluded_series": (700,)}


def check_fallback(lib, where, B=1500):
    """Missing data met on the streaming path: the fused kernel has run (status 3 for the panels with NaNs), the deferred
    scan finds the NaNs and the whole batch is re-run on the general path from the initial parameters.  excluded_series:
    clean data, but one series of one panel is out of the model (NaN loadings and variance in the caller's start), which
    only the general path handles; the deferred scan finds it in the caller's buffers without a kernel."""
    x = dgp_inputs(B, seed=SEED + 2, **SMALL)
    holes = [b % B for b in FALLBACK_PLACEMENTS[where]]
    for b in holes:
        if where == "excluded_series":
            x.Lam[b, 3], x.R[b, 3] = np.nan, np.nan
        else:
            x.X[b, 5:9, 3] = np.nan
    with no_pipeline():
        ref, n_ref = run(lib, x)
    got, n = run(lib, x)
    # the streaming attempt (EM kernel, k_unpack_psf, deferred scan) replaces the up-front scan of the other host path
    assert n == n_ref + 2 - int(where == "excluded_series"), "with missing data: %d launches, upload-then-compute %d" % (n, n_ref)
    assert np.array_equal(got["status"], ref["status"]) and np.array_equal(got["iters"], ref["iters"])
    assert (got["status"] == 0).all()
    for k in OUTPUTS[:-2]:
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-12, atol=1e-13, err_msg=k)
    for b in sorted(set(holes) | {1, B - 2}):
        compare_with_oracle(x, got, b)


def check_fallback_refused(lib, B=1500):
    """path = 3 (the TMA fused kernel or nothing) with a NaN in the batch: DFM_ERR_UNSUPPORTED, raised after the kernel has
    run; the handle is fit for the next call."""
    import dynamic_factor_models_b200 as D
    x = dgp_inputs(B, seed=SEED + 2, **SMALL)
    clean = run_monolithic(lib, x)
    X = x.X.copy()
    X[640, 5:9, 3] = np.nan
    try:
        run(lib, x._replace(X=X), path=3)
        raise AssertionError("path 3 accepted a panel with missing data")
    except D.DFMError as e:
        assert e.code == 6, e.code
    assert_same(run_streaming(lib, x, path=3), clean, "clean call after the refused one")


def failed_panel_inputs(B, value, bad=(700,)):
    x = dgp_inputs(B, seed=SEED + 3, **SMALL)
    for b in bad:
        x.R[b, 3] = value
    return x


def check_failed_panel(lib, value, B=1500, bad=(700,)):
    """A panel that fails numerically with clean data (an idiosyncratic variance <= 0 at the start): status 3 for that
    panel on both host paths, and the batch stays on the fused kernel -- the deferred scan of the streaming path looks for
    missing data in what the caller passed, not at the NaNs the failed panel left in its own parameters."""
    x = failed_panel_inputs(B, value, bad)
    ref = run_monolithic(lib, x)
    got = run_streaming(lib, x)                                     # EM kernel + k_unpack_psf + the scan, no general path
    ok = np.setdiff1d(np.arange(B), bad)
    for res in (got, ref):
        assert (res["status"][list(bad)] == 3).all() and (res["status"][ok] == 0).all(), np.nonzero(res["status"])[0]
    assert_same(got, ref, "batch with a failed panel", ok)
    assert np.array_equal(got["iters"], ref["iters"])
    for b in (bad[0] - 1, bad[0] + 1):
        compare_with_oracle(x, got, b)
