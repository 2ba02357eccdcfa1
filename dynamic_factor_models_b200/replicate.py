"""Replication-level drivers -- row (e) of SURVEY.md section 8 and configs C4 / C5 of BASELINE.json.

Replications (Monte-Carlo panels, bootstrap draws) are independent: rank g of G owns the contiguous
shard dfm_shard_range(n_rep, g, G); every replication's random stream is a pure function of its
replication id (counter-based Philox4x32-10 on the DEVICE: dfm_simulate_panels / dfm_bootstrap_panels),
so results do not depend on the GPU count; the per-shard work is a handful of batched calls into the
CUDA library; the path's single collective is one all-gather of the per-replication records at the very
end (torch.distributed: NCCL over NVLink on GPUs, gloo in the CPU tests); the percentile bands are a
device sort per statistic (dfm_percentiles).  The reference has no bootstrap / Monte-Carlo / RNG code at
all (SURVEY.md section 0).
"""
import numpy as np

SEED = 20260922


def simulate_panel(N, r, T, rep=0, seed=SEED, lib=None):
    """Frozen synthetic DGP of SURVEY.md 8d, generated on the device: Lam~N(0,1); f_t = diag(a) f_{t-1} + eta_t,
    a~U(.2,.8), burn-in 100; e_it~N(0,s2_i), s2_i~U(.5,1.5); column-standardised (population std).  (T, N)."""
    from .api import get_library
    return (lib or get_library()).simulate_panels(int(rep), 1, N, r, T, seed)[0]


def gather_records(rec_local, n_rep, rank, world, lib):
    """All-gather per-replication records (n_local, d) -> (n_rep, d) on every rank.  One collective."""
    if world == 1:
        return np.asarray(rec_local)
    import torch
    import torch.distributed as dist
    b, e = lib.shard_range(n_rep, rank, world)
    nmax = max(lib.shard_range(n_rep, g, world)[1] - lib.shard_range(n_rep, g, world)[0] for g in range(world))
    d = rec_local.shape[1]
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    buf = torch.full((nmax, d), float("nan"), dtype=torch.float64, device=dev)
    buf[:e - b] = torch.from_numpy(np.ascontiguousarray(rec_local)).to(dev)
    out = torch.empty((world * nmax, d), dtype=torch.float64, device=dev)
    dist.all_gather_into_tensor(out, buf)
    out = out.cpu().numpy().reshape(world, nmax, d)
    return np.concatenate([out[g, :lib.shard_range(n_rep, g, world)[1] - lib.shard_range(n_rep, g, world)[0]] for g in range(world)])


def monte_carlo_em(lib, n_rep, N, r, T, p=1, em_iters=50, tol=0.0, rank=0, world=1, seed=SEED):
    """C5: EM on n_rep simulated panels.  Record per replication: [final loglik, iterations, status,
    trace R2 of the ALS start].  Returns the gathered (n_rep, 4) array (identical on all ranks)."""
    b, e = lib.shard_range(n_rep, rank, world)
    rec = np.empty((e - b, 4))
    if e > b:
        X = lib.simulate_panels(b, e - b, N, r, T, seed)                    # device generator, ids b .. e-1
        als = lib.estimate_factor(X, r, max_iter=1, compute_r2=False)
        Lam, R, A, Q = lib.em_init_from_factors(X, als["F"], p)
        em = lib.em_kalman(X, Lam, R, A, Q, p=p, max_iter=em_iters, tol=tol, want_PF=False)
        it = np.asarray(em["iters"]).reshape(-1)
        ll = np.asarray(em["loglik"]).reshape(e - b, em_iters)
        rec[:, 0] = ll[np.arange(e - b), it - 1]; rec[:, 1] = it; rec[:, 2] = np.asarray(em["status"]).reshape(-1)
        st = als["stats"] if isinstance(als["stats"], list) else [als["stats"]]
        rec[:, 3] = [1 - s["ssr"] / s["tss"] for s in st]
    return gather_records(rec, n_rep, rank, world, lib)


def bootstrap_panels(m, ids, seed=SEED, burn=50, lib=None):
    """Residual bootstrap of a fitted non-parametric model `m` (api.DFMModel after estimate()), on the device:
    resample the factor-VAR residuals with replacement and rebuild f* through the VAR, draw the idiosyncratic
    AR(n_uarlag) processes from (uar_coef, uar_ser), x* = Lam f* + u*, original missing pattern re-imposed
    (SURVEY.md 8d, config C4).  `ids` must be consecutive replication ids.  Returns (len(ids), T_w, ns)."""
    from .api import get_library
    lib = lib or get_library()
    ids = list(ids)
    assert ids == list(range(ids[0], ids[0] + len(ids))), "replication ids must be consecutive"
    i0, i1 = m.initperiod, m.lastperiod
    v = m.factor_var_model; p = v.nlag
    return lib.bootstrap_panels(m.factor[i0 - 1:i1], v.resid[i0 - 1:i1][p:], v.betahat, m.lambda_, m.uar_coef, m.uar_ser,
                                m.data[i0 - 1:i1], ids[0], len(ids), seed, burn=burn)


BAND_PERCENTILES = (5, 16, 50, 84, 95)


def bootstrap_irf(lib, m, n_rep, H=24, rank=0, world=1, seed=SEED):
    """C4: bootstrap distribution of the factor-VAR impulse responses.  Every replication is
    re-estimated with the full non-parametric pipeline (ALS factors -> VAR -> IRF) inside ONE device-resident
    call (dfm_bootstrap_irf); factor signs are aligned with the original estimate; replications whose
    re-estimation fails (ALS status 2/3, singular VAR) are NaN records and are ignored by the bands.  Returns
    (irfs (n_rep, r, H, r), bands dict of 5/16/50/84/95 percentiles)."""
    b, e = lib.shard_range(n_rep, rank, world)
    r = m.nfac_t; p = m.factor_var_model.nlag
    rec = np.full((e - b, r * H * r), np.nan)
    if e > b:
        i0, i1 = m.initperiod, m.lastperiod
        v = m.factor_var_model; incl = m.inclcode == 1
        irf, _, _ = lib.bootstrap_irf(m.factor[i0 - 1:i1], v.resid[i0 - 1:i1][p:], v.betahat, m.lambda_[incl], m.uar_coef[incl],
                                      m.uar_ser[incl], m.data[i0 - 1:i1][:, incl], b, e - b, seed, H,
                                      nt_min=m.nt_min_factor_estimation, tol=m.tol)
        rec[:] = irf.reshape(e - b, -1)                                      # one device-resident call per shard
    allrec = gather_records(rec, n_rep, rank, world, lib)
    irfs = allrec.reshape(n_rep, r, H, r)
    pb = lib.percentiles(allrec, BAND_PERCENTILES)                           # device sort per statistic
    bands = {q: pb[k].reshape(r, H, r) for k, q in enumerate(BAND_PERCENTILES)}
    return irfs, bands


def ss_bootstrap(lib, m, n_rep, H_irf=24, H_fc=0, fc_rows=0, max_iter=50, tol=0.0, rank=0, world=1, seed=SEED):
    """Parametric bootstrap of a model estimated with `estimate(m, Parametric())`, sharded over ranks: rank g runs ONE
    dfm_ss_bootstrap call on replication ids dfm_shard_range(n_rep, g, world) (simulate -> EM from m.em -> align -> IRF, device
    resident), then one all-gather of the records.  A replicate's panel is a pure function of (seed, replication id), so the
    result does not depend on the number of ranks.  Record per replicate: [irf (r * H_irf * r), loglik, iters, status, xhat
    (fc_rows * ns)].  Returns (irfs (n_rep, r, H_irf, r) [variable, horizon, shock], bands dict of 5/16/50/84/95 percentiles,
    records (n_rep, d))."""
    from .api import _state_space_block
    blk = _state_space_block(m, H_fc, lib, "ss_bootstrap")
    e = blk["em"]
    r = e["Q"].shape[0]; ns = blk["Xs"].shape[1]
    nirf = r * H_irf * r
    b, en = lib.shard_range(n_rep, rank, world)
    rec = np.full((en - b, nirf + 3 + fc_rows * ns), np.nan)
    if en > b:
        o = lib.ss_bootstrap(blk["Xs"], blk["Lam"], e["R"], e["A"], e["Q"], e["P0"], p=blk["p"], n_rep=en - b, seed=seed, rep0=b,
                             H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, max_iter=max_iter, tol=tol,
                             outputs=("irf", "xhat") if fc_rows > 0 else ("irf",))
        rec[:, :nirf] = o["irf"].transpose(0, 3, 2, 1).reshape(en - b, -1)      # dfm_irf's record layout [shock][horizon][variable]
        rec[:, nirf] = o["loglik"]; rec[:, nirf + 1] = o["iters"]; rec[:, nirf + 2] = o["status"]
        if fc_rows > 0:
            rec[:, nirf + 3:] = o["xhat"].reshape(en - b, -1)
    allrec = gather_records(rec, n_rep, rank, world, lib)
    irfs = np.ascontiguousarray(allrec[:, :nirf].reshape(n_rep, r, H_irf, r).transpose(0, 3, 2, 1))
    pb = lib.percentiles(allrec[:, :nirf], BAND_PERCENTILES)
    bands = {q: pb[k].reshape(r, H_irf, r).transpose(2, 1, 0) for k, q in enumerate(BAND_PERCENTILES)}
    return irfs, bands, allrec
