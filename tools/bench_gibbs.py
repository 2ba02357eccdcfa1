#!/usr/bin/env python
"""bench_gibbs.py -- throughput of dfm_gibbs (batched Gibbs chains of the state-space DFM) on two workloads:
  c2     a C2-shaped model (N=200, r=8, T=500, p=1, balanced; all chains started at the parameters after 50 EM iterations on
         bench.py's panel 0), 264 chains (one sub-batch), H_irf = 24;
  c1     the hom_fac_1 Parametric model (r=8, p=4, 139 estimation series, T=222, 5.7 % missing; estimate(m, Parametric())),
         264 chains, H_irf = 24, H_fc = 8 with the last 12 rows of predictive draws.
Every step runs `--sweeps` sweeps per chain (half burn-in, half kept).  Prints one JSON line in bench.py's line format (value =
chain-sweeps/s of the c2 workload, device resident; the c1 workload, the end-to-end rates from host buffers, per-kernel times,
each stage's share of a sweep, the bytes / flops model of k_gibbs_stats, clocks, split-R^ of a 4-chain run and the NumPy spec
on one core under "config" / "e2e" / "roofline" / "cpu_baseline").

python tools/bench_gibbs.py --steps K --warmup W [--json profiles/h100_bench_gibbs.json] [--no-cpu]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ESTEP = ("k_em_filter_smooth", "k_em_contract", "k_em_contract_bal", "k_em_prep", "k_em_scan", "k_em_state_init", "k_em_collect")
STAGES = dict(estep=ESTEP, gains=("k_sim_gains",), paths=("k_gibbs_paths",), stats=("k_gibbs_stats",), draw=("k_gibbs_draw",))
PEAK_DMMA_TFLOPS = 66.9          # H100 SXM5 FP64 tensor-core data-sheet rate


def _fit_c2(lib, iters):
    N, r, T = bench.NS, bench.R_, bench.T_
    X = lib.simulate_panels(0, 1, N, r, T, bench.SEED)[0]
    F0 = lib.estimate_factor(X, r, max_iter=1)["F"]
    Lam, R, A, Q = lib.em_init_from_factors(X, F0, 1)
    em = lib.em_kalman(X, Lam, R, A, Q, p=1, max_iter=iters, tol=0.0, want_PF=False)
    return X, dict(Lam=em["Lam"], R=em["R"], A=em["A"], Q=em["Q"], P0=em["P0"]), 1


def _fit_c1(lib):
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200.api import _state_space_block
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    m = D.DFMModel(z["all_bpdata"], z["all_inclcode"], 20, 40, 3, 224, 0, 8, 1e-8, 4, 4)
    D.estimate(m, D.Parametric(max_iter=50, tol=1e-6), lib=lib)
    b = _state_space_block(m, 0, lib, "bench")
    e = m.em
    return b["Xs"], dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"]), b["p"]


def _stats_model(T, N, r, C):
    """k_gibbs_stats per sweep: X' [F~_1 .. F~_C] as tiles of 32 series x 32 columns; every column tile re-reads the panel (from
    L2 after the first), every series tile the factor columns; s_i written once."""
    nct = -(-C * r // 32); nst = -(-N // 32)
    flops = 2.0 * T * N * C * r
    l2_bytes = 8.0 * T * N * nct + 8.0 * T * C * r * nst + 8.0 * N * C * r
    hbm_bytes = 8.0 * T * N + 8.0 * T * C * r + 8.0 * N * C * r
    return flops, l2_bytes, hbm_bytes


def _workload(lib, torch, dev, X, th, p, n_chain, n_sweep, H_irf, H_fc, fc_rows, K_, W_, no_cpu):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm, gibbs_default_prior
    T, N = X.shape; r = th["Lam"].shape[1]; k = r * p; Tp = T + H_fc
    n_burn = n_sweep // 2; n_keep = n_sweep - n_burn
    cm = lambda a: torch.from_numpy(np.ascontiguousarray(to_cm(a))).to(dev)
    rep = lambda a: np.stack([a] * n_chain)
    init = {n: rep(th[n]) for n in ("Lam", "R", "A", "Q", "P0")}
    dX = cm(X); dref = {n: cm(th[n]) for n in ("Lam", "R", "A", "Q")}
    # per-chain arrays back to back: matrices column-major per chain, R (n_chain, N) row by row
    dini = {n: (cm(init[n]) if n != "R" else torch.from_numpy(np.ascontiguousarray(init[n]).ravel()).to(dev)) for n in init}
    f64 = lambda n: torch.empty(max(n, 1), dtype=torch.float64, device=dev)
    sizes = dict(Lam=N * r, R=N, A=r * k, Q=r * r, irf=r * H_irf * r, X=fc_rows * N)
    if fc_rows == 0:
        del sizes["X"]
    dout = {n: f64(n_chain * n_keep * s) for n, s in sizes.items()}
    dll = f64(n_chain * n_sweep); dst = torch.empty(n_chain, dtype=torch.int32, device=dev)
    outs = {**{n: t.data_ptr() for n, t in dout.items()}, "loglik": dll.data_ptr(), "status": dst.data_ptr()}
    prior = gibbs_default_prior(r)
    kw = dict(n_chain=n_chain, n_burn=n_burn, n_keep=n_keep, seed=bench.SEED, H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, prior=prior)

    def step():
        lib.gibbs_raw(dX.data_ptr(), T, N, r, p, {n: t.data_ptr() for n, t in dini.items()}, {n: t.data_ptr() for n, t in dref.items()},
                      outs, MEM_DEVICE, **kw)
        lib.sync()

    for _ in range(W_):
        step()
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    l0 = lib.launches
    ms = bench._timed(torch, None, 1, dev, step, K_)
    launches = (lib.launches - l0) // K_
    clk = clocks.stop()
    status = dst.cpu().numpy()
    # end to end: host arrays through Library.gibbs (uploads, sweeps, downloads of every kept draw)
    hkw = {k_: v for k_, v in kw.items()}
    lib.gibbs(X, init, p=p, ref=th, **hkw)
    t0 = time.perf_counter()
    host = lib.gibbs(X, init, p=p, ref=th, **hkw)
    ms_e = (time.perf_counter() - t0) * 1e3
    dev_ll = dll.cpu().numpy().reshape(n_chain, n_sweep)
    same = np.array_equal(host["loglik"], dev_ll) and np.array_equal(host["status"], status)
    # per-kernel times of one profiled step (outside the timed region)
    lib.profile(True); step(); prof = lib.profile_report(); lib.profile(False)
    tot = sum(v_[0] for v_ in prof.values()) or 1.0
    stage_ms = {s: sum(prof[n][0] for n in prof if n.split("<")[0] in names) for s, names in STAGES.items()}
    stage_ms["other"] = tot - sum(stage_ms.values())
    C = 264 if n_chain <= 264 else n_chain
    flops, l2b, hbmb = _stats_model(T, N, r, C)
    st_ms = prof["k_gibbs_stats"][0] / prof["k_gibbs_stats"][1]
    tfl = flops / (st_ms * 1e-3) / 1e12
    hbm = hbmb / (st_ms * 1e-3) / 1e9
    l2 = l2b / (st_ms * 1e-3) / 1e9
    peak, peak_src = bench._peak()
    cpu = None
    if not no_cpu:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import gibbs_oracle as O
        th0 = dict(th)
        O.sweep(X, th0, p, H_fc, prior, bench.SEED, O.gibbs_id(0, 0))
        t0 = time.perf_counter()
        ns_ = 3
        for s in range(ns_):
            th0, _, _, _, _ = O.sweep(X, th0, p, H_fc, prior, bench.SEED, O.gibbs_id(0, s))
        dt = time.perf_counter() - t0
        cpu = {"value": ns_ / dt, "unit": "chain-sweeps/s", "cores": 1, "kind": "port",
               "sample": f"{ns_} sweeps of one chain, NumPy spec (tests/gibbs_oracle.py), 1 process, {dt:.2f} s"}
    return dict(value=n_chain * n_sweep * K_ / (ms * 1e-3), ms_per_step=ms / K_, launches=launches, clocks=clk,
                all_status_ok=bool((status == 0).all()), e2e_value=n_chain * n_sweep / (ms_e * 1e-3), e2e_ms=ms_e, e2e_equals_device=bool(same),
                stage_ms={s: round(v_, 3) for s, v_ in stage_ms.items()}, stage_share={s: v_ / tot for s, v_ in stage_ms.items()},
                kernel_ms={n: round(v_[0], 3) for n, v_ in sorted(prof.items(), key=lambda kv: -kv[1][0])},
                stats=dict(flops_per_sweep=flops, l2_bytes_per_sweep=l2b, hbm_bytes_per_sweep=hbmb, ms_per_sweep=st_ms, tflops=tfl,
                           frac_dmma_peak=tfl / PEAK_DMMA_TFLOPS, hbm_gbs=hbm, frac_hbm_peak=hbm / peak, l2_gbs=l2,
                           bound="dmma" if tfl / PEAK_DMMA_TFLOPS > hbm / peak else "hbm"),
                cpu=cpu, peak=peak, peak_src=peak_src,
                shape=dict(T=T, N=N, r=r, p=p, n_chain=n_chain, sub_batch=C, sweeps_per_step=n_sweep, n_burn=n_burn, n_keep=n_keep,
                           H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, observed_frac=float(np.mean(~np.isnan(X)))))


def _rhat_c2(lib, X, th):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import gibbs_oracle as O
    got = lib.gibbs(X, th, p=1, n_chain=4, n_burn=500, n_keep=500, seed=11, outputs=("R",))
    return {"n_chain": 4, "n_burn": 500, "n_keep": 500, "loglik": float(O.split_rhat(got["loglik"][:, 500:])),
            "R_max": float(np.nanmax(O.split_rhat(got["R"]))), "status_ok": bool((got["status"] == 0).all())}


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    X2, th2, p2 = _fit_c2(lib, 50)
    c2 = _workload(lib, torch, dev, X2, th2, p2, args.chains, args.sweeps, 24, 0, 0, args.steps, args.warmup, args.no_cpu)
    X1, th1, p1 = _fit_c1(lib)
    c1 = _workload(lib, torch, dev, X1, th1, p1, args.chains, args.sweeps, 24, 8, 12, args.steps, args.warmup, args.no_cpu)
    rh = _rhat_c2(lib, X2, th2)
    st = c2["stats"]
    roof = {"bound": st["bound"], "kernel": "k_gibbs_stats", "achieved": st["tflops"], "peak": PEAK_DMMA_TFLOPS, "unit": "TFLOP/s",
            "frac": st["frac_dmma_peak"], "traffic": None, "peak_source": "H100 SXM5 data sheet (FP64 tensor core)",
            "stats_model": st, "stage_share_of_sweep": c2["stage_share"], "stage_ms_per_step": c2["stage_ms"], "kernel_ms": c2["kernel_ms"],
            "c1": {"stats_model": c1["stats"], "stage_share_of_sweep": c1["stage_share"], "stage_ms_per_step": c1["stage_ms"],
                   "kernel_ms": c1["kernel_ms"]},
            "note": "k_gibbs_stats: 2 T N C r flops of X' [F_1 .. F_C] per sweep (C = 264 chains of the sub-batch); HBM bytes = the panel, "
                    "the factor paths and s_i once; L2 bytes = the panel per column tile of 32, the paths per series tile of 32"}
    line = {"metric": f"Gibbs chain-sweeps/sec (C2-shaped model N={bench.NS} r={bench.R_} T={bench.T_} p=1, {args.chains} chains)",
            "value": c2["value"], "unit": "chain-sweeps/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": c2["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "C2: synthetic (device-generated frozen DGP, SURVEY.md 8d); C1: hom_fac_1 (tests/golden)",
            "config": {"workload": f"{args.chains} chains x {args.sweeps} sweeps per step of dfm_gibbs from the fitted parameters "
                                   f"(half burn-in, half kept with records and IRFs of all shocks, H_irf = 24)", **c2["shape"],
                       "all_status_ok": c2["all_status_ok"], "e2e_equals_device": c2["e2e_equals_device"], "rhat_c2": rh,
                       "c1": {**c1["shape"], "value": c1["value"], "unit": "chain-sweeps/s", "ms_per_step": c1["ms_per_step"],
                              "e2e_value": c1["e2e_value"], "all_status_ok": c1["all_status_ok"], "e2e_equals_device": c1["e2e_equals_device"],
                              "gpu_launches": c1["launches"], "cpu_baseline": c1["cpu"]}},
            "e2e": {"value": c2["e2e_value"], "unit": "chain-sweeps/s", "ms_per_step": c2["e2e_ms"], "c1_value": c1["e2e_value"],
                    "c1_ms_per_step": c1["e2e_ms"]},
            "gpu_launches": int(c2["launches"]), "clocks": c2["clocks"], "roofline": roof, "cpu_baseline": c2["cpu"]}
    s = json.dumps(line)
    print(s)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(s + "\n")
    lib.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chains", type=int, default=264, help="chains per workload")
    ap.add_argument("--sweeps", type=int, default=20, help="sweeps per chain and step")
    ap.add_argument("--json", default=None, help="also write the line to this file")
    ap.add_argument("--no-cpu", action="store_true")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
