#!/usr/bin/env python
"""bench_ss_bootstrap.py -- throughput of dfm_ss_bootstrap (parametric bootstrap of a fitted state-space DFM: simulate -> EM
from the fitted parameters -> align -> IRF -> forecasts) on two workloads of 1000 replicates each:
  c2     a C2-shaped model (N=200, r=8, T=500, p=1, balanced; the parameters after 50 EM iterations on bench.py's panel 0),
         50 EM iterations per replicate on dfm_em_kalman's fused path, H_irf = 24, no forecasts;
  c1     the hom_fac_1 Parametric model (r=8, p=4, 139 estimation series, T=222, 5.7 % missing; estimate(m, Parametric())),
         20 EM iterations per replicate on the general path, H_irf = 24, H_fc = 8 with the last 12 rows returned.
Prints one JSON line in bench.py's line format (value = replicates/s of the c2 workload, device resident; the c1 workload,
the end-to-end rates from host buffers, per-kernel times, the EM share of the step, the bytes model of k_ss_sim_project over
the 3.35 TB/s data-sheet rate, clocks and the NumPy spec on one core under "config" / "e2e" / "roofline" / "cpu_baseline").

python tools/bench_ss_bootstrap.py --steps K --warmup W [--json profiles/h100_bench_ss-bootstrap.json] [--no-cpu]
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

EM_KERNELS = ("k_em_fused2", "k_em_fused", "k_em_filter_smooth", "k_em_contract", "k_em_contract_bal", "k_em_mstep_series", "k_em_prep",
              "k_em_scan", "k_em_scan_fused", "k_em_state_init", "k_em_collect", "k_emb_contract", "k_emb_mstep", "k_emb_close",
              "k_emb_cinit", "k_em_count_active", "k_em_count_missing", "k_fill")


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


def _workload(lib, torch, dev, X, th, p, n_rep, mi, H_irf, H_fc, fc_rows, K_, W_, no_cpu):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    T, N = X.shape; r = th["Lam"].shape[1]; k = r * p
    cm = lambda a: torch.from_numpy(np.ascontiguousarray(to_cm(a))).to(dev)
    dX = cm(X); dpar = {n: cm(th[n]) for n in ("Lam", "R", "A", "Q", "P0")}
    f64 = lambda n: torch.empty(max(n, 1), dtype=torch.float64, device=dev)
    sizes = dict(Lam=N * r, R=N, A=r * k, Q=r * r, irf=r * H_irf * r, xhat=fc_rows * N, xvar=fc_rows * N, loglik=1)
    if fc_rows == 0:
        del sizes["xhat"], sizes["xvar"]
    dout = {n: f64(n_rep * s) for n, s in sizes.items()}
    dit = torch.empty(n_rep, dtype=torch.int32, device=dev); dst = torch.empty(n_rep, dtype=torch.int32, device=dev)
    outs = {**{n: t.data_ptr() for n, t in dout.items()}, "iters": dit.data_ptr(), "status": dst.data_ptr()}
    kw = dict(n_rep=n_rep, rep0=0, seed=bench.SEED, H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, max_iter=mi, tol=0.0)

    def step():
        lib.ss_bootstrap_raw(dX.data_ptr(), T, N, r, p, {n: t.data_ptr() for n, t in dpar.items()}, outs, MEM_DEVICE, **kw)
        lib.sync()

    for _ in range(W_):
        step()
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    l0 = lib.launches
    ms = bench._timed(torch, None, 1, dev, step, K_)
    launches = (lib.launches - l0) // K_
    clk = clocks.stop()
    status = dst.cpu().numpy()
    # end to end: host arrays through Library.ss_bootstrap (uploads, sub-batched device work, downloads)
    lib.ss_bootstrap(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, **{k_: v for k_, v in kw.items() if k_ != "rep0"})
    t0 = time.perf_counter()
    host = lib.ss_bootstrap(X, th["Lam"], th["R"], th["A"], th["Q"], th["P0"], p=p, **{k_: v for k_, v in kw.items() if k_ != "rep0"})
    ms_e = (time.perf_counter() - t0) * 1e3
    dev_irf = bench._cm(dout["irf"], n_rep, r * H_irf * r, 1).reshape(n_rep, r, H_irf, r).transpose(0, 3, 2, 1)
    same = np.array_equal(np.nan_to_num(host["irf"], nan=7.0), np.nan_to_num(dev_irf, nan=7.0)) and np.array_equal(host["status"], status)
    # per-kernel times of one profiled step (outside the timed region)
    lib.profile(True); step(); prof = lib.profile_report(); lib.profile(False)
    tot = sum(v_[0] for v_ in prof.values()) or 1.0
    em_ms = sum(prof[n][0] for n in prof if n.split("<")[0] in EM_KERNELS)
    proj_ms = prof["k_ss_sim_project"][0]
    sim_ms = proj_ms + prof["k_ss_simulate"][0] + prof.get("k_ss_sim_chol", (0.0,))[0]
    nst = (N + 63) // 64; ntt = (T + 31) // 32
    obs_frac = float(np.mean(~np.isnan(X)))
    # k_ss_sim_project: the panels written (8 T N per replicate), the factors read once per series tile (8 T r nst), the
    # template's NaN pattern and the loadings per tile of SIM_PD = 8 replicates
    alg = n_rep * (8.0 * T * N + 8.0 * T * r * nst) + np.ceil(n_rep / 8) * (8.0 * T * N + ntt * 8.0 * N * (r + 1))
    peak, peak_src = bench._peak()
    ach = alg / (proj_ms * 1e-3) / 1e9
    cpu = None
    if not no_cpu:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import ss_bootstrap_oracle as O
        t0 = time.perf_counter()
        ref = O.replicate(X, th, p, bench.SEED, 0, mi, 0.0, H_irf, H_fc, fc_rows)
        dt = time.perf_counter() - t0
        dev0 = dev_irf[0]
        cpu = {"value": 1.0 / dt, "unit": "replicates/s", "cores": 1, "kind": "port",
               "sample": f"1 replicate, NumPy spec (tests/ss_bootstrap_oracle.py: simulate, oracle EM {mi} iterations, align, IRF"
                         f"{', forecasts' if fc_rows else ''}), 1 process, {dt:.2f} s",
               "irf_max_abs_diff_vs_device": float(np.max(np.abs(dev0 - ref["irf"].transpose(2, 1, 0)))) if ref["aligned"] is not None else None}
    return dict(value=n_rep * K_ / (ms * 1e-3), ms_per_step=ms / K_, launches=launches, clocks=clk, all_status_ok=bool((status == 0).all()),
                n_failed=int((status != 0).sum()), e2e_value=n_rep / (ms_e * 1e-3), e2e_ms=ms_e, e2e_equals_device=bool(same),
                h2d=8 * (T * N + N * r + N + r * k + r * r + k * k), d2h=8 * n_rep * sum(sizes.values()) + 8 * n_rep,
                em_share=em_ms / tot, sim_share=sim_ms / tot, proj_ms=proj_ms, alg=alg, ach=ach, peak=peak, peak_src=peak_src,
                kernel_ms={n: round(v_[0], 3) for n, v_ in sorted(prof.items(), key=lambda kv: -kv[1][0])}, cpu=cpu,
                shape=dict(T=T, N=N, r=r, p=p, n_rep=n_rep, em_iters=mi, H_irf=H_irf, H_fc=H_fc, fc_rows=fc_rows, observed_frac=obs_frac))


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    X2, th2, p2 = _fit_c2(lib, 50)
    c2 = _workload(lib, torch, dev, X2, th2, p2, args.reps, 50, 24, 0, 0, args.steps, args.warmup, args.no_cpu)
    X1, th1, p1 = _fit_c1(lib)
    c1 = _workload(lib, torch, dev, X1, th1, p1, args.reps, 20, 24, 8, 12, args.steps, args.warmup, args.no_cpu)
    roof = {"bound": "hbm", "kernel": "k_ss_sim_project", "achieved": c2["ach"], "peak": c2["peak"], "unit": "GB/s",
            "frac": c2["ach"] / c2["peak"], "traffic": None, "peak_source": c2["peak_src"],
            "algorithmic_bytes_per_step": c2["alg"], "kernel_ms_per_step": c2["proj_ms"],
            "em_share_of_step": c2["em_share"], "simulator_share_of_step": c2["sim_share"], "kernel_ms": c2["kernel_ms"],
            "c1": {"achieved": c1["ach"], "frac": c1["ach"] / c1["peak"], "algorithmic_bytes_per_step": c1["alg"],
                   "em_share_of_step": c1["em_share"], "simulator_share_of_step": c1["sim_share"], "kernel_ms": c1["kernel_ms"]},
            "note": "k_ss_sim_project bytes: 8 T N per replicate written (the panels), 8 T r per replicate and series tile read (the "
                    "factors), and per tile of 8 replicates the template (8 T N) and the loadings; over the data-sheet rate"}
    line = {"metric": f"parametric bootstrap replicates/sec (C2-shaped model N={bench.NS} r={bench.R_} T={bench.T_}, 50 EM iterations, "
                      f"fused path)", "value": c2["value"], "unit": "replicates/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": c2["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "C2: synthetic (device-generated frozen DGP, SURVEY.md 8d); C1: hom_fac_1 (tests/golden)",
            "config": {"workload": f"{args.reps} replicates per step of dfm_ss_bootstrap: simulate at the fitted parameters, EM from "
                                   f"them, align, IRF of all shocks (H_irf = 24)", **c2["shape"], "all_status_ok": c2["all_status_ok"],
                       "n_failed": c2["n_failed"], "e2e_equals_device": c2["e2e_equals_device"],
                       "c1": {**c1["shape"], "value": c1["value"], "unit": "replicates/s", "ms_per_step": c1["ms_per_step"],
                              "e2e_value": c1["e2e_value"], "n_failed": c1["n_failed"], "all_status_ok": c1["all_status_ok"],
                              "e2e_equals_device": c1["e2e_equals_device"], "gpu_launches": c1["launches"], "cpu_baseline": c1["cpu"]}},
            "e2e": {"value": c2["e2e_value"], "unit": "replicates/s", "h2d_bytes_per_step": c2["h2d"], "d2h_bytes_per_step": c2["d2h"],
                    "ms_per_step": c2["e2e_ms"], "c1_value": c1["e2e_value"], "c1_ms_per_step": c1["e2e_ms"]},
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
    ap.add_argument("--reps", type=int, default=1000, help="replicates per step and workload")
    ap.add_argument("--json", default=None, help="also write the line to this file")
    ap.add_argument("--no-cpu", action="store_true")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
