#!/usr/bin/env python
"""bench_forecast.py -- throughput of dfm_kalman_smooth (smoothing, nowcasting, forecasting at fixed parameters) on the
C5 workload of bench.py: 1250 C2-shaped panels per GPU (N=200, r=8, T=500) at the parameters after bench.py's 50 EM
iterations, H = 8 forecast periods.  Prints one JSON line in the format of bench.py's lines (value = panels/s device
resident, e2e = pinned host buffers through the C ABI, roofline of k_ss_project, clocks, launches, CPU arm = the NumPy
spec on a sample of panels).  Inputs, timing, clocks and the --dump-outputs format are bench.py's own helpers.

python tools/bench_forecast.py --steps K --warmup W [--horizon H] [--dump-outputs DIR] [--no-cpu]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def run(args):
    """The C5 shard (C2-shaped panels N=200, r=8, T=500) at the parameters its EM step ends with, then
    dfm_kalman_smooth with H periods: smoothed factors, the H-period forecasts and, for every cell, the common component, the
    imputed / forecast value and its variance.  `value` = panels/s device resident; `e2e` = the same with pinned host
    buffers.  Roofline of k_ss_project: 8 N (T + 3 (T + H)) bytes per panel (one read of the panel, common / xhat / xvar
    written)."""
    torch, dist, world, rank, local, dev = bench._dist_setup()
    from dynamic_factor_models_b200 import Library
    from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST
    import ctypes as C
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    B, iters, K_, W_, H = args.panels, args.em_iters, args.steps, args.warmup, args.horizon
    N, r, T, p = bench.NS, bench.R_, bench.T_, bench.P_
    k = r * p; Tp = T + H
    f64 = lambda n: torch.empty(n, dtype=torch.float64, device=dev)
    dX, dF0 = f64(B * T * N), f64(B * T * r)
    lib.simulate_panels_raw(rank * B, B, N, r, T, bench.SEED, dX.data_ptr())
    lib.estimate_factor_raw(dX.data_ptr(), T, N, r, B, MEM_DEVICE, F=dF0.data_ptr(), max_iter=1)
    d0 = {n: f64(sz) for n, sz in dict(Lam=B * N * r, R=B * N, A=B * r * k, Q=B * r * r).items()}
    lib.check(lib.lib.dfm_em_init_from_factors(lib.h, C.c_void_p(dX.data_ptr()), C.c_void_p(dF0.data_ptr()), T, N, r, p, B, MEM_DEVICE,
                                               *[C.c_void_p(d0[n].data_ptr()) for n in ("Lam", "R", "A", "Q")]), "em_init")
    # the parameters after the c5 EM step (em_iters iterations)
    par = {n: f64(sz) for n, sz in dict(Lam=B * N * r, R=B * N, A=B * r * k, Q=B * r * r, loglik=B * iters).items()}
    dit = torch.empty(B, dtype=torch.int32, device=dev); dst = torch.empty(B, dtype=torch.int32, device=dev)
    lib.em_kalman_raw(dX.data_ptr(), T, N, r, p, B, iters, 0.0, {n: d0[n].data_ptr() for n in d0},
                      dict(Lam=par["Lam"].data_ptr(), R=par["R"].data_ptr(), A=par["A"].data_ptr(), Q=par["Q"].data_ptr(),
                           loglik=par["loglik"].data_ptr(), iters=dit.data_ptr(), status=dst.data_ptr()), MEM_DEVICE, args.path)
    lib.sync()
    params_d = {n: par[n].data_ptr() for n in ("Lam", "R", "A", "Q")}
    sizes = dict(F=B * Tp * r, common=B * Tp * N, xhat=B * Tp * N, xvar=B * Tp * N, loglik=B)
    dout = {n: f64(sz) for n, sz in sizes.items()}
    sst = torch.empty(B, dtype=torch.int32, device=dev)
    out_d = {**{n: t.data_ptr() for n, t in dout.items()}, "status": sst.data_ptr()}

    def step_device():
        lib.kalman_smooth_raw(dX.data_ptr(), T, N, r, p, H, B, params_d, out_d, MEM_DEVICE)
        lib.sync()

    for _ in range(W_):
        step_device()
    clocks = bench.ClockSampler(local); clocks.start()
    l0 = lib.launches
    ms = bench._timed(torch, dist, world, dev, step_device, K_)
    launches = lib.launches - l0
    clk = clocks.stop()
    if args.dump_outputs:
        cm = bench._cm
        bench.dump_outputs(args.dump_outputs, dict(F=cm(dout["F"], B, Tp, r), common=cm(dout["common"], B, Tp, N), xhat=cm(dout["xhat"], B, Tp, N),
                                                   xvar=cm(dout["xvar"], B, Tp, N), loglik=dout["loglik"].cpu(), status=sst.cpu()))
    value = world * B * K_ / (ms * 1e-3)
    status_ok = bool((sst == 0).all().item())

    # ---- e2e: pinned host buffers (upload of panels + parameters, download of the outputs inside the call)
    hX = dX.cpu().pin_memory()
    hpar = {n: par[n].cpu().pin_memory() for n in ("Lam", "R", "A", "Q")}
    hout = {n: torch.empty(sz, dtype=torch.float64).pin_memory() for n, sz in sizes.items()}
    hst = torch.empty(B, dtype=torch.int32).pin_memory()
    out_h = {**{n: t.data_ptr() for n, t in hout.items()}, "status": hst.data_ptr()}

    def step_e2e():
        lib.kalman_smooth_raw(hX.data_ptr(), T, N, r, p, H, B, {n: t.data_ptr() for n, t in hpar.items()}, out_h, MEM_HOST)

    step_e2e()
    Ke = max(2, min(K_, 3))
    ms_e = bench._timed(torch, dist, world, dev, step_e2e, Ke)
    h2d = 8 * (hX.numel() + sum(t.numel() for t in hpar.values()))
    d2h = 8 * sum(t.numel() for t in hout.values()) + 4 * B

    # ---- roofline of k_ss_project: per-kernel CUDA-event timing of one profiled step (outside the timed region)
    lib.profile(True); step_device(); prof = lib.profile_report(); lib.profile(False)
    tot = sum(v_[0] for v_ in prof.values()) or 1.0
    dom = max(prof, key=lambda n: prof[n][0])
    peak, peak_src = bench._peak()
    p_ms, p_cnt = prof["k_ss_project"]
    alg = 8.0 * N * (T + 3 * Tp) * B
    ach = alg / (p_ms * 1e-3) / 1e9
    roof = {"bound": "hbm", "kernel": "k_ss_project", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "traffic": None,
            "peak_source": peak_src, "kernel_share_of_step": p_ms / tot, "dominant_kernel_of_step": dom, "avg_launch_ms": p_ms / p_cnt,
            "algorithmic_bytes_per_launch": alg / p_cnt,
            "note": "8 N (T + 3 (T + H)) bytes per panel: one read of the panel, common / xhat / xvar written",
            "kernel_ms": {n: round(v_[0], 3) for n, v_ in sorted(prof.items(), key=lambda kv: -kv[1][0])}}
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from forecast_oracle import smooth_forecast
        nb = 4
        Xh = bench._cm(dX[:nb * T * N], nb, T, N)
        ph = dict(Lam=bench._cm(par["Lam"][:nb * N * r], nb, N, r), R=par["R"][:nb * N].cpu().numpy().reshape(nb, N),
                  A=bench._cm(par["A"][:nb * r * k], nb, r, k), Q=bench._cm(par["Q"][:nb * r * r], nb, r, r))
        t0 = time.perf_counter()
        for b in range(nb):
            smooth_forecast(Xh[b], ph["Lam"][b], ph["R"][b], ph["A"][b], ph["Q"][b], None, p, H)
        dt = time.perf_counter() - t0
        cpu = {"value": nb / dt, "unit": "panels/s", "cores": 1, "kind": "port",
               "sample": f"{nb} panels, NumPy spec smooth_forecast (tests/forecast_oracle.py: Kalman filter + RTS smoother on the padded panel "
                         f"+ projection), 1 process, {dt:.2f} s"}
    if rank == 0:
        print(json.dumps({"metric": f"forecast panels/sec (C5 shard, N={N} r={r} T={T}, H={H})", "value": value, "unit": "panels/s",
                          "n_gpus": world, "steps": K_, "warmup": W_, "ms_per_step": ms / K_, "higher_is_better": True, "scaling": "weak",
                          "vs_baseline": None, "dtype": "f64", "data": "synthetic (device-generated frozen DGP, SURVEY.md 8d)",
                          "config": {"workload": f"C5 shard: {B} C2-shaped panels/GPU at the parameters after {iters} EM iterations; "
                                                 f"dfm_kalman_smooth with H={H}: F, common, xhat, xvar, loglik",
                                     "panels_per_gpu": B, "H": H, "em_iters_before": iters, "all_status_ok": status_ok,
                                     "l2": f"inputs {B * T * N * 8 / 1e6:.0f} MB/GPU, outputs {3 * B * Tp * N * 8 / 1e6:.0f} MB/GPU, "
                                           f"L2 {bench._l2_mb(dev):.0f} MB"},
                          "e2e": {"value": world * B * Ke / (ms_e * 1e-3), "unit": "panels/s", "h2d_bytes_per_step": h2d,
                                  "d2h_bytes_per_step": d2h, "ms_per_step": ms_e / Ke},
                          "gpu_launches": int(launches), "clocks": clk, "roofline": roof, "cpu_baseline": cpu}))
    if world > 1:
        dist.destroy_process_group()
    lib.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--panels", type=int, default=1250, help="panels per GPU (C5 shard = 10000/8)")
    ap.add_argument("--em-iters", type=int, default=50, help="EM iterations that produce the parameters (bench.py's c5 step)")
    ap.add_argument("--horizon", type=int, default=8, help="forecast periods H")
    ap.add_argument("--path", type=int, default=0, help="dfm_em_kalman path of the EM step that produces the parameters")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step to DIR/<name>.npy (float64, <= 64 MB in all)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
