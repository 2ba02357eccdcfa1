#!/usr/bin/env python
"""bench_simsmooth.py -- throughput of dfm_simulation_smoother (draws from the joint posterior of the factor path and the
missing / forecast cells at fixed parameters), 10,000 draws with H = 8 on two models:
  c1  the hom_fac_1 panel at its Parametric estimates (r = 8, p = 4, k = 32; estimate(m, Parametric()) with its defaults)
  c2  a C2-shaped model (N = 200, r = 8, T = 500, p = 1, k = 8) at the parameters after 50 EM iterations
Prints one JSON line: per workload draws/s with F only and with F + X (device-resident outputs), per-kernel times
(dfm_profile_*), the bytes model of k_sim_project over the HBM peak, the time of the shared E-step, the NumPy spec on one core
as the CPU arm, and the card name, power limit and SM clock sampled during the timed runs.

python tools/bench_simsmooth.py [--steps K] [--warmup W] [--draws 10000] [--horizon 8] [--json FILE] [--no-cpu]
"""
import os
for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):      # the CPU arm is one core
    os.environ.setdefault(_v, "1")
import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402

SIM_KERNELS = ("k_sim_gains", "k_sim_paths", "k_sim_project")


def c1_model(lib):
    """Standardized C1 block and its Parametric estimates, as api.posterior_draws passes them."""
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200 import api
    import parity_checks as P
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    m = P.gpu_model(z["all_bpdata"], z["all_inclcode"], 8)
    D.estimate(m, D.Parametric(), lib=lib)
    b = api._state_space_block(m, 0, lib, "bench")
    e = b["em"]
    return dict(X=b["Xs"], Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"], p=b["p"], em_iters=int(e["iters"]))


def c2_model(lib, iters=50):
    N, r, T = bench.NS, bench.R_, bench.T_
    X = lib.simulate_panels(0, 1, N, r, T, bench.SEED)[0]
    F0 = lib.estimate_factor(X, r, max_iter=1)["F"]
    Lam, Rv, A, Q = lib.em_init_from_factors(X, F0, 1)
    e = lib.em_kalman(X, Lam, Rv, A, Q, p=1, max_iter=iters, tol=0.0)
    return dict(X=X, Lam=e["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"], p=1, em_iters=int(e["iters"]))


def run_workload(torch, lib, dev, name, mod, n, H, K_, W_, no_cpu):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    X = mod["X"]; T, N = X.shape; r = mod["Lam"].shape[1]; p = mod["p"]; k = r * p; Tp = T + H
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ins = dict(X=up(to_cm(X)), Lam=up(to_cm(mod["Lam"])), R=up(np.asarray(mod["R"], float)), A=up(to_cm(mod["A"])), Q=up(to_cm(mod["Q"])),
               P0=up(to_cm(mod["P0"])))
    params = {q: ins[q].data_ptr() for q in ("Lam", "R", "A", "Q", "P0")}
    dF = torch.empty(n * Tp * r, dtype=torch.float64, device=dev)
    dX = torch.empty(n * Tp * N, dtype=torch.float64, device=dev)
    st = torch.full((1,), -1, dtype=torch.int32, device=dev)
    seed = 20261016

    def call(want_x):
        out = {"F": dF.data_ptr(), "status": st.data_ptr()}
        if want_x:
            out["X"] = dX.data_ptr()
        lib.simulation_smoother_raw(ins["X"].data_ptr(), T, N, r, p, H, n, 0, seed, params, out, MEM_DEVICE)
        lib.sync()

    res = {}
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    for want_x, key in ((False, "F"), (True, "F+X")):
        for _ in range(W_):
            call(want_x)
        ms = bench._timed(torch, None, 1, dev, lambda: call(want_x), K_)
        res[key] = {"draws_per_s": n * K_ / (ms * 1e-3), "ms_per_call": ms / K_}
    clk = clocks.stop()
    status = int(st.item())
    # per-kernel device times of one call with F + X (CUDA events, outside the timed runs)
    lib.profile(True); call(True); prof = lib.profile_report(); lib.profile(False)
    kernel_ms = {q: round(v[0], 4) for q, v in sorted(prof.items(), key=lambda kv: -kv[1][0])}
    estep_ms = sum(v[0] for q, v in prof.items() if q not in SIM_KERNELS)
    pj_ms = prof["k_sim_project"][0]
    peak, peak_src = bench._peak()
    pj_bytes = 8.0 * n * Tp * (N + r)                      # panel draws written + factor draws read (the panel tile is read once per 8 draws)
    pj_gbs = pj_bytes / (pj_ms * 1e-3) / 1e9
    out = {"model": name, "T": T, "N": N, "r": r, "p": p, "k": k, "H": H, "n_draw": n, "em_iters_of_parameters": mod["em_iters"],
           "status": status, **res, "kernel_ms_one_call_FX": kernel_ms, "estep_ms": round(estep_ms, 4),
           "k_sim_project_roofline": {"bytes_model": "8 n_draw (T+H) (N + r): panel draws written, factor draws read",
                                      "bytes": pj_bytes, "ms": round(pj_ms, 4), "achieved_gbs": pj_gbs, "peak_gbs": peak,
                                      "peak_source": peak_src, "frac_of_peak": pj_gbs / peak},
           "clocks": clk}
    if not no_cpu:
        from simsmooth_oracle import draw_prepared, normals, prepare
        t0 = time.perf_counter()
        g = prepare(X, mod["Lam"], mod["R"], mod["A"], mod["Q"], mod["P0"], p, H)
        t1 = time.perf_counter()
        nc = 5
        for d in range(nc):
            draw_prepared(g, *normals(seed, d, k, r, Tp, N))
        t2 = time.perf_counter()
        out["cpu_baseline"] = {"draws_per_s": nc / (t2 - t1), "estep_s": t1 - t0, "cores": 1, "kind": "spec",
                               "sample": f"{nc} draws of the NumPy spec (tests/simsmooth_oracle.py: draw_prepared with F and X) after "
                                         f"one prepare() ({t1 - t0:.2f} s), 1 thread"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--draws", type=int, default=10000)
    ap.add_argument("--horizon", type=int, default=8)
    ap.add_argument("--json", default=None, help="also write the JSON line to this file")
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_simsmooth.py needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"))
    props = torch.cuda.get_device_properties(dev)
    rows = [run_workload(torch, lib, dev, nm, f(lib), a.draws, a.horizon, a.steps, a.warmup, a.no_cpu)
            for nm, f in (("c1 hom_fac_1 Parametric", c1_model), ("c2-shaped", c2_model))]
    line = json.dumps({"metric": f"simulation smoother draws/sec ({a.draws} draws, H={a.horizon})", "unit": "draws/s", "gpu": props.name,
                       "steps": a.steps, "warmup": a.warmup, "dtype": "f64", "workloads": rows})
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        open(a.json, "w").write(line + "\n")
    lib.close()


if __name__ == "__main__":
    main()
