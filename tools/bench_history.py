#!/usr/bin/env python
"""bench_history.py -- cost of the historical decompositions (dfm_historical_decomposition, api.identified_history) on an H100:
  kernels    dfm_historical_decomposition on 4096 Figure-7-shaped models (Stock & Watson's Figure 7 fit, hom_fac_1 1985Q1-2014Q4,
             N = 139, r = 8, p = 4, Tp = 120, the oil series pinned to e_1; Lam, R, A, Q and the smoothed path scaled per model:
             about 4 chains x 1000 Gibbs draws), t0 = p - 1, device resident, all four outputs, n_shock = 1 and n_shock = r:
             kernel times of k_hd_paths and k_hd_series, the bytes k_hd_series writes and reads and the flops it does (from the
             shapes), its HBM rate and share of the 3.35 TB/s HBM3 data-sheet rate, its FP64 rate and share of the 34 TFLOP/s
             FP64 data-sheet rate (the larger share names the bound), and the time of the whole call;
  e2e        api.identified_history on the Figure 7 model at the GPU test's chain sizes (4 chains, 40 + 80 sweeps), end to end.
Prints one JSON line in bench.py's line format (value = models decomposed per second at n_shock = r, whole call).

python tools/bench_history.py --steps K --warmup W [--json profiles/h100_bench_history.json]
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

OIL = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]
PEAK_HBM_TBS = 3.35              # H100 SXM5 HBM3 data-sheet rate
PEAK_FP64_TFLOPS = 34.0          # H100 SXM5 FP64 (non-tensor) data-sheet rate
N_MODEL = 4096


def _figure7(lib):
    """The Figure 7 fit of tests/test_gpu_identified.py (20 restricted EM iterations)."""
    import dynamic_factor_models_b200 as D
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    data, incl = z["all_bpdata"], z["all_inclcode"]
    names = [str(s) for s in z["all_names"]]
    calds = [tuple(x) for x in z["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    r = 8
    Rm = np.eye(r); rv = np.r_[1.0, np.zeros(r - 1)]
    used = [n for n, c in zip(names, incl) if c == 1]
    m = D.DFMModel(data, incl, 20, 40, i0, i1, 0, r, 1e-8, 4, 4)
    gf = D.construct_constraint(OIL, used, Rm, rv); gfl = D.construct_constraint(OIL, names, Rm, rv)
    D.estimate(m, D.Parametric(max_iter=20, tol=0.0), lam_constr_f=gf, lam_constr_fl=gfl, lam_constr_em=gf, lib=lib)
    return m


def _kernels(lib, torch, dev, m, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    from dynamic_factor_models_b200.api import _state_space_block, _history_rows
    b = _state_space_block(m, 0, lib, "bench")
    e = m.em
    _, t0, F = _history_rows(m, b, None, "bench")
    N, r = b["Lam"].shape; p = b["p"]; Tp = F.shape[0]; B = N_MODEL
    s = 1.0 + 0.05 * np.linspace(-1, 1, B)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Lam = np.stack([b["Lam"]] * B) * s[:, None, None]
    dm = dict(Lam=t(to_cm(Lam)), R=t(np.stack([e["R"]] * B).ravel()), A=t(to_cm(np.stack([e["A"]] * B) * (s[:, None, None] ** 0.1))),
              Q=t(to_cm(np.stack([e["Q"]] * B) * s[:, None, None])))
    dF = t(to_cm(np.stack([F] * B) * s[:, None, None]))
    dsc = t(b["xstd"])
    n_in = int((~np.isnan(b["Lam"][:, 0])).sum())
    out = {}
    for ns in (1, r):
        nc = ns + 2
        o = dict(shocks=torch.empty(B * Tp * r, dtype=torch.float64, device=dev),
                 contrib=torch.empty(B * N * Tp * ns, dtype=torch.float64, device=dev),
                 rest=torch.empty(B * N * Tp, dtype=torch.float64, device=dev), base=torch.empty(B * N * Tp, dtype=torch.float64, device=dev))
        st = torch.empty(B, dtype=torch.int32, device=dev)

        def call():
            lib.historical_decomposition_raw({n: v.data_ptr() for n, v in dm.items()}, dF.data_ptr(), N, r, p, Tp, t0, ns, B, dsc.data_ptr(),
                                             MEM_DEVICE, status=st.data_ptr(), **{n: v.data_ptr() for n, v in o.items()})
            lib.sync()

        for _ in range(W_):
            call()
        l0 = lib.launches
        call()
        launches = lib.launches - l0
        ms_call = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
        lib.profile(True)
        for _ in range(K_):
            call()
        prof = lib.profile_report(); lib.profile(False)
        kname = next(n for n in prof if n.startswith("k_hd_series"))
        kt = prof[kname][0] / prof[kname][1]
        kp = prof["k_hd_paths"][0] / prof["k_hd_paths"][1]
        wbytes = 8.0 * B * N * Tp * (ns + 2)                              # contrib, rest, base: every cell written once
        rbytes = 8.0 * B * (nc * Tp * r + N * r + N) + 8.0 * N            # recursions once per model, Lam, R, scale
        flops = 2.0 * B * n_in * Tp * nc * r                              # lam_i' y_{c,t} for the series in the model
        hbm = (wbytes + rbytes) / (kt * 1e-3) / 1e12
        tfl = flops / (kt * 1e-3) / 1e12
        t_mem, t_fl = (wbytes + rbytes) / (PEAK_HBM_TBS * 1e12), flops / (PEAK_FP64_TFLOPS * 1e12)
        sv = st.cpu().numpy()
        out[f"n_shock_{ns}"] = dict(call_ms=ms_call, k_hd_paths_ms=kp, k_hd_series_ms=kt, kernels_ms={n: round(v[0] / v[1], 4) for n, v in prof.items()},
                                   bytes_written=wbytes, bytes_read=rbytes, flops=flops, hbm_tbs=hbm, frac_hbm_datasheet=hbm / PEAK_HBM_TBS,
                                   fp64_tflops=tfl, frac_fp64_datasheet=tfl / PEAK_FP64_TFLOPS, bound="hbm" if t_mem >= t_fl else "fp64",
                                   frac_of_bound=max(t_mem, t_fl) / (kt * 1e-3), launches_per_call=launches,
                                   status_ok=bool((sv == 0).all()))
        del o
    return dict(n_model=B, N=N, r=r, p=p, Tp=Tp, t0=t0, **out)


def _e2e(lib, torch, m):
    import dynamic_factor_models_b200 as D
    kw = dict(shocks=1, n_chain=4, n_burn=40, n_keep=80, seed=7, lib=lib)
    D.identified_history(m, **kw)                                        # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o = D.identified_history(m, **kw)
    torch.cuda.synchronize()
    return dict(ms=(time.perf_counter() - t0) * 1e3, status_ok=bool((o["status"] == 0).all()), n_chain=4, n_burn=40, n_keep=80)


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    m = _figure7(lib)
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    ks = _kernels(lib, torch, dev, m, args.steps, args.warmup)
    e2e = _e2e(lib, torch, m)
    clk = clocks.stop()
    r = ks["r"]
    r1, rr = ks["n_shock_1"], ks[f"n_shock_{r}"]
    roof = {"bound": rr["bound"], "kernel": "k_hd_series", "achieved": rr["hbm_tbs"], "peak": PEAK_HBM_TBS, "unit": "TB/s",
            "frac": rr["hbm_tbs"] / PEAK_HBM_TBS, "traffic": {"bytes_written": rr["bytes_written"], "bytes_read": rr["bytes_read"]},
            "peak_source": "H100 SXM5 data sheet (3.35 TB/s HBM3, 34 TFLOP/s FP64)", "history": ks,
            "note": "k_hd_series at n_shock = r; bytes = contrib, rest, base written once, the recursions, Lam, R read once per "
                    "model; flops = 2 r (n_shock + 2) per (series in the model, period); the bound is the larger of bytes / 3.35 TB/s "
                    "and flops / 34 TFLOP/s"}
    value = ks["n_model"] / (rr["call_ms"] * 1e-3)
    line = {"metric": f"historical decompositions/sec ({ks['n_model']} Figure-7-shaped models N={ks['N']} r={r} p={ks['p']} "
                      f"Tp={ks['Tp']}, n_shock = r)",
            "value": value, "unit": "models/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": rr["call_ms"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "hom_fac_1 (tests/golden), 1985Q1-2014Q4, oil series pinned to e_1",
            "config": {"workload": f"dfm_historical_decomposition on {ks['n_model']} models, device resident, shocks / contrib / rest / "
                                   "base written, t0 = p - 1, n_shock = 1 and r; api.identified_history at 4 chains x (40 + 80) sweeps",
                       "N": ks["N"], "r": r, "p": ks["p"], "Tp": ks["Tp"], "t0": ks["t0"], "n_model": ks["n_model"],
                       "n_shock_1": r1, f"n_shock_{r}": rr, "identified_history": e2e},
            "e2e": {"value": value, "unit": "models/s", "ms_per_step": rr["call_ms"], "identified_history_ms": e2e["ms"]},
            "gpu_launches": rr["launches_per_call"], "clocks": clk, "roofline": roof, "cpu_baseline": None}
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
    ap.add_argument("--json", default=None)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
