#!/usr/bin/env python
"""bench_narrative.py -- cost of narrative sign restrictions (dfm_narrative_sign_restrictions, api.narrative_restricted_responses)
on an H100, on the Figure-7-shaped model of tools/bench_sign.py (N = 139, r = 8, p = 4, H = 24, Tp = 120):
  set_most     n_rot = 2^24 candidates, n_keep = 4096, device resident: the 16 oil sign rows plus two narrative rows at 1990Q3
               (shock 1 positive; shock 1 the most important contributor to the first oil series, h = 0); whole call,
               candidates/s and per-kernel ms;
  set_over     the same with the second row overwhelming (kind 2) over 1990Q3 .. 1990Q4 (h = 1);
  omega        k_narr_omega of set_most (n_keep = 4096 slots x n_sim = 2^14): simulations/s, FP64 flops per simulation counted
               from the rows (fma = 2; Box-Muller and Philox not counted), and the share of the 34 TFLOP/s FP64 data-sheet rate;
  posterior    16 384 models (the Figure 7 estimates scaled per model) x 16 candidates, set_most's rows, whole call;
  e2e          api.narrative_restricted_responses on the Figure 7 fit at the GPU test's sizes (4 chains, 40 + 80 sweeps, 4
               rotations, n_sim = 2^14);
  cpu          the NumPy spec (tests/narrative_oracle.py) on one core: candidates/s of set_most.
Prints one JSON line in bench.py's line format (value = candidates per second of set_most, whole call).

python tools/bench_narrative.py --steps K --warmup W [--json profiles/h100_bench_narrative.json]
"""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):   # (the CPU arm runs on one core)
    os.environ.setdefault(_v, "1")

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import bench_sign as BS  # noqa: E402

PEAK_FP64_TFLOPS = 34.0          # H100 SXM5 FP64 (non-tensor) data-sheet rate
N_ROT, N_KEEP, H, N_SIM = 1 << 24, 4096, 24, 1 << 14
N_POST, ROT_POST = 16384, 16


def _narrative(m, used, row, kind):
    """Shock 1 positive at 1990Q3, and shock 1 most important (kind 1, h = 0) or overwhelming (kind 2, h = 1) for the first oil
    series: the library's six arrays."""
    i = used.index(BS.OIL[0])
    h = 0 if kind == 1 else 1
    rows = [(0, 1, 0, row, 0, 1), (kind, 1, i, row, h, 1)]
    return [np.array([rw[q] for rw in rows], np.int64) for q in range(6)]


def _omega_flops(narr, r):
    """FP64 flops per simulation: kind 0 none; kinds 1 / 2: (h + 1) r fma and r |.| and compares; kind 3: (h + 1) fma."""
    f = 0.0
    for kd, h in zip(narr[0], narr[4]):
        f += 0.0 if kd == 0 else (2.0 * (h + 1) * (r if kd in (1, 2) else 1) + (2.0 * r if kd in (1, 2) else 1.0))
    return f


def _set(lib, torch, dev, b, F, rows, narr, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]; Tp = F.shape[0]
    ns = 1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(b["Lam"])), R=t(e["R"]), A=t(to_cm(e["A"])), Q=t(to_cm(e["Q"])))
    dF, dsc = t(to_cm(F)), t(b["xstd"])
    o = {n: torch.empty(N_KEEP * N * H * ns, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    rot = torch.empty(N_KEEP * r * r, dtype=torch.float64, device=dev)
    eps = torch.empty(N_KEEP * Tp * ns, dtype=torch.float64, device=dev)
    w = torch.empty(N_KEEP, dtype=torch.float64, device=dev)
    nok = torch.empty(N_KEEP, dtype=torch.int64, device=dev)
    na, ca = torch.empty(1, dtype=torch.int64, device=dev), torch.empty(N_KEEP, dtype=torch.int64, device=dev)
    st = torch.empty(1, dtype=torch.int32, device=dev)

    def call():
        lib.narrative_sign_restrictions_raw({n: v.data_ptr() for n, v in dm.items()}, dF.data_ptr(), None, N, r, p, 1, H, ns, N_ROT, N_KEEP,
                                            11, Tp, N_SIM, rows, narr, dsc.data_ptr(), MEM_DEVICE, n_accept=na.data_ptr(),
                                            cand=ca.data_ptr(), rot=rot.data_ptr(), status=st.data_ptr(), n_ok=nok.data_ptr(),
                                            weight=w.data_ptr(), eps=eps.data_ptr(), **{n: v.data_ptr() for n, v in o.items()})
        lib.sync()

    for _ in range(W_):
        call()
    l0 = lib.launches
    call()
    launches = lib.launches - l0
    ms = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
    lib.profile(True)
    for _ in range(K_):
        call()
    prof = lib.profile_report(); lib.profile(False)
    per = lambda n: prof[n][0] / K_ if n in prof else 0.0
    nacc = int(na.cpu()[0])
    nk = min(nacc, N_KEEP)
    wv = w.cpu().numpy()[:nk]
    fin = np.isfinite(wv)
    return dict(rows=int(len(rows[0])), narrative_rows=int(len(narr[0])), narrative_kinds=[int(v) for v in narr[0]], n_rot=N_ROT,
                n_keep=N_KEEP, n_sim=N_SIM, Tp=Tp, call_ms=ms, cand_per_s=N_ROT / (ms * 1e-3), k_narr_cand_ms=per("k_narr_cand"),
                k_sign_pick_ms=per("k_sign_pick"), k_narr_rot_ms=per("k_narr_rot"), k_narr_omega_ms=per("k_narr_omega"),
                kernels_ms={n: round(v[0] / K_, 4) for n, v in prof.items()}, n_accept=nacc, accept_rate=nacc / N_ROT, n_kept=nk,
                ess=float(wv[fin].sum() ** 2 / (wv[fin] ** 2).sum()) if fin.any() else 0.0, n_zero_omega=int((~fin).sum()),
                launches_per_call=launches, status_ok=bool(int(st.cpu()[0]) == 0))


def _posterior(lib, torch, dev, b, F, rows, narr, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]; B = N_POST; Tp = F.shape[0]
    s = 1.0 + 0.05 * np.linspace(-1, 1, B)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(np.stack([b["Lam"]] * B) * s[:, None, None])), R=t(np.stack([e["R"]] * B).ravel()),
              A=t(to_cm(np.stack([e["A"]] * B) * (s[:, None, None] ** 0.1))), Q=t(to_cm(np.stack([e["Q"]] * B) * s[:, None, None])))
    dF = t(to_cm(np.stack([F] * B)))
    dsc = t(b["xstd"])
    o = {n: torch.empty(B * ROT_POST * N * H, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    w = torch.empty(B * ROT_POST, dtype=torch.float64, device=dev)
    na, st = torch.empty(B, dtype=torch.int64, device=dev), torch.empty(B, dtype=torch.int32, device=dev)
    ids = np.arange(B, dtype=np.uint64)

    def call():
        lib.narrative_sign_restrictions_raw({n: v.data_ptr() for n, v in dm.items()}, dF.data_ptr(), ids, N, r, p, B, H, 1, ROT_POST,
                                            ROT_POST, 11, Tp, N_SIM, rows, narr, dsc.data_ptr(), MEM_DEVICE, n_accept=na.data_ptr(),
                                            status=st.data_ptr(), weight=w.data_ptr(), **{n: v.data_ptr() for n, v in o.items()})
        lib.sync()

    for _ in range(W_):
        call()
    ms = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
    lib.profile(True)
    call()
    prof = lib.profile_report(); lib.profile(False)
    return dict(n_model=B, n_rot=ROT_POST, n_keep=ROT_POST, n_sim=N_SIM, H=H, call_ms=ms, models_per_s=B / (ms * 1e-3),
                kernels_ms={n: round(v[0], 4) for n, v in prof.items()}, accept_rate=float(na.cpu().numpy().mean() / ROT_POST),
                status_ok=bool((st.cpu().numpy() == 0).all()))


def _e2e(lib, torch, m, used, per):
    import dynamic_factor_models_b200 as D
    kw = dict(n_chain=4, n_burn=40, n_keep=80, rot_per_draw=4, seed=7, lib=lib)
    rs = BS._restrictions(used, "oil")
    narrative = [("shock", 1, per, 1), ("most", 1, used.index(BS.OIL[0]), per, 0)]
    D.narrative_restricted_responses(m, rs, narrative, 12, **kw)              # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o = D.narrative_restricted_responses(m, rs, narrative, 12, **kw)
    torch.cuda.synchronize()
    return dict(ms=(time.perf_counter() - t0) * 1e3, status_ok=bool((o["status"] == 0).all()), accept_rate=o["accept_rate"],
                ess=o["ess"], n_chain=4, n_burn=40, n_keep=80, rot_per_draw=4, n_sim=N_SIM, H=12)


def _cpu(b, F, rows, narr, n=2000):
    import narrative_oracle as NO
    e = b["em"]
    rl = [tuple(int(v[q]) for v in rows) for q in range(len(rows[0]))]
    nl = [tuple(int(v[q]) for v in narr) for q in range(len(narr[0]))]
    t0 = time.perf_counter()
    NO.identify(b["Lam"], e["R"], e["A"], e["Q"], F, b["p"], rl, nl, H, 1, n, 1, 1, seed=5)
    s = time.perf_counter() - t0
    return dict(value=n / s, unit="candidates/s", cores=1, kind="spec", sample=n,
                note="tests/narrative_oracle.py (NumPy: Philox normals, numpy.linalg.qr, the sign and narrative tests per candidate), "
                     "set_most's rows, one thread")


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    from dynamic_factor_models_b200.api import _history_rows, _sign_rows, _state_space_block
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    m, used = BS._figure7(lib)
    b = _state_space_block(m, 0, lib, "bench")
    _, _, F = _history_rows(m, b, None, "bench")
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    per = [tuple(x) for x in z["calds"]].index((1990, 3)) + 1
    row = per - m.initperiod
    rows = _sign_rows(BS._restrictions(used, "oil"), b["Xs"].shape[1], H, None, "bench")[0]
    narr = {k: _narrative(m, used, row, kd) for k, kd in (("most", 1), ("over", 2))}
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    sets = {k: _set(lib, torch, dev, b, F, rows, narr[k], args.steps, args.warmup) for k in ("most", "over")}
    post = _posterior(lib, torch, dev, b, F, rows, narr["most"], args.steps, args.warmup)
    e2e = _e2e(lib, torch, m, used, per)
    clk = clocks.stop()
    most = sets["most"]
    r = b["Lam"].shape[1]
    fl = _omega_flops(narr["most"], r)
    om_ms = most["k_narr_omega_ms"]
    sims = most["n_kept"] * N_SIM
    tfl = fl * sims / (om_ms * 1e-3) / 1e12 if om_ms > 0 else 0.0
    omega = dict(kernel="k_narr_omega", n_keep=N_KEEP, n_kept=most["n_kept"], n_sim=N_SIM, ms=om_ms,
                 sims_per_s=sims / (om_ms * 1e-3) if om_ms > 0 else 0.0, flops_per_sim=fl, fp64_tflops=tfl,
                 frac_fp64_datasheet=tfl / PEAK_FP64_TFLOPS)
    cpu = _cpu(b, F, rows, narr["most"])
    roof = {"bound": "neither" if omega["frac_fp64_datasheet"] < 0.5 else "fp64", "kernel": "k_narr_omega", "achieved": tfl,
            "peak": PEAK_FP64_TFLOPS, "unit": "TFLOP/s", "frac": tfl / PEAK_FP64_TFLOPS,
            "traffic": {"flops_per_sim": fl},
            "peak_source": "H100 SXM5 data sheet (34 TFLOP/s FP64)",
            "note": "flops = the rows' FP64 arithmetic per simulation (fma = 2); the Philox normals (integer multiplies, log, sqrt, "
                    "sin, cos), which dominate, are not counted, so the FP64 share is a lower bound"}
    value = most["cand_per_s"]
    line = {"metric": f"narrative sign-restriction candidates/sec (one Figure-7-shaped model N=139 r=8 p=4 H={H} Tp=120, 16 oil rows "
                      "+ 2 narrative rows, n_rot=2^24)",
            "value": value, "unit": "candidates/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": most["call_ms"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": value / cpu["value"], "dtype": "f64",
            "data": "hom_fac_1 (tests/golden), 1985Q1-2014Q4, plain Parametric() fit (20 EM iterations), smoothed path at m.em",
            "config": {"workload": "dfm_narrative_sign_restrictions identified set (n_rot 2^24, n_keep 4096, n_sim 2^14, device "
                                   "resident), oil rows + shock 1 positive and most important (or overwhelming) at 1990Q3; 16384 "
                                   "models x 16 candidates; api.narrative_restricted_responses at 4 chains x (40 + 80) sweeps x 4 "
                                   "rotations", "N": int(b["Lam"].shape[0]), "r": r, "p": int(b["p"]), "H": H, "Tp": int(F.shape[0]),
                       "set_most": most, "set_over": sets["over"], "omega": omega, "posterior": post,
                       "narrative_restricted_responses": e2e},
            "e2e": {"value": value, "unit": "candidates/s", "ms_per_step": most["call_ms"], "posterior_call_ms": post["call_ms"],
                    "narrative_restricted_responses_ms": e2e["ms"]},
            "gpu_launches": most["launches_per_call"], "clocks": clk, "roofline": roof, "cpu_baseline": cpu}
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
