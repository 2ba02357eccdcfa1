#!/usr/bin/env python
"""bench_proxy.py -- cost of the proxy (external instrument) identification (dfm_proxy_identification,
api.proxy_restricted_responses) on an H100:
  boot       one Figure-7-shaped model (Stock & Watson's Figure 7 block, hom_fac_1 1985Q1-2014Q4, plain Parametric() fit, N = 139,
             r = 8, p = 4, H = 24, the smoothed path at m.em) with 3 synthetic instruments (the fit's own innovations u_t times fixed
             unit vectors plus seeded noise, NaN in the first 10 rows), n_boot = 16383 moving-block replicates (block 5, q = 4),
             device resident: the whole call, each kernel's time, and the bytes the records and outputs take against the 3.35
             TB/s HBM3 data-sheet rate;
  posterior  16 384 models (the Figure 7 estimates scaled per model) x 1 instrument x replicate 0 (n_boot = 0): the whole call;
  e2e        api.proxy_restricted_responses on the Figure 7 fit at the GPU test's sizes (4 chains, 40 + 80 sweeps, 1 replicate);
  cpu        the NumPy spec (tests/proxy_oracle.py) on one core: records (instrument x replicate) per second of the boot workload.
Prints one JSON line in bench.py's line format (value = records per second of the boot workload, whole call).

python tools/bench_proxy.py --steps K --warmup W [--json profiles/h100_bench_proxy.json]
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

H, N_INST, N_BOOT, BLOCK, Q = 24, 3, 16383, 5, 4
N_POST = 16384
HBM_TBPS = 3.35                  # H100 SXM5 HBM3 data-sheet bandwidth


def _instruments(b, F, seed=5, lead=10):
    import proxy_oracle as PO
    e = b["em"]
    eta = PO.innovations(e["A"], F, b["p"])
    u = np.linalg.solve(np.linalg.cholesky(e["Q"]), np.nan_to_num(eta).T).T
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((u.shape[1], N_INST))
    Z = u @ (W / np.linalg.norm(W, axis=0)) + 0.5 * rng.standard_normal((len(u), N_INST))
    Z[:lead] = np.nan
    return Z


def _boot(lib, torch, dev, b, F, Z, i0, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]; Tp = F.shape[0]; nr = N_BOOT + 1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(b["Lam"])), R=t(e["R"]), A=t(to_cm(e["A"])), Q=t(to_cm(e["Q"])))
    dF, dZ, dsc = t(to_cm(F)), t(to_cm(Z)), t(b["xstd"])
    o = {n: torch.empty(N_INST * nr * N * H, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    om = torch.empty(N_INST * nr * r, dtype=torch.float64, device=dev)
    ep = torch.empty(N_INST * Tp, dtype=torch.float64, device=dev)
    st = torch.empty(N_INST, dtype=torch.int32, device=dev)

    def call():
        lib.proxy_identification_raw({n: v.data_ptr() for n, v in dm.items()}, dF.data_ptr(), dZ.data_ptr(), None, N, r, p, 1, Tp, H,
                                     N_INST, i0, Q, BLOCK, N_BOOT, 11, dsc.data_ptr(), MEM_DEVICE, omega=om.data_ptr(),
                                     eps=ep.data_ptr(), status=st.data_ptr(), **{n: v.data_ptr() for n, v in o.items()})
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
    rec = N_INST * nr
    # bytes: k_iv_rot writes the r x r x H records and reads Psi; k_series_resp reads the records and the loadings and writes
    # resp and fevd (N x H each); counted once per record
    b_rot = rec * r * r * H * 8
    b_resp = rec * (r * r * H * 8 + 2 * N * H * 8)
    kr, ks = per("k_iv_rot"), per("k_series_resp")
    return dict(n_inst=N_INST, n_boot=N_BOOT, block=BLOCK, q=Q, Tp=Tp, records=rec, call_ms=ms, records_per_s=rec / (ms * 1e-3),
                k_iv_prep_ms=per("k_iv_prep"), k_iv_boot_ms=per("k_iv_boot"), k_iv_rot_ms=kr, k_series_resp_ms=ks,
                kernels_ms={n: round(v[0] / K_, 4) for n, v in prof.items()},
                k_iv_rot_bytes=b_rot, k_series_resp_bytes=b_resp,
                k_iv_rot_tbps=b_rot / (kr * 1e-3) / 1e12 if kr > 0 else 0.0,
                k_series_resp_tbps=b_resp / (ks * 1e-3) / 1e12 if ks > 0 else 0.0,
                frac_hbm_k_series_resp=(b_resp / (ks * 1e-3) / 1e12) / HBM_TBPS if ks > 0 else 0.0,
                launches_per_call=launches, status_ok=bool((st.cpu().numpy() == 0).all()))


def _posterior(lib, torch, dev, b, F, Z, i0, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]; B = N_POST; Tp = F.shape[0]
    s = 1.0 + 0.05 * np.linspace(-1, 1, B)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(np.stack([b["Lam"]] * B) * s[:, None, None])), R=t(np.stack([e["R"]] * B).ravel()),
              A=t(to_cm(np.stack([e["A"]] * B) * (s[:, None, None] ** 0.1))), Q=t(to_cm(np.stack([e["Q"]] * B) * s[:, None, None])))
    dF, dZ, dsc = t(to_cm(np.stack([F] * B))), t(to_cm(Z[:, :1])), t(b["xstd"])
    o = {n: torch.empty(B * N * H, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    st = torch.empty(B, dtype=torch.int32, device=dev)
    ids = np.arange(B, dtype=np.uint64)

    def call():
        lib.proxy_identification_raw({n: v.data_ptr() for n, v in dm.items()}, dF.data_ptr(), dZ.data_ptr(), ids, N, r, p, B, Tp, H, 1,
                                     i0, Q, BLOCK, 0, 11, dsc.data_ptr(), MEM_DEVICE, status=st.data_ptr(),
                                     **{n: v.data_ptr() for n, v in o.items()})
        lib.sync()

    for _ in range(W_):
        call()
    ms = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
    lib.profile(True)
    call()
    prof = lib.profile_report(); lib.profile(False)
    return dict(n_model=B, n_inst=1, n_boot=0, H=H, call_ms=ms, models_per_s=B / (ms * 1e-3),
                kernels_ms={n: round(v[0], 4) for n, v in prof.items()}, status_ok=bool((st.cpu().numpy() == 0).all()))


def _e2e(lib, torch, m, z, i0):
    import dynamic_factor_models_b200 as D
    kw = dict(n_chain=4, n_burn=40, n_keep=80, boot_per_draw=1, block=BLOCK, seed=7, lib=lib)
    D.proxy_restricted_responses(m, z, i0, 12, **kw)                           # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o = D.proxy_restricted_responses(m, z, i0, 12, **kw)
    torch.cuda.synchronize()
    return dict(ms=(time.perf_counter() - t0) * 1e3, status_ok=bool((o["status"] == 0).all() and (o["proxy_status"] == 0).all()),
                n_chain=4, n_burn=40, n_keep=80, boot_per_draw=1, H=12)


def _cpu(b, F, Z, i0, n_boot=64):
    import proxy_oracle as PO
    e = b["em"]
    t0 = time.perf_counter()
    PO.identify(b["Lam"], e["R"], e["A"], e["Q"], F, Z, b["p"], H, i0, q=Q, block=BLOCK, n_boot=n_boot, seed=11, scale=b["xstd"])
    s = time.perf_counter() - t0
    n = N_INST * (n_boot + 1)
    return dict(value=n / s, unit="records/s", cores=1, kind="spec", sample=n,
                note="tests/proxy_oracle.py (NumPy: innovations, block resamples, omega, the HAC first stage and each record's "
                     "responses and FEVD), the boot workload's model and instruments, one thread")


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    from dynamic_factor_models_b200.api import _history_rows, _state_space_block
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    m, used = BS._figure7(lib)
    b = _state_space_block(m, 0, lib, "bench")
    _, _, F = _history_rows(m, b, None, "bench")
    Z = _instruments(b, F)
    i0 = used.index(BS.OIL[1])
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    boot = _boot(lib, torch, dev, b, F, Z, i0, args.steps, args.warmup)
    post = _posterior(lib, torch, dev, b, F, Z, i0, args.steps, args.warmup)
    e2e = _e2e(lib, torch, m, Z[:, 0], i0)
    clk = clocks.stop()
    cpu = _cpu(b, F, Z, i0)
    fr = boot["frac_hbm_k_series_resp"]
    roof = {"bound": "hbm" if fr >= 0.5 else "neither", "kernel": "k_series_resp", "achieved": boot["k_series_resp_tbps"],
            "peak": HBM_TBPS, "unit": "TB/s", "frac": fr,
            "traffic": {"k_series_resp_bytes": boot["k_series_resp_bytes"], "k_iv_rot_bytes": boot["k_iv_rot_bytes"]},
            "peak_source": "H100 SXM5 data sheet (3.35 TB/s HBM3)",
            "note": "bytes = the records k_series_resp reads (r r H doubles each) and the resp and fevd it writes (N H doubles each), "
                    "once per record; the loadings it re-reads per record (from L2) and its FP64 work are not counted"}
    value = boot["records_per_s"]
    line = {"metric": f"proxy-identification records/sec (one Figure-7-shaped model N=139 r=8 p=4 H={H}, {N_INST} instruments, "
                      f"n_boot={N_BOOT})",
            "value": value, "unit": "records/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": boot["call_ms"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": value / cpu["value"], "dtype": "f64",
            "data": "hom_fac_1 (tests/golden), 1985Q1-2014Q4, plain Parametric() fit (20 EM iterations), smoothed path at m.em, "
                    "synthetic instruments from its innovations",
            "config": {"workload": "dfm_proxy_identification (3 instruments, n_boot 16383, device resident); 16384 models x 1 instrument "
                                   "x replicate 0; api.proxy_restricted_responses at 4 chains x (40 + 80) sweeps x 1 replicate",
                       "N": int(b["Lam"].shape[0]), "r": int(b["Lam"].shape[1]), "p": int(b["p"]), "H": H, "Tp": int(F.shape[0]),
                       "boot": boot, "posterior": post, "proxy_restricted_responses": e2e},
            "e2e": {"value": value, "unit": "records/s", "ms_per_step": boot["call_ms"], "posterior_call_ms": post["call_ms"],
                    "proxy_restricted_responses_ms": e2e["ms"]},
            "gpu_launches": boot["launches_per_call"], "clocks": clk, "roofline": roof, "cpu_baseline": cpu}
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
