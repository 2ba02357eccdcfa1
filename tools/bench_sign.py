#!/usr/bin/env python
"""bench_sign.py -- cost of the sign-restriction identification (dfm_sign_restrictions, api.sign_restricted_responses) on an H100:
  set        the identified set of one Figure-7-shaped model (Stock & Watson's Figure 7 block, hom_fac_1 1985Q1-2014Q4, plain
             Parametric() fit, N = 139, r = 8, p = 4, H = 24), n_rot = 2^24 candidates, n_keep = 4096, device resident, under two
             restriction sets: "oil" (shock 1, the four oil series + at h = 0..3: 16 rows) and "three" (40 rows on shocks 1-3, an
             illustrative workload shape).  Candidates/s of the whole call, k_sign_cand's time, and the FP64 operations and Philox
             integer multiplies k_sign_cand needs, counted from the shapes and the share of candidates reaching each shock (from
             the NumPy spec on 20 000 candidates of the same model), against the FP64 data-sheet rate and the SMs' integer
             multiply rate at the measured SM clock;
  posterior  16 384 models (the Figure 7 estimates scaled per model) x 16 candidates, oil rows, whole call;
  e2e        api.sign_restricted_responses on the Figure 7 fit at the GPU test's sizes (4 chains, 40 + 80 sweeps, 4 rotations);
  cpu        the NumPy spec (tests/sign_oracle.py) on one core: candidates/s of the oil set.
Prints one JSON line in bench.py's line format (value = candidates per second of the oil identified set, whole call).

python tools/bench_sign.py --steps K --warmup W [--json profiles/h100_bench_sign.json]
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
import bench  # noqa: E402

OIL = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]
SHOCK2 = [("IPDMAT", 1), ("PCESVC96_Q", 1), ("USCONS", 1)]
SHOCK3 = [("TCU", 1), ("PERMIT", -1), ("HOUSTS", -1)]
PEAK_FP64_TFLOPS = 34.0          # H100 SXM5 FP64 (non-tensor) data-sheet rate
IMAD_PER_SM_CLK = 64             # 32-bit integer multiply-adds per SM per clock (sm_90)
N_ROT, N_KEEP, H = 1 << 24, 4096, 24
N_POST, ROT_POST = 16384, 16


def _figure7(lib):
    """Figure 7 block, plain Parametric() (20 EM iterations), and the estimation series' names."""
    import dynamic_factor_models_b200 as D
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    data, incl = z["all_bpdata"], z["all_inclcode"]
    names = [str(s) for s in z["all_names"]]
    calds = [tuple(x) for x in z["calds"]]
    i0, i1 = calds.index((1985, 1)) + 1, calds.index((2014, 4)) + 1
    m = D.DFMModel(data, incl, 20, 40, i0, i1, 0, 8, 1e-8, 4, 4)
    D.estimate(m, D.Parametric(max_iter=20, tol=0.0), lib=lib)
    return m, [n for n, c in zip(names, incl) if c == 1]


def _restrictions(used, which):
    rs = [(used.index(n), 1, 1, (0, 3)) for n in OIL]
    if which == "three":
        rs += [(used.index(n), 2, s, (0, 3)) for n, s in SHOCK2] + [(used.index(n), 3, s, (0, 3)) for n, s in SHOCK3]
    return rs


def _counts(b, rows, r):
    """Per candidate, from the shapes and the spec's share of candidates reaching each restricted shock: FP64 flops of the column
    algebra (Gram-Schmidt with one re-orthogonalisation, normalisation, the row tests; fma = 2) and Philox 32 x 32 -> 64-bit
    multiplies (2 per round, 10 rounds, one block per 2 normals).  The elementary functions of Box-Muller (log, sqrt, sin, cos)
    are not counted."""
    import sign_oracle as SO
    e = b["em"]; p = b["p"]
    rl = [tuple(int(v[q]) for v in rows) for q in range(len(rows[0]))]
    C = SO.row_vectors(b["Lam"], e["A"], e["Q"], p, rl, H)
    shocks = np.array([j for _, _, j, _ in rl])
    nj = int(shocks.max())
    Om = SO.omegas(123, 0, np.arange(20000), r)
    reach = np.ones(len(Om), bool)
    flops = philox = 0.0
    for j in range(1, nj + 1):
        f = reach.mean()
        sel = np.flatnonzero(shocks == j)
        col = 8.0 * (j - 1) * r + 3.0 * r + 2.0 + 2.0 * r * len(sel)        # 2 passes x (j-1) x (dot + axpy), norm + scale, tests
        flops += f * col
        philox += f * 20.0 * r / 2.0
        if len(sel):
            v = np.einsum("qa,ca->cq", C[sel], Om[:, :, j - 1])
            reach &= (v > 0).all(1) | (v < 0).all(1)
    return dict(flops_per_cand=flops, philox_mul_per_cand=philox, spec_accept=float(reach.mean()))


def _set(lib, torch, dev, b, rows, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]
    ns = int(rows[2].max())
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(b["Lam"])), R=t(e["R"]), A=t(to_cm(e["A"])), Q=t(to_cm(e["Q"])))
    dsc = t(b["xstd"])
    o = {n: torch.empty(N_KEEP * N * H * ns, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    rot = torch.empty(N_KEEP * r * r, dtype=torch.float64, device=dev)
    na, ca = torch.empty(1, dtype=torch.int64, device=dev), torch.empty(N_KEEP, dtype=torch.int64, device=dev)
    st = torch.empty(1, dtype=torch.int32, device=dev)

    def call():
        lib.sign_restrictions_raw({n: v.data_ptr() for n, v in dm.items()}, None, N, r, p, 1, H, ns, N_ROT, N_KEEP, 11, rows,
                                  dsc.data_ptr(), MEM_DEVICE, n_accept=na.data_ptr(), cand=ca.data_ptr(), rot=rot.data_ptr(),
                                  status=st.data_ptr(), **{n: v.data_ptr() for n, v in o.items()})
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
    per = lambda n: prof[n][0] / K_                                           # ms per call, summed over the call's launches
    kc = per("k_sign_cand")
    cnt = _counts(b, rows, r)
    fl, im = cnt["flops_per_cand"] * N_ROT, cnt["philox_mul_per_cand"] * N_ROT
    tfl = fl / (kc * 1e-3) / 1e12
    imul = im / (kc * 1e-3) / 1e12
    nacc = int(na.cpu()[0])
    return dict(rows=int(len(rows[0])), n_shock=ns, n_rot=N_ROT, n_keep=N_KEEP, call_ms=ms, cand_per_s=N_ROT / (ms * 1e-3),
                k_sign_cand_ms=kc, k_sign_pick_ms=per("k_sign_pick"), k_sign_rot_ms=per("k_sign_rot"),
                k_series_resp_ms=per("k_series_resp"), kernels_ms={n: round(v[0] / K_, 4) for n, v in prof.items()},
                n_accept=nacc, accept_rate=nacc / N_ROT, spec_accept_20000=cnt["spec_accept"],
                flops_per_cand=cnt["flops_per_cand"], philox_mul_per_cand=cnt["philox_mul_per_cand"], fp64_tflops=tfl,
                frac_fp64_datasheet=tfl / PEAK_FP64_TFLOPS, int_mul_tera_per_s=imul, launches_per_call=launches, status_ok=bool(int(st.cpu()[0]) == 0))


def _posterior(lib, torch, dev, b, rows, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    e = b["em"]; N, r = b["Lam"].shape; p = b["p"]; B = N_POST
    s = 1.0 + 0.05 * np.linspace(-1, 1, B)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dm = dict(Lam=t(to_cm(np.stack([b["Lam"]] * B) * s[:, None, None])), R=t(np.stack([e["R"]] * B).ravel()),
              A=t(to_cm(np.stack([e["A"]] * B) * (s[:, None, None] ** 0.1))), Q=t(to_cm(np.stack([e["Q"]] * B) * s[:, None, None])))
    dsc = t(b["xstd"])
    o = {n: torch.empty(B * ROT_POST * N * H, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
    na, st = torch.empty(B, dtype=torch.int64, device=dev), torch.empty(B, dtype=torch.int32, device=dev)
    ids = np.arange(B, dtype=np.uint64)

    def call():
        lib.sign_restrictions_raw({n: v.data_ptr() for n, v in dm.items()}, ids, N, r, p, B, H, 1, ROT_POST, ROT_POST, 11, rows,
                                  dsc.data_ptr(), MEM_DEVICE, n_accept=na.data_ptr(), status=st.data_ptr(),
                                  **{n: v.data_ptr() for n, v in o.items()})
        lib.sync()

    for _ in range(W_):
        call()
    ms = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
    lib.profile(True)
    call()
    prof = lib.profile_report(); lib.profile(False)
    return dict(n_model=B, n_rot=ROT_POST, n_keep=ROT_POST, H=H, call_ms=ms, models_per_s=B / (ms * 1e-3),
                kernels_ms={n: round(v[0], 4) for n, v in prof.items()}, accept_rate=float(na.cpu().numpy().mean() / ROT_POST),
                status_ok=bool((st.cpu().numpy() == 0).all()))


def _e2e(lib, torch, m, used):
    import dynamic_factor_models_b200 as D
    kw = dict(n_chain=4, n_burn=40, n_keep=80, rot_per_draw=4, seed=7, lib=lib)
    rs = _restrictions(used, "oil")
    D.sign_restricted_responses(m, rs, 12, **kw)                           # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o = D.sign_restricted_responses(m, rs, 12, **kw)
    torch.cuda.synchronize()
    return dict(ms=(time.perf_counter() - t0) * 1e3, status_ok=bool((o["status"] == 0).all()), accept_rate=o["accept_rate"], n_chain=4,
                n_burn=40, n_keep=80, rot_per_draw=4, H=12)


def _cpu(b, rows, n=20000):
    import sign_oracle as SO
    e = b["em"]
    rl = [tuple(int(v[q]) for v in rows) for q in range(len(rows[0]))]
    C = SO.row_vectors(b["Lam"], e["A"], e["Q"], b["p"], rl, H)
    sh = [j for _, _, j, _ in rl]
    t0 = time.perf_counter()
    SO.decide(C, sh, SO.omegas(5, 0, np.arange(n), b["Lam"].shape[1]))
    s = time.perf_counter() - t0
    return dict(value=n / s, unit="candidates/s", cores=1, kind="spec", sample=n,
                note="tests/sign_oracle.py (NumPy: Philox normals, batched numpy.linalg.qr, the row tests), oil rows, one thread")


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    from dynamic_factor_models_b200.api import _sign_rows, _state_space_block
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    m, used = _figure7(lib)
    b = _state_space_block(m, 0, lib, "bench")
    ns_ser = b["Xs"].shape[1]
    rows = {w: _sign_rows(_restrictions(used, w), ns_ser, H, None, "bench")[0] for w in ("oil", "three")}
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    sets = {w: _set(lib, torch, dev, b, rows[w], args.steps, args.warmup) for w in ("oil", "three")}
    post = _posterior(lib, torch, dev, b, rows["oil"], args.steps, args.warmup)
    e2e = _e2e(lib, torch, m, used)
    clk = clocks.stop()
    mhz = clk.get("sm_mhz") or clk.get("sm_max_mhz") or 1980.0
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    for s in sets.values():                       # integer-multiply shares at the SM clock measured in this run
        s["int_mul_peak_tera_per_s"] = nsm * IMAD_PER_SM_CLK * mhz * 1e6 / 1e12
        s["frac_int_mul"] = s["int_mul_tera_per_s"] / s["int_mul_peak_tera_per_s"]
        s["nearer_bound"] = "fp64" if s["frac_fp64_datasheet"] >= s["frac_int_mul"] else "int_mul"
        s["bound"] = s["nearer_bound"] if max(s["frac_fp64_datasheet"], s["frac_int_mul"]) >= 0.5 else "neither"
    cpu = _cpu(b, rows["oil"])
    oil = sets["oil"]
    near = oil["nearer_bound"]
    ach, pk, unit = ((oil["fp64_tflops"], PEAK_FP64_TFLOPS, "TFLOP/s") if near == "fp64"
                     else (oil["int_mul_tera_per_s"], oil["int_mul_peak_tera_per_s"], "Tmul/s"))
    roof = {"bound": oil["bound"], "nearer": near, "kernel": "k_sign_cand", "achieved": ach, "peak": pk, "unit": unit, "frac": ach / pk,
            "traffic": {"flops_per_cand": oil["flops_per_cand"], "philox_mul_per_cand": oil["philox_mul_per_cand"]},
            "peak_source": "H100 SXM5 data sheet (34 TFLOP/s FP64); integer multiplies: SMs x 64 per clock at the measured SM clock",
            "note": "oil set; flops = Gram-Schmidt, normalisation and row tests per candidate weighted by the share reaching each "
                    "shock, Box-Muller's log / sqrt / sin / cos not counted (so the FP64 share is a lower bound); 'neither' when "
                    "both shares are below 0.5"}
    value = oil["cand_per_s"]
    line = {"metric": f"sign-restriction candidates/sec (one Figure-7-shaped model N=139 r=8 p=4 H={H}, 16 oil rows, n_rot=2^24)",
            "value": value, "unit": "candidates/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": oil["call_ms"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": value / cpu["value"], "dtype": "f64",
            "data": "hom_fac_1 (tests/golden), 1985Q1-2014Q4, plain Parametric() fit (20 EM iterations)",
            "config": {"workload": "dfm_sign_restrictions identified set (n_rot 2^24, n_keep 4096, device resident) under the oil and "
                                   "three-shock rows; 16384 models x 16 candidates; api.sign_restricted_responses at 4 chains x "
                                   "(40 + 80) sweeps x 4 rotations", "N": int(b["Lam"].shape[0]), "r": 8, "p": int(b["p"]), "H": H,
                       "set_oil": oil, "set_three": sets["three"], "posterior": post, "sign_restricted_responses": e2e},
            "e2e": {"value": value, "unit": "candidates/s", "ms_per_step": oil["call_ms"], "posterior_call_ms": post["call_ms"],
                    "sign_restricted_responses_ms": e2e["ms"]},
            "gpu_launches": oil["launches_per_call"], "clocks": clk, "roofline": roof, "cpu_baseline": cpu}
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
