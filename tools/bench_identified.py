#!/usr/bin/env python
"""bench_identified.py -- cost of the named-factor bands (api.identified_responses) on an H100:
  chains     dfm_gibbs_constrained vs dfm_gibbs on Stock & Watson's Figure 7 model (hom_fac_1, 1985Q1-2014Q4, r=8, p=4, the four
             oil series pinned to e_1 in the ALS steps and a 50-iteration restricted EM), 264 chains x `--sweeps` sweeps per step,
             device resident, the two calls alternating in one process; per-kernel times of k_gibbs_draw / k_gibbs_draw_constr;
  responses  dfm_series_responses on 16384 Figure-7-shaped models (the fit's Lam, R, A, Q scaled per model), H = 24, device
             resident, n_shock = 1 and n_shock = r: kernel time of k_series_resp, bytes it writes and reads, and its share of the
             3.35 TB/s HBM3 data-sheet rate and of the 34 TFLOP/s FP64 data-sheet rate, the larger naming the bound.
Prints one JSON line in bench.py's line format (value = restricted chain-sweeps/s).

python tools/bench_identified.py --steps K --warmup W [--json profiles/h100_bench_identified.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

OIL = ["WPU0561", "MCOILWTICO", "MCOILBRENTEU", "RAC_IMP"]
PEAK_FP64_TFLOPS = 34.0          # H100 SXM5 FP64 (non-tensor) data-sheet rate
N_MODEL, H_RESP = 16384, 24


def _figure7(lib):
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200.api import _state_space_block
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
    D.estimate(m, D.Parametric(max_iter=50, tol=0.0), lam_constr_f=gf, lam_constr_fl=gfl, lam_constr_em=gf, lib=lib)
    b = _state_space_block(m, 0, lib, "bench")
    e = m.em
    return m, b["Xs"], dict(Lam=b["Lam"], R=e["R"], A=e["A"], Q=e["Q"], P0=e["P0"]), b["p"], e["lam_constr"], b["xstd"]


def _chains(lib, torch, dev, X, th, p, constr, n_chain, n_sweep, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm, gibbs_default_prior
    T, N = X.shape; r = th["Lam"].shape[1]; k = r * p
    n_burn = n_sweep // 2; n_keep = n_sweep - n_burn
    cm = lambda a: torch.from_numpy(np.ascontiguousarray(to_cm(a))).to(dev)
    rep = lambda a: np.stack([a] * n_chain)
    init = {n: rep(th[n]) for n in ("Lam", "R", "A", "Q", "P0")}
    dX = cm(X)
    dini = {n: (cm(init[n]) if n != "R" else torch.from_numpy(np.ascontiguousarray(init[n]).ravel()).to(dev)) for n in init}
    f64 = lambda n: torch.empty(max(n, 1), dtype=torch.float64, device=dev)
    sizes = dict(Lam=N * r, R=N, A=r * k, Q=r * r)
    dout = {n: f64(n_chain * n_keep * s) for n, s in sizes.items()}
    dll = f64(n_chain * n_sweep); dst = torch.empty(n_chain, dtype=torch.int32, device=dev)
    outs = {**{n: t.data_ptr() for n, t in dout.items()}, "loglik": dll.data_ptr(), "status": dst.data_ptr()}
    kw = dict(n_chain=n_chain, n_burn=n_burn, n_keep=n_keep, seed=bench.SEED, prior=gibbs_default_prior(r))

    def step(c):
        lib.gibbs_raw(dX.data_ptr(), T, N, r, p, {n: t.data_ptr() for n, t in dini.items()}, None, outs, MEM_DEVICE, constr=c, **kw)
        lib.sync()

    for _ in range(W_):
        step(constr); step(None)
    ms = {"restricted": 0.0, "unrestricted": 0.0}
    status_ok = {}
    for _ in range(K_):                                  # alternating, one step each
        for name, c in (("restricted", constr), ("unrestricted", None)):
            ms[name] += bench._timed(torch, None, 1, dev, lambda: step(c), 1)
            status_ok[name] = bool((dst.cpu().numpy() == 0).all())
    kern = {}
    for name, c in (("restricted", constr), ("unrestricted", None)):
        lib.profile(True); step(c); prof = lib.profile_report(); lib.profile(False)
        kern[name] = {n: dict(ms=round(v[0], 4), launches=v[1]) for n, v in prof.items() if n.startswith("k_gibbs_draw")}
    oil_on_e1 = None
    if constr is not None:
        step(constr)
        lam = dout["Lam"].cpu().numpy().reshape(n_chain * n_keep, r, N).transpose(0, 2, 1)
        idx = sorted(set(int(i) for i in constr[0]))
        idx = [i for i in idx if not np.isnan(th["Lam"][i, 0])]
        hv = {int(i): v for i, v in zip(constr[0], constr[2]) if v != 0}
        oil_on_e1 = float(max(np.max(np.abs(lam[:, i] - np.r_[hv[i], np.zeros(r - 1)])) for i in idx))
    rate = {n: n_chain * n_sweep * K_ / (v * 1e-3) for n, v in ms.items()}
    return dict(rate=rate, ms_per_step={n: v / K_ for n, v in ms.items()}, status_ok=status_ok, kernels=kern,
                max_oil_dev_from_h=oil_on_e1, shape=dict(T=T, N=N, r=r, p=p, n_chain=n_chain, sweeps_per_step=n_sweep))


def _responses(lib, torch, dev, th, p, xstd, K_, W_):
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    N, r = th["Lam"].shape; k = r * p; B, H = N_MODEL, H_RESP
    s = 1.0 + 0.05 * np.linspace(-1, 1, B)
    Lam = np.stack([th["Lam"]] * B) * s[:, None, None]
    Lam[:, np.isnan(th["Lam"][:, 0])] = np.nan
    dm = dict(Lam=torch.from_numpy(np.ascontiguousarray(to_cm(Lam))).to(dev),
              R=torch.from_numpy(np.ascontiguousarray(np.stack([th["R"]] * B)).ravel()).to(dev),
              A=torch.from_numpy(np.ascontiguousarray(to_cm(np.stack([th["A"]] * B) * (s[:, None, None] ** 0.1)))).to(dev),
              Q=torch.from_numpy(np.ascontiguousarray(to_cm(np.stack([th["Q"]] * B) * s[:, None, None]))).to(dev))
    dsc = torch.from_numpy(np.ascontiguousarray(xstd)).to(dev)
    n_in = int((~np.isnan(th["Lam"][:, 0])).sum())
    out = {}
    for ns in (1, r):
        o = {n: torch.empty(B * N * H * ns, dtype=torch.float64, device=dev) for n in ("resp", "fevd")}
        st = torch.empty(B, dtype=torch.int32, device=dev)

        def call():
            lib.series_responses_raw({n: t.data_ptr() for n, t in dm.items()}, N, r, p, B, H, ns, dsc.data_ptr(), MEM_DEVICE,
                                     resp=o["resp"].data_ptr(), fevd=o["fevd"].data_ptr(), status=st.data_ptr())
            lib.sync()

        for _ in range(W_):
            call()
        ms_call = bench._timed(torch, None, 1, dev, lambda: [call() for _ in range(K_)], 1) / K_
        lib.profile(True)
        for _ in range(K_):
            call()
        prof = lib.profile_report(); lib.profile(False)
        kt = prof["k_series_resp"][0] / prof["k_series_resp"][1]
        wbytes = 2.0 * 8 * B * N * H * ns
        rbytes = 8.0 * B * (N * r + N + r * r * H) + 8.0 * N
        flops = 2.0 * B * n_in * H * (r * r + r)
        hbm = (wbytes + rbytes) / (kt * 1e-3) / 1e12
        tfl = flops / (kt * 1e-3) / 1e12
        t_mem, t_fl = (wbytes + rbytes) / 3.35e12, flops / (PEAK_FP64_TFLOPS * 1e12)
        out[f"n_shock_{ns}"] = dict(kernel_ms=kt, call_ms=ms_call, kernels_ms={n: round(v[0] / v[1], 4) for n, v in prof.items()},
                                   bytes_written=wbytes, bytes_read=rbytes, flops=flops, hbm_tbs=hbm, frac_hbm_datasheet=hbm / 3.35,
                                   fp64_tflops=tfl, frac_fp64_datasheet=tfl / PEAK_FP64_TFLOPS,
                                   bound="hbm" if t_mem >= t_fl else "fp64", frac_of_bound=max(t_mem, t_fl) / (kt * 1e-3),
                                   status_ok=bool((st.cpu().numpy() == 0).all()))
    return dict(n_model=B, N=N, r=r, p=p, H=H, **out)


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    m, X, th, p, constr, xstd = _figure7(lib)
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    ch = _chains(lib, torch, dev, X, th, p, constr, args.chains, args.sweeps, args.steps, args.warmup)
    rs = _responses(lib, torch, dev, th, p, xstd, args.steps, args.warmup)
    clk = clocks.stop()
    r1, rr = rs["n_shock_1"], rs[f"n_shock_{th['Lam'].shape[1]}"]
    roof = {"bound": rr["bound"], "kernel": "k_series_resp", "achieved": rr["hbm_tbs"], "peak": 3.35, "unit": "TB/s",
            "frac": rr["hbm_tbs"] / 3.35, "traffic": {"bytes_written": rr["bytes_written"], "bytes_read": rr["bytes_read"]},
            "peak_source": "H100 SXM5 data sheet (3.35 TB/s HBM3, 34 TFLOP/s FP64)", "responses": rs,
            "note": "k_series_resp at n_shock = r; bytes = resp + fevd written once, Lam, R, Psi read once; flops = 2 r (r + 1) per "
                    "(series in the model, horizon); the bound is the larger of bytes / 3.35 TB/s and flops / 34 TFLOP/s"}
    line = {"metric": f"restricted Gibbs chain-sweeps/sec (Figure 7 model r=8 p=4, {args.chains} chains)",
            "value": ch["rate"]["restricted"], "unit": "chain-sweeps/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ch["ms_per_step"]["restricted"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "hom_fac_1 (tests/golden), 1985Q1-2014Q4, oil series pinned to e_1",
            "config": {"workload": f"dfm_gibbs_constrained vs dfm_gibbs alternating, {args.chains} chains x {args.sweeps} sweeps per step "
                                   f"(half burn-in, half kept: Lam, R, A, Q); dfm_series_responses on {N_MODEL} models, H = {H_RESP}",
                       **ch["shape"], "unrestricted_value": ch["rate"]["unrestricted"],
                       "unrestricted_ms_per_step": ch["ms_per_step"]["unrestricted"], "status_ok": ch["status_ok"],
                       "draw_kernels": ch["kernels"], "max_oil_dev_from_h": ch["max_oil_dev_from_h"],
                       "responses_n_shock_1": r1},
            "e2e": {"value": ch["rate"]["restricted"], "unit": "chain-sweeps/s", "ms_per_step": ch["ms_per_step"]["restricted"]},
            "gpu_launches": int(sum(v["launches"] for v in ch["kernels"]["restricted"].values())), "clocks": clk, "roofline": roof,
            "cpu_baseline": None}
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
    ap.add_argument("--chains", type=int, default=264)
    ap.add_argument("--sweeps", type=int, default=20)
    ap.add_argument("--json", default=None)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
