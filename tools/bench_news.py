#!/usr/bin/env python
"""bench_news.py -- throughput of dfm_news (the news decomposition of nowcast revisions at fixed parameters) on the C5
workload of bench.py: 1250 C2-shaped vintage pairs per GPU (N=200, r=8, T=500) at the parameters after bench.py's 50 EM
iterations.  The new vintage is the simulated panel; the old one hides about 30 % of the series in each of the last two
rows; 4 targets (series 0..3) at periods T-1 .. T+2 (1-based), H = 2.  Prints one JSON line in the format of bench.py's lines
(value = pairs/s device resident, e2e = pinned host buffers through the C ABI, per-kernel times, the bytes model of
k_news_project, the share of the step taken by the shared E-step, clocks, launches, CPU arm = the NumPy spec on one core).

python tools/bench_news.py --steps K --warmup W [--no-cpu]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ESTEP = ("k_em_filter_smooth", "k_em_contract", "k_em_contract_bal", "k_em_scan", "k_em_prep", "k_em_state_init", "k_em_collect",
         "k_lyapunov", "k_ss_pad")


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    from dynamic_factor_models_b200 import Library
    from dynamic_factor_models_b200._lib import MEM_DEVICE, MEM_HOST
    import ctypes as C
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    B, iters, K_, W_, H, nr = args.pairs, args.em_iters, args.steps, args.warmup, 2, 2
    N, r, T, p = bench.NS, bench.R_, bench.T_, bench.P_
    k = r * p
    targets = [(q, T - 2 + q) for q in range(4)]
    nq = len(targets)
    f64 = lambda n: torch.empty(n, dtype=torch.float64, device=dev)
    dXn, dF0 = f64(B * T * N), f64(B * T * r)
    lib.simulate_panels_raw(rank * B, B, N, r, T, bench.SEED, dXn.data_ptr())
    lib.estimate_factor_raw(dXn.data_ptr(), T, N, r, B, MEM_DEVICE, F=dF0.data_ptr(), max_iter=1)
    d0 = {n: f64(sz) for n, sz in dict(Lam=B * N * r, R=B * N, A=B * r * k, Q=B * r * r).items()}
    lib.check(lib.lib.dfm_em_init_from_factors(lib.h, C.c_void_p(dXn.data_ptr()), C.c_void_p(dF0.data_ptr()), T, N, r, p, B, MEM_DEVICE,
                                               *[C.c_void_p(d0[n].data_ptr()) for n in ("Lam", "R", "A", "Q")]), "em_init")
    par = {n: f64(sz) for n, sz in dict(Lam=B * N * r, R=B * N, A=B * r * k, Q=B * r * r, loglik=B * iters).items()}
    dit = torch.empty(B, dtype=torch.int32, device=dev); dst = torch.empty(B, dtype=torch.int32, device=dev)
    lib.em_kalman_raw(dXn.data_ptr(), T, N, r, p, B, iters, 0.0, {n: d0[n].data_ptr() for n in d0},
                      dict(Lam=par["Lam"].data_ptr(), R=par["R"].data_ptr(), A=par["A"].data_ptr(), Q=par["Q"].data_ptr(),
                           loglik=par["loglik"].data_ptr(), iters=dit.data_ptr(), status=dst.data_ptr()), MEM_DEVICE, args.path)
    lib.sync()
    # the old vintage: ~30 % of the series hidden in each of the last two rows (column-major panels: row t of series i of
    # pair b at (b N + i) T + t)
    g = torch.Generator().manual_seed(20261016 + rank)
    hide = (torch.rand((B, N, nr), generator=g) < 0.3).to(dev)
    dXo = dXn.clone().view(B, N, T)
    dXo[:, :, T - nr:] = torch.where(hide, torch.full_like(dXo[:, :, T - nr:], float("nan")), dXo[:, :, T - nr:])
    dXo = dXo.reshape(-1).contiguous()
    params_d = {n: par[n].data_ptr() for n in ("Lam", "R", "A", "Q")}
    sizes = dict(old_est=B * nq, new_est=B * nq, news=B * nr * N, weight=B * nr * N * nq, contrib=B * nr * N * nq)
    dout = {n: f64(sz) for n, sz in sizes.items()}
    sst = torch.empty(B, dtype=torch.int32, device=dev)
    out_d = {**{n: t.data_ptr() for n, t in dout.items()}, "status": sst.data_ptr()}

    def step_device():
        lib.news_raw(dXo.data_ptr(), dXn.data_ptr(), T, N, r, p, H, B, nr, targets, params_d, out_d, MEM_DEVICE)
        lib.sync()

    for _ in range(W_):
        step_device()
    clocks = bench.ClockSampler(local); clocks.start()
    l0 = lib.launches
    ms = bench._timed(torch, dist, world, dev, step_device, K_)
    launches = lib.launches - l0
    clk = clocks.stop()
    value = world * B * K_ / (ms * 1e-3)
    status_ok = bool((sst == 0).all().item())
    # identity sum_j w_j I_j = new - old, and the share of news cells
    con = dout["contrib"].view(B, nq, N * nr).sum(2)
    ident = float(((dout["new_est"].view(B, nq) - dout["old_est"].view(B, nq)) - con).abs().max().item())
    news_cells = int((~torch.isnan(dout["news"])).sum().item())

    # ---- e2e: pinned host buffers
    hXo, hXn = dXo.cpu().pin_memory(), dXn.cpu().pin_memory()
    hpar = {n: par[n].cpu().pin_memory() for n in ("Lam", "R", "A", "Q")}
    hout = {n: torch.empty(sz, dtype=torch.float64).pin_memory() for n, sz in sizes.items()}
    hst = torch.empty(B, dtype=torch.int32).pin_memory()
    out_h = {**{n: t.data_ptr() for n, t in hout.items()}, "status": hst.data_ptr()}

    def step_e2e():
        lib.news_raw(hXo.data_ptr(), hXn.data_ptr(), T, N, r, p, H, B, nr, targets, {n: t.data_ptr() for n, t in hpar.items()}, out_h,
                     MEM_HOST)

    step_e2e()
    Ke = max(2, min(K_, 3))
    ms_e = bench._timed(torch, dist, world, dev, step_e2e, Ke)
    e2e_same = all(torch.equal(torch.isnan(hout[n].to(dev)), torch.isnan(dout[n])) and
                   torch.equal(torch.nan_to_num(hout[n].to(dev), nan=0.0), torch.nan_to_num(dout[n], nan=0.0)) for n in sizes)
    h2d = 8 * (hXo.numel() + B * N * nr + sum(t.numel() for t in hpar.values()))
    d2h = 8 * sum(t.numel() for t in hout.values()) + 4 * B

    # ---- per-kernel times of one profiled step (outside the timed region), bytes model of k_news_project
    lib.profile(True); step_device(); prof = lib.profile_report(); lib.profile(False)
    tot = sum(v_[0] for v_ in prof.values()) or 1.0
    dom = max(prof, key=lambda n: prof[n][0])
    peak, peak_src = bench._peak()
    p_ms, p_cnt = prof["k_news_project"]
    alg = float(B) * (8 * nr * N * (2 + 2 * nq) + nr * N + 8 * N * (r + 1) + 8 * nr * r + 8 * nq * nr * r)
    ach = alg / (p_ms * 1e-3) / 1e9
    estep_ms = sum(prof[n][0] for n in ESTEP if n in prof)
    roof = {"bound": "hbm", "kernel": "k_news_project", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "traffic": None,
            "peak_source": peak_src, "kernel_share_of_step": p_ms / tot, "dominant_kernel_of_step": dom, "avg_launch_ms": p_ms / p_cnt,
            "algorithmic_bytes_per_launch": alg / p_cnt, "estep_share_of_step": estep_ms / tot,
            "note": "per pair 8 nr N (2 + 2 nq) + nr N + 8 N (r + 1) + 8 nr r (1 + nq) bytes: X_new window read, news / weight / "
                    "contrib written, the mask byte, loadings and R, the factors and g vectors of the window rows",
            "kernel_ms": {n: round(v_[0], 3) for n, v_ in sorted(prof.items(), key=lambda kv: -kv[1][0])}}
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from news_oracle import news as news_spec
        nb = 2
        Xo = bench._cm(dXo[:nb * T * N], nb, T, N); Xn = bench._cm(dXn[:nb * T * N], nb, T, N)
        ph = dict(Lam=bench._cm(par["Lam"][:nb * N * r], nb, N, r), R=par["R"][:nb * N].cpu().numpy().reshape(nb, N),
                  A=bench._cm(par["A"][:nb * r * k], nb, r, k), Q=bench._cm(par["Q"][:nb * r * r], nb, r, r))
        t0 = time.perf_counter()
        for b in range(nb):
            news_spec(Xo[b], Xn[b], ph["Lam"][b], ph["R"][b], ph["A"][b], ph["Q"][b], None, p, H, targets, nr)
        dt = time.perf_counter() - t0
        cpu = {"value": nb / dt, "unit": "pairs/s", "cores": 1, "kind": "port",
               "sample": f"{nb} pairs, NumPy spec news (tests/news_oracle.py: Kalman filter + RTS smoother on the padded old panel, "
                         f"Sigma, Woodbury weights), 1 process, {dt:.2f} s"}
    if rank == 0:
        print(json.dumps({"metric": f"news decomposition pairs/sec (C5 shard, N={N} r={r} T={T}, H={H}, {nq} targets)", "value": value,
                          "unit": "pairs/s", "n_gpus": world, "steps": K_, "warmup": W_, "ms_per_step": ms / K_, "higher_is_better": True,
                          "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic (device-generated frozen DGP, SURVEY.md 8d)",
                          "config": {"workload": f"C5 shard: {B} C2-shaped vintage pairs/GPU at the parameters after {iters} EM iterations; "
                                                 f"~30% of the series released in each of the last {nr} rows; dfm_news with {nq} targets "
                                                 f"(series 0..3 at periods T-1 .. T+2), H={H}: old/new estimates, news, weights, contributions",
                                     "pairs_per_gpu": B, "H": H, "news_rows": nr, "n_target": nq, "em_iters_before": iters,
                                     "all_status_ok": status_ok, "news_cells": news_cells, "identity_max_abs": ident,
                                     "e2e_equals_device": bool(e2e_same)},
                          "e2e": {"value": world * B * Ke / (ms_e * 1e-3), "unit": "pairs/s", "h2d_bytes_per_step": h2d,
                                  "d2h_bytes_per_step": d2h, "ms_per_step": ms_e / Ke},
                          "gpu_launches": int(launches), "clocks": clk, "roofline": roof, "cpu_baseline": cpu}))
    if world > 1:
        dist.destroy_process_group()
    lib.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pairs", type=int, default=1250, help="vintage pairs per GPU (C5 shard = 10000/8)")
    ap.add_argument("--em-iters", type=int, default=50, help="EM iterations that produce the parameters (bench.py's c5 step)")
    ap.add_argument("--path", type=int, default=0, help="dfm_em_kalman path of the EM step that produces the parameters")
    ap.add_argument("--no-cpu", action="store_true")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
