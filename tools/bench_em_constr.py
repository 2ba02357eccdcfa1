#!/usr/bin/env python
"""bench_em_constr.py -- cost of restrictions on the loadings in the state-space EM (dfm_em_kalman_constrained) on two
workloads, restricted and unrestricted calls alternating in one process:
  c1   296 C1-shaped panels (bootstrap draws of the hom_fac_1 model as tools/bench_c1_em.py builds them: T = 222, 139 estimation
       series, r = 8, VAR(4) state, 5.7 % missing), 20 EM iterations, the Figure 7 restriction (WPU0561, MCOILWTICO,
       MCOILBRENTEU, RAC_IMP load e_1 only; standardized h = e_1).  Both calls run the general path (k_em_mstep_series); the
       difference is the correction of the restricted M-step.
  c5   bench.py's C5 shard (1250 C2-shaped panels, N = 200, r = 8, T = 500, p = 1, balanced), 50 EM iterations, series 0-3
       restricted to e_1.  Restricted: the general path (k_emb_mstep_constr); unrestricted: k_em_fused2.  This documents the
       cost of the route, not a target.
Device-resident inputs and outputs.  Prints one JSON line in bench.py's line format (value = restricted panel-EM-iterations/s
of c1) with both workloads, per-kernel times of one profiled call each, and clocks sampled during the run.

python tools/bench_em_constr.py --steps K --warmup W [--json profiles/h100_bench_em-constr.json]
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


def _c1_batch(lib, B, p):
    import dynamic_factor_models_b200 as D
    from dynamic_factor_models_b200 import replicate
    z = np.load(os.path.join(ROOT, "tests", "golden", "hom_fac_1_panels.npz"))
    m = D.DFMModel(z["all_bpdata"], z["all_inclcode"], 20, 40, 3, 224, 0, 8, 1e-8, 4, 4)
    D.estimate(m, lib=lib)
    X = replicate.bootstrap_panels(m, range(B), lib=lib)[:, :, m.inclcode == 1]
    Xs, _, _ = lib.standardize(X)
    als = lib.estimate_factor(X, 8, compute_r2=False)
    Lam, R, A, Q = lib.em_init_from_factors(Xs, als["F"], p)
    used = [str(n) for n, c in zip(z["all_names"], z["all_inclcode"]) if c == 1]
    idx = [used.index(n) for n in OIL]
    return Xs, (Lam, R, A, Q), idx


def _c5_batch(lib, B):
    X = lib.simulate_panels(0, B, bench.NS, bench.R_, bench.T_, bench.SEED)           # replication ids 0 .. B-1, as bench.py
    F0 = lib.estimate_factor(X, bench.R_, max_iter=1, compute_r2=False)["F"]
    return X, lib.em_init_from_factors(X, F0, 1)


def _ab(lib, torch, dev, X, th, p, iters, cons, K_, W_):
    """Alternating restricted / unrestricted device-resident calls: ms per call of each, per-kernel ms of one profiled call of
    each, and the statuses."""
    from dynamic_factor_models_b200._lib import MEM_DEVICE, to_cm
    B, T, N = X.shape; r = th[0].shape[-1]; k = r * p
    cm = lambda a: torch.from_numpy(np.ascontiguousarray(to_cm(a))).to(dev)
    dX = cm(X); dth = dict(Lam=cm(th[0]), R=torch.from_numpy(np.ascontiguousarray(th[1])).to(dev), A=cm(th[2]), Q=cm(th[3]))
    outs = {n: torch.empty(B * s, dtype=torch.float64, device=dev) for n, s in
            dict(Lam=N * r, R=N, A=r * k, Q=r * r, F=T * r, loglik=iters).items()}
    dit = torch.empty(B, dtype=torch.int32, device=dev); dst = torch.empty(B, dtype=torch.int32, device=dev)
    init = {n: t.data_ptr() for n, t in dth.items()}
    out = {**{n: t.data_ptr() for n, t in outs.items()}, "iters": dit.data_ptr(), "status": dst.data_ptr()}

    def call(c):
        lib.em_kalman_raw(dX.data_ptr(), T, N, r, p, B, iters, 0.0, init, out, MEM_DEVICE, 0, constr=c)
        lib.sync()

    for _ in range(W_):
        call(cons); call(None)
    ms = {"restricted": 0.0, "unrestricted": 0.0}
    for _ in range(K_):
        ms["restricted"] += bench._timed(torch, None, 1, dev, lambda: call(cons), 1)
        ms["unrestricted"] += bench._timed(torch, None, 1, dev, lambda: call(None), 1)
    res = {}
    for name, c in (("restricted", cons), ("unrestricted", None)):
        call(c)
        st = dst.cpu().numpy()
        lam = outs["Lam"].cpu().numpy().reshape(B, r, N).transpose(0, 2, 1)
        lib.profile(True); call(c); prof = lib.profile_report(); lib.profile(False)
        res[name] = dict(ms_per_call=ms[name] / K_, panel_em_iters_per_s=B * iters / (ms[name] / K_ * 1e-3),
                         all_status_ok=bool((st == 0).all()), n_failed=int((st != 0).sum()),
                         kernel_ms={n_: round(v[0], 3) for n_, v in sorted(prof.items(), key=lambda kv: -kv[1][0])})
        if c is not None:
            ix, H, h = c
            ok = st == 0
            res[name]["restriction_max_abs_violation"] = float(np.max(np.abs(np.einsum("qa,bqa->bq", H, lam[ok][:, ix, :]) - h)))
    kr, ku = res["restricted"]["kernel_ms"], res["unrestricted"]["kernel_ms"]
    res["shape"] = dict(B=B, T=T, N=N, r=r, p=p, em_iters=iters, n_constr=len(cons[0]), restricted_series=sorted(set(int(i) for i in cons[0])))
    res["slowdown"] = res["restricted"]["ms_per_call"] / res["unrestricted"]["ms_per_call"]
    res["mstep_kernel_ms_delta"] = {n_: round(kr.get(n_, 0.0) - ku.get(n_, 0.0), 3) for n_ in set(kr) | set(ku)
                                    if "mstep" in n_}
    return res


def run(args):
    torch, dist, world, rank, local, dev = bench._dist_setup()
    assert world == 1, "single-GPU tool"
    from dynamic_factor_models_b200 import Library
    lib = Library(path=os.environ.get("DFM_BENCH_LIB"), device=local)
    clocks = bench.ClockSampler(dev.index or 0); clocks.start()
    r = 8
    X1, th1, idx = _c1_batch(lib, 296, 4)
    e1 = np.r_[1.0, np.zeros(r - 1)]
    c1cons = (np.repeat(idx, r), np.tile(np.eye(r), (len(idx), 1)), np.tile(e1, len(idx)))
    c1 = _ab(lib, torch, dev, X1, th1, 4, 20, c1cons, args.steps, args.warmup)
    X5, th5 = _c5_batch(lib, args.c5_panels)
    c5cons = (np.repeat(np.arange(4), r), np.tile(np.eye(r), (4, 1)), np.tile(e1, 4))
    c5 = _ab(lib, torch, dev, X5, th5, 1, 50, c5cons, args.steps, args.warmup)
    clk = clocks.stop()
    v = c1["restricted"]["panel_em_iters_per_s"]
    line = {"metric": "restricted state-space EM panel-iterations/sec (296 C1-shaped panels, Figure 7 restriction, 20 EM iterations, "
                      "general path)", "value": v, "unit": "panel-EM-iterations/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": c1["restricted"]["ms_per_call"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "C1: bootstrap draws of hom_fac_1 (tests/golden); C5: synthetic (device-generated frozen DGP, SURVEY.md 8d)",
            "config": {"workload": "dfm_em_kalman_constrained vs dfm_em_kalman on the same device-resident batch, alternating in one "
                                   "process", "c1": c1, "c5": c5},
            "e2e": {"value": v, "unit": "panel-EM-iterations/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                    "note": "device-resident inputs and outputs; the restriction table (a few hundred bytes) is uploaded per call"},
            "gpu_launches": None, "clocks": clk,
            "roofline": {"bound": None, "note": "the correction is O(m_i r^2) flops per restricted series and iteration on one thread; "
                                                "the report gives its measured cost (mstep_kernel_ms_delta, slowdown), not a bound"},
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
    ap.add_argument("--c5-panels", type=int, default=1250)
    ap.add_argument("--json", default=None, help="also write the line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
