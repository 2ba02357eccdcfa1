#!/usr/bin/env python
"""SASS evidence: per-kernel counts of the mnemonics that show the Hopper-native paths (FP64 tensor MMA,
TMA tensor copies, mbarriers) and the E- / M-pass consumer loops of k_em_fused2<8>.  usage: sass_evidence.py lib.so > out.txt"""
import re, subprocess, sys
lib = sys.argv[1]
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
funcs = re.split(r"\n\s*Function : ", sass)[1:]
keys = ["DMMA", "UTMALDG", "SYNCS", "UBLKCP", "LDS", "STS", "LDG", "STG", "SHFL", "BAR", "ATOM", "MUFU", "DFMA", "DMUL", "DADD", "LDL", "STL", "HMMA", "UTC"]
print("# SASS mnemonic counts per kernel (cuobjdump -sass of the in-tree libdfm_b200.so, sm_90a)")
print("# FP64 tensor MMA = DMMA (mma.sync.m8n8k4.f64; wgmma has no f64 kind); TMA 2-D tensor copies = UTMALDG; mbarrier ops = SYNCS")
print(f"{'kernel':70s} " + " ".join(f"{k:>7s}" for k in keys) + "   instr")
em8 = None
for f in funcs:
    name = f.split("\n", 1)[0].strip()
    body = [l for l in f.split("\n") if re.search(r"/\*[0-9a-f]{4,}\*/\s+\S", l)]
    ins = [re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", l).split("/*")[0].strip() for l in body]
    dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
    short = re.sub(r"\(.*", "", dem).replace("void ", "").replace("dfm::", "")
    if not re.search(r"<(\(int\))?[1-7]>", short):        # keep the r = 8 instantiation of the templated kernels
        print(f"{short[:70]:70s} " + " ".join(f"{sum(1 for i in ins if re.match(r'(@!?U?P\d+\s+)?' + k, i)):7d}" for k in keys) + f"  {len(ins):6d}")
    if re.search(r"k_em_fused2<(\(int\))?8>", short):
        em8 = ins
print()
if em8:
    dm = [i for i, x in enumerate(em8) if "DMMA" in x]
    # the two consumer loops are the two densest DMMA clusters
    clusters = []
    for i in dm:
        if clusters and i - clusters[-1][-1] < 40: clusters[-1].append(i)
        else: clusters.append([i])
    clusters = sorted(clusters, key=len, reverse=True)[:2]
    for c, nm in zip(sorted(clusters), ("E pass (b_t = Lam' R^-1 x_t): consumer stage loop", "M pass (S_xf = X' E[f]): consumer stage loop")):
        lo, hi = max(0, c[0] - 45), min(len(em8), c[-1] + 12)
        print(f"## k_em_fused2<8>, {nm}  [SASS instructions {lo}..{hi}]")
        for x in em8[lo:hi]:
            print("    " + x)
        print()
