"""CPU only: the committed bench line of narrative sign restrictions (profiles/h100_bench_narrative.json, written on an H100 by
tools/bench_narrative.py in bench.py's line format) carries the candidate rates and kernel times of both narrative sets, the
simulation kernel's rate and FP64 share, the posterior-path call, api.narrative_restricted_responses end to end, the CPU arm, and
the card it was measured on."""
from test_bench_contract import BASE, _load


def test_narrative_bench_line_has_contract_keys():
    d = _load("h100_bench_narrative.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "candidates/s" and d["value"] > 0
    c = d["config"]
    assert (c["N"], c["r"], c["p"], c["H"], c["Tp"]) == (139, 8, 4, 24, 120)
    for k, kinds in (("set_most", [0, 1]), ("set_over", [0, 2])):
        m = c[k]
        assert m["rows"] == 16 and m["narrative_kinds"] == kinds and m["n_rot"] == 1 << 24 and m["n_keep"] == 4096, k
        assert m["n_sim"] == 1 << 14 and m["status_ok"] is True
        for key in ("call_ms", "cand_per_s", "k_narr_cand_ms", "k_sign_pick_ms", "k_narr_rot_ms", "k_narr_omega_ms", "kernels_ms",
                    "n_accept", "ess", "n_zero_omega"):
            assert key in m, (k, key)
        assert m["k_narr_cand_ms"] > 0
    om = c["omega"]
    assert om["kernel"] == "k_narr_omega" and om["n_keep"] == 4096 and om["n_sim"] == 1 << 14
    assert om["sims_per_s"] > 0 and om["flops_per_sim"] > 0 and abs(om["frac_fp64_datasheet"] - om["fp64_tflops"] / 34.0) < 1e-9
    post = c["posterior"]
    assert (post["n_model"], post["n_rot"]) == (16384, 16) and post["status_ok"] is True and post["call_ms"] > 0
    e = c["narrative_restricted_responses"]
    assert e["status_ok"] is True and e["ms"] > 0 and (e["n_chain"], e["n_burn"], e["n_keep"], e["rot_per_draw"]) == (4, 40, 80, 4)
    cb = d["cpu_baseline"]
    assert cb["value"] > 0 and cb["cores"] == 1 and cb["unit"] == "candidates/s"
    r = d["roofline"]
    assert r["kernel"] == "k_narr_omega" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
