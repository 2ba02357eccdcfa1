"""CPU only: the committed Gibbs bench line (profiles/h100_bench_gibbs.json, written on an H100 by tools/bench_gibbs.py in
bench.py's line format) carries the keys a consumer of the bench line reads, both workloads, each stage's share of a sweep and the
bytes / flops model of k_gibbs_stats."""
from test_bench_contract import BASE, _load

STAGES = ("estep", "gains", "paths", "stats", "draw", "other")


def test_gibbs_bench_line_has_contract_keys():
    d = _load("h100_bench_gibbs.json")
    for k in BASE:
        assert k in d, k
    assert "workload" in d["config"] and d["dtype"] == "f64" and d["higher_is_better"] is True and d["unit"] == "chain-sweeps/s"
    assert d["value"] > 0 and d["e2e"]["value"] > 0 and d["e2e"]["c1_value"] > 0
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic", "stats_model", "stage_share_of_sweep", "kernel_ms", "c1"):
        assert k in r, k
    assert r["kernel"] == "k_gibbs_stats" and r["bound"] in ("dmma", "hbm")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    for sm in (r["stats_model"], r["c1"]["stats_model"]):
        for k in ("flops_per_sweep", "l2_bytes_per_sweep", "hbm_bytes_per_sweep", "ms_per_sweep", "frac_dmma_peak", "frac_hbm_peak", "bound"):
            assert k in sm, k
        assert sm["flops_per_sweep"] > 0 and sm["hbm_bytes_per_sweep"] > 0
    for sh in (r["stage_share_of_sweep"], r["c1"]["stage_share_of_sweep"]):
        assert set(STAGES) == set(sh) and abs(sum(sh.values()) - 1.0) < 1e-9
    for n in ("k_em_filter_smooth", "k_sim_gains", "k_gibbs_paths", "k_gibbs_stats", "k_gibbs_draw"):
        assert n in r["kernel_ms"] and n in r["c1"]["kernel_ms"], n
    assert d["gpu_launches"] > 0 and set(("sm_mhz", "sm_max_mhz", "reasons", "power_limit_w", "gpu")) <= set(d["clocks"])
    c = d["config"]
    assert (c["N"], c["r"], c["T"], c["p"], c["n_chain"]) == (200, 8, 500, 1, 264)
    assert c["all_status_ok"] is True and c["e2e_equals_device"] is True
    assert c["c1"]["p"] == 4 and c["c1"]["r"] == 8 and c["c1"]["all_status_ok"] is True and c["c1"]["e2e_equals_device"] is True
    assert c["rhat_c2"]["n_chain"] == 4 and c["rhat_c2"]["n_burn"] == 500
    assert d["cpu_baseline"]["cores"] == 1 and c["c1"]["cpu_baseline"]["cores"] == 1
