"""CPU only: the committed ss-bootstrap bench line (profiles/h100_bench_ss-bootstrap.json, written on an H100 by
tools/bench_ss_bootstrap.py in bench.py's line format) carries the keys a consumer of the bench line reads, both workloads, and
the bytes model of k_ss_sim_project it reports."""
from test_bench_contract import BASE, _load


def test_ss_bootstrap_bench_line_has_contract_keys():
    d = _load("h100_bench_ss-bootstrap.json")
    for k in BASE:
        assert k in d, k
    assert "workload" in d["config"] and d["dtype"] == "f64" and d["higher_is_better"] is True and d["unit"] == "replicates/s"
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step", "c1_value"):
        assert k in d["e2e"], k
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic", "em_share_of_step", "simulator_share_of_step", "kernel_ms", "c1"):
        assert k in r, k
    assert r["kernel"] == "k_ss_sim_project" and r["bound"] == "hbm"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert any(n.startswith("k_em_fused2") for n in r["kernel_ms"]) and "k_em_filter_smooth" in r["c1"]["kernel_ms"]
    assert d["gpu_launches"] > 0 and set(("sm_mhz", "sm_max_mhz", "reasons", "power_limit_w", "gpu")) <= set(d["clocks"])
    c = d["config"]
    assert c["n_rep"] == 1000 and c["all_status_ok"] is True and c["e2e_equals_device"] is True
    assert c["c1"]["n_rep"] == 1000 and c["c1"]["p"] == 4 and c["c1"]["all_status_ok"] is True and c["c1"]["e2e_equals_device"] is True
    assert d["cpu_baseline"]["cores"] == 1 and c["c1"]["cpu_baseline"]["cores"] == 1
