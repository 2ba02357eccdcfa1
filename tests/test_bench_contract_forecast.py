"""CPU only: the committed c5-forecast bench line (profiles/h100_bench_c5-forecast.json, written on an H100 by
tools/bench_forecast.py in bench.py's line format) carries the keys a consumer of the bench line reads, and the roofline of k_ss_project it reports."""
from test_bench_contract import BASE, _load


def test_forecast_bench_line_has_contract_keys():
    d = _load("h100_bench_c5-forecast.json")
    for k in BASE:
        assert k in d, k
    assert "workload" in d["config"] and d["dtype"] == "f64" and d["higher_is_better"] is True and d["unit"] == "panels/s"
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"], k
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic", "kernel_share_of_step"):
        assert k in r, k
    assert r["kernel"] == "k_ss_project" and r["bound"] == "hbm"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["gpu_launches"] > 0 and set(("sm_mhz", "sm_max_mhz", "reasons", "power_limit_w")) <= set(d["clocks"])
    assert d["config"]["all_status_ok"] is True
