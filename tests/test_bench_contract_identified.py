"""CPU only: the committed bench line of the named-factor bands (profiles/h100_bench_identified.json, written on an H100 by
tools/bench_identified.py in bench.py's line format) carries the restricted and unrestricted chain rates, the k_gibbs_draw kernel
times, and the k_series_resp measurements at n_shock = 1 and r with their bound."""
from test_bench_contract import BASE, _load


def test_identified_bench_line_has_contract_keys():
    d = _load("h100_bench_identified.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "chain-sweeps/s" and d["value"] > 0
    c = d["config"]
    assert (c["N"], c["r"], c["p"], c["n_chain"]) == (139, 8, 4, 264) and c["unrestricted_value"] > 0
    assert c["status_ok"] == {"restricted": True, "unrestricted": True}
    assert "k_gibbs_draw_constr" in c["draw_kernels"]["restricted"] and "k_gibbs_draw" in c["draw_kernels"]["unrestricted"]
    assert c["max_oil_dev_from_h"] < 1e-12
    r = d["roofline"]
    assert r["kernel"] == "k_series_resp" and r["bound"] in ("hbm", "fp64") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    rs = r["responses"]
    assert (rs["n_model"], rs["H"]) == (16384, 24)
    for k in ("n_shock_1", f"n_shock_{rs['r']}"):
        m = rs[k]
        for key in ("kernel_ms", "bytes_written", "bytes_read", "hbm_tbs", "frac_hbm_datasheet", "fp64_tflops", "bound", "status_ok"):
            assert key in m, key
        assert m["status_ok"] is True and m["kernel_ms"] > 0 and m["bytes_written"] > 0
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
