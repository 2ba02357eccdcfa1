"""CPU only: the committed bench line of the historical decompositions (profiles/h100_bench_history.json, written on an H100 by
tools/bench_history.py in bench.py's line format) carries the k_hd_paths / k_hd_series times, bytes, rates and bound at
n_shock = 1 and r, the whole call, api.identified_history end to end, and the card it was measured on."""
from test_bench_contract import BASE, _load


def test_history_bench_line_has_contract_keys():
    d = _load("h100_bench_history.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "models/s" and d["value"] > 0
    c = d["config"]
    assert (c["n_model"], c["N"], c["r"], c["p"], c["Tp"], c["t0"]) == (4096, 139, 8, 4, 120, 3)
    for k in ("n_shock_1", f"n_shock_{c['r']}"):
        m = c[k]
        for key in ("call_ms", "k_hd_paths_ms", "k_hd_series_ms", "bytes_written", "bytes_read", "hbm_tbs", "frac_hbm_datasheet",
                    "fp64_tflops", "frac_fp64_datasheet", "bound", "status_ok"):
            assert key in m, key
        assert m["status_ok"] is True and m["k_hd_series_ms"] > 0 and m["bytes_written"] > 0 and m["bound"] in ("hbm", "fp64")
    ih = c["identified_history"]
    assert ih["status_ok"] is True and ih["ms"] > 0 and (ih["n_chain"], ih["n_burn"], ih["n_keep"]) == (4, 40, 80)
    r = d["roofline"]
    assert r["kernel"] == "k_hd_series" and r["bound"] in ("hbm", "fp64") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
