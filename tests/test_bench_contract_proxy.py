"""CPU only: the committed bench line of the proxy identification (profiles/h100_bench_proxy.json, written on an H100 by
tools/bench_proxy.py in bench.py's line format) carries the boot workload's call and kernel times and bytes, the posterior-shaped
call, api.proxy_restricted_responses end to end, the CPU arm, and the card it was measured on."""
from test_bench_contract import BASE, _load


def test_proxy_bench_line_has_contract_keys():
    d = _load("h100_bench_proxy.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "records/s" and d["value"] > 0
    c = d["config"]
    assert (c["N"], c["r"], c["p"], c["H"]) == (139, 8, 4, 24)
    bt = c["boot"]
    assert (bt["n_inst"], bt["n_boot"]) == (3, 16383) and bt["status_ok"] is True
    for key in ("call_ms", "records_per_s", "k_iv_prep_ms", "k_iv_boot_ms", "k_iv_rot_ms", "k_series_resp_ms", "kernels_ms",
                "k_series_resp_bytes", "k_series_resp_tbps", "frac_hbm_k_series_resp", "launches_per_call"):
        assert key in bt, key
    post = c["posterior"]
    assert (post["n_model"], post["n_inst"], post["n_boot"]) == (16384, 1, 0) and post["status_ok"] is True and post["call_ms"] > 0
    e = c["proxy_restricted_responses"]
    assert e["status_ok"] is True and e["ms"] > 0 and (e["n_chain"], e["n_burn"], e["n_keep"], e["boot_per_draw"]) == (4, 40, 80, 1)
    cb = d["cpu_baseline"]
    assert cb["value"] > 0 and cb["cores"] == 1 and cb["unit"] == "records/s"
    r = d["roofline"]
    assert r["kernel"] == "k_series_resp" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
