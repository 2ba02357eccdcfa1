"""CPU only: the committed bench line of the sign-restriction identification (profiles/h100_bench_sign.json, written on an H100 by
tools/bench_sign.py in bench.py's line format) carries the candidate rates, k_sign_cand's time, the operation counts and the bound
of both restriction sets, the posterior-path call, api.sign_restricted_responses end to end, the CPU arm, and the card it was
measured on."""
from test_bench_contract import BASE, _load


def test_sign_bench_line_has_contract_keys():
    d = _load("h100_bench_sign.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "candidates/s" and d["value"] > 0
    c = d["config"]
    assert (c["N"], c["r"], c["p"], c["H"]) == (139, 8, 4, 24)
    for k, rows in (("set_oil", 16), ("set_three", 40)):
        m = c[k]
        assert m["rows"] == rows and m["n_rot"] == 1 << 24 and m["n_keep"] == 4096, k
        for key in ("call_ms", "cand_per_s", "k_sign_cand_ms", "k_sign_pick_ms", "k_sign_rot_ms", "flops_per_cand", "philox_mul_per_cand",
                    "fp64_tflops", "frac_fp64_datasheet", "int_mul_tera_per_s", "frac_int_mul", "nearer_bound", "bound", "n_accept",
                    "status_ok"):
            assert key in m, (k, key)
        assert m["status_ok"] is True and m["k_sign_cand_ms"] > 0 and m["bound"] in ("fp64", "int_mul", "neither")
    post = c["posterior"]
    assert (post["n_model"], post["n_rot"]) == (16384, 16) and post["status_ok"] is True and post["call_ms"] > 0
    e = c["sign_restricted_responses"]
    assert e["status_ok"] is True and e["ms"] > 0 and (e["n_chain"], e["n_burn"], e["n_keep"], e["rot_per_draw"]) == (4, 40, 80, 4)
    cb = d["cpu_baseline"]
    assert cb["value"] > 0 and cb["cores"] == 1 and cb["unit"] == "candidates/s"
    r = d["roofline"]
    assert r["kernel"] == "k_sign_cand" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
