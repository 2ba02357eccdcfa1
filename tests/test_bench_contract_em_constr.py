"""CPU only: the committed bench line of the restricted state-space EM (profiles/h100_bench_em-constr.json, written on an H100
by tools/bench_em_constr.py in bench.py's line format) carries the keys a consumer of the bench line reads and both workloads:
296 C1-shaped panels with the Figure 7 restriction, and the C5 shard with a named-factor restriction, each against the same
batch unrestricted in the same process."""
from test_bench_contract import BASE, _load


def test_em_constr_bench_line_has_contract_keys():
    d = _load("h100_bench_em-constr.json")
    for k in BASE:
        assert k in d, k
    assert d["dtype"] == "f64" and d["higher_is_better"] is True and d["unit"] == "panel-EM-iterations/s" and d["value"] > 0
    assert set(("sm_mhz", "sm_max_mhz", "power_limit_w", "gpu")) <= set(d["clocks"])
    c1, c5 = d["config"]["c1"], d["config"]["c5"]
    assert c1["shape"]["B"] == 296 and c1["shape"]["p"] == 4 and c1["shape"]["em_iters"] == 20 and c1["shape"]["n_constr"] == 32
    assert c5["shape"]["B"] == 1250 and c5["shape"]["p"] == 1 and c5["shape"]["em_iters"] == 50
    for w in (c1, c5):
        for leg in ("restricted", "unrestricted"):
            assert w[leg]["all_status_ok"] is True and w[leg]["panel_em_iters_per_s"] > 0 and w[leg]["kernel_ms"]
        assert w["restricted"]["restriction_max_abs_violation"] < 1e-12
    assert "k_em_mstep_series" in c1["restricted"]["kernel_ms"] and "k_em_mstep_series" in c1["unrestricted"]["kernel_ms"]
    assert "k_emb_mstep_constr<NCB>" in c5["restricted"]["kernel_ms"]
    assert any(n.startswith("k_em_fused2") for n in c5["unrestricted"]["kernel_ms"])
    assert not any(n.startswith("k_em_fused") for n in c5["restricted"]["kernel_ms"])
