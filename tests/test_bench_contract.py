"""CPU only: the committed bench lines (profiles/h100_bench_*.json, written by bench.py on an H100) carry every key a
consumer of the bench line reads -- a guard against silently dropping one when bench.py is edited."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
        "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"]


def _load(name):
    p = os.path.join(ROOT, "profiles", name)
    if not os.path.exists(p):
        pytest.skip(name + " not committed")
    return json.load(open(p))


@pytest.mark.parametrize("config", ["c5", "c4", "c3", "c2-single"])
def test_bench_line_has_contract_keys(config):
    d = _load(f"h100_bench_{config}.json")
    for k in BASE:
        assert k in d, k
    assert "workload" in d["config"] and d["dtype"] == "f64" and d["higher_is_better"] is True
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"], k
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in d["roofline"], k
    assert abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-9
    assert d["gpu_launches"] > 0 and set(("sm_mhz", "sm_max_mhz", "reasons")) <= set(d["clocks"])


def test_headline_line():
    d = _load("h100_bench_c5.json")
    assert d["metric"].startswith("EM iters/sec") and d["scaling"] == "weak" and d["n_gpus"] == 1
    cb = d["cpu_baseline"]
    assert cb and set(("value", "unit", "cores", "kind", "sample")) <= set(cb) and cb["kind"] in ("port", "reference")
    assert d["roofline"]["bound"] == "hbm" and 0.3 < d["roofline"]["frac"] < 1.0
    assert d["e2e_to_convergence"]["all_status_ok"] is True


def test_reference_arm_line():
    d = _load("h100_bench_ref.json")
    assert d["impl"] == "reference" and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["value"] == d["value"]
