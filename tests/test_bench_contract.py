"""The bench line committed under profiles/ carries every key of the bench.py contract (checked on CPU: the line itself was
produced on an H100 by `python bench.py`)."""
import json, os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_committed_bench_line_has_contract_keys():
    d = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_n16384.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks"):
        assert k in d, k
    assert d["dtype"] == "f64" and d["unit"] == "TFLOP/s" and d["vs_baseline"] is None and "workload" in d["config"]
    r = d["roofline"]
    assert r["bound"] == "tensor" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["unit"] == "TFLOP/s"
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] >= 1
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] < d["value"]
    assert d["gpu_launches"] > 0 and d["residual"] < 1e-12
    assert d["roofline"]["peak_source"].startswith("DMMA.16x8x16 register loop")  # the peak is measured in the run, not a constant
    assert d["cacqr"]["residual"] < 1e-12 and d["cacqr"]["orthogonality"] < 1e-12 and d["strong"]["residual"] < 1e-12
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


def test_bench_workloads_match_baseline_configs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert b.WORKLOADS[1][0] == 16384 and b.WORKLOADS[8][0] == 49152  # BASELINE.json configs[1], configs[2]
    assert b.workload_config(1, 16384, 1, -5)["base_case"] == 512 and b.workload_config(8, 49152, 2, -4)["base_case"] == 768
