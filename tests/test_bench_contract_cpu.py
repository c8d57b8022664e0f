"""The bench.py output contract, checked on the committed result lines (profiles/h100_bench_*.json: one H100) and on the
helpers that do not need a GPU."""
import importlib.util
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    return json.loads(open(os.path.join(ROOT, "profiles", name)).read())


def _bench():
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_committed_gpu_lines_carry_every_contract_key():
    for name, n in (("h100_bench_1gpu.json", 1),):
        d = _load(name)
        for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                  "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline"):
            assert k in d, (name, k)
        assert d["n_gpus"] == n and d["scaling"] == "weak" and d["higher_is_better"] is True
        assert "workload" in d["config"] and "model" not in d["config"]
        assert d["gpu_launches"] > 0
        assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
        r = d["roofline"]
        for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
            assert k in r, (name, k)
        assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
        assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    one = _load("h100_bench_1gpu.json")
    # the CPU arm times the reference's own eager code (oracle/_ref recipe), not the port
    assert one["cpu_baseline"]["kind"] == "reference" and one["cpu_baseline"]["cores"] >= 1
    assert one["roofline"]["traffic"] is not None


def test_reference_arm_line():
    d = _load("h100_bench_reference_arm.json")
    assert d["impl"] == "reference" and d["cpu_baseline"]["kind"] == "reference"
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["e2e"]["value"] == d["value"] == d["cpu_baseline"]["value"]


def test_research_lines():
    # BASELINE configs 2 / 3 (bench.py --workload ml20m | amzn_books), one line each
    lines = [json.loads(line) for line in open(os.path.join(ROOT, "profiles", "h100_bench_research.json"))]
    assert len(lines) == 2
    for d in lines:
        assert d["unit"] == "sequences/s" and d["value"] > 0 and "research" in d["metric"]
        assert d["n_gpus"] == 1 and d["steps"] >= 1 and d["gpu_launches"] > 0
        assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
