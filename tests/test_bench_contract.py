"""The bench.py contract (SURVEY §8d): the reference arm runs here on CPU (small workload) and must print ONE JSON line
with the agreed keys; the committed H100 line (tests/golden/bench_line_h100.json) must carry the same keys plus the GPU-only ones."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
             "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"}


def test_reference_arm_prints_one_contract_line():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "tinyllamas-15m-q8_0",
                        "--steps", "3", "--warmup", "3"], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert BASE_KEYS <= set(d), BASE_KEYS - set(d)
    assert d["impl"] == "reference" and d["metric"] == "decode_tokens_per_s" and d["unit"] == "tok/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "tok/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0 and "workload" in d["config"]


def test_reference_arm_other_ranks_stay_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=120)
    assert p.returncode == 0 and p.stdout.strip() == ""


def test_committed_h100_line_has_the_contract_keys():
    with open(os.path.join(ROOT, "tests", "golden", "bench_line_h100.json")) as f:
        d = json.load(f)
    assert BASE_KEYS | {"roofline", "clocks", "gpu"} <= set(d)
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(r) and r["bound"] == "hbm" and r["unit"] == "GB/s"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(r["achieved"] - r["algorithmic_bytes_per_launch"] / (r["us_per_launch"] * 1e-6) / 1e9) < 1e-3 * r["achieved"]
    assert r["traffic"] is None or r["traffic"] >= r["algorithmic_bytes_per_launch"]     # measured DRAM bytes, when a profiler gave them
    assert d["gpu_launches"] == d["steps"] and d["n_gpus"] == 1 and d["warmup"] >= 3
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] == 32000 * 4 + 8      # logits + sampled id
    assert d["clocks"]["samples"] > 0 and d["cpu_baseline"]["kind"] == "port"
    assert d["gpu"]["name"].startswith("NVIDIA H100") and d["gpu"]["power_limit_w"] > 0       # what the numbers were measured on
