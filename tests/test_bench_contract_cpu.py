"""bench.py's driver contract, checked without a GPU: the reference arm (`--impl reference`, the reference op sequence on
the host cores) prints one JSON line carrying every key the contract names, and its `config` is the SAME dict as the one
the CUDA arm printed on an H100 (tests/golden/bench_line_1gpu.json) - the two arms are compared on it."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONTRACT_KEYS = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                 "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline", "gpu_launches")


def test_reference_arm_line_and_shared_config():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    lines = [ln for ln in p.stdout.decode().splitlines() if ln.startswith("{")]
    assert len(lines) == 1, "exactly one JSON line"
    d = json.loads(lines[0])
    assert d["impl"] == "reference"
    for k in CONTRACT_KEYS:
        assert k in d, k
    assert d["metric"] == "seed_nodes_per_sec" and d["higher_is_better"] is True and d["value"] > 0
    assert d["steps"] == 1 and d["warmup"] == 1 and d["n_gpus"] == 1 and d["gpu_launches"] == 0
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "seeds" in cb["sample"]
    gpu_line = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_line_1gpu.json")))
    assert gpu_line["config"] == d["config"], "both arms must describe the workload with the same config dict"
    for k in ("metric", "unit", "higher_is_better", "scaling", "data"):
        assert gpu_line[k] == d[k], k
    assert "model" not in d["config"] and "workload" in d["config"]


def test_reference_arm_on_other_ranks_does_no_work():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1",
                        "--warmup", "1"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    assert p.returncode == 0 and p.stdout.decode().strip() == ""
