"""bench.py contract checks that need no GPU: the reference arm runs on the CPU and prints ONE JSON
line with the keys a consumer reads; the GPU arm refuses to run without a CUDA device."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, "bench.py")


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, BENCH, "--impl", "reference", "--workload", "c2", "--steps", "1",
                          "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "utterances/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["vs_baseline"] is None and d["dtype"] == "f32" and d["data"] == "synthetic"
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert "workload" in d["config"] and "model" not in d["config"]


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, BENCH, "--impl", "reference", "--gpus", "2", "--steps", "1",
                          "--warmup", "1"], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_b200_arm_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        return
    out = subprocess.run([sys.executable, BENCH, "--steps", "1", "--warmup", "1"], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode != 0 and "no CUDA device" in (out.stderr + out.stdout)
