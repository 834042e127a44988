"""bench.py's measurement contract, as far as it can be exercised without a GPU: the reference arm (CPU oracle port)
prints ONE JSON line with the agreed keys, and our arm refuses to run without an H100 instead of falling back."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=600, cwd=ROOT, env=env)


def test_reference_arm_prints_the_contract_line_on_cpu():
    r = _run("--impl", "reference", "--workload", "C1", "--steps", "1", "--warmup", "0", "--cpu-threads", "4")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["value"] > 0 and d["unit"] == "maps/s" and d["higher_is_better"] is True
    for k in ("metric", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline", "dtype", "data", "config"):
        assert k in d, k
    assert "workload" in d["config"] and "model" not in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] == 4 and cb["value"] == d["value"] and cb["sample"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["unit"] == d["unit"]
    assert e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0


def test_our_arm_refuses_to_run_without_a_gpu():
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    r = _run("--steps", "1", "--warmup", "0")
    assert r.returncode != 0
    assert "no CPU path" in (r.stderr + r.stdout)
