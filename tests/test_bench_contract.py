"""bench.py contract on CPU: the reference arm (oracle C/OpenMP port on host cores) prints ONE JSON line with the keys the
driver reads; the GPU arm refuses to run without a GPU instead of falling back to the CPU."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True,
                          cwd=ROOT, env=dict(os.environ, **(env or {})), timeout=600)


def test_reference_arm_json_line():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "1", "--cpu-sample-rows", "20000"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["metric"] == "kmeans_fit_samples_per_sec" and j["unit"] == "samples/s"
    assert j["higher_is_better"] is True and j["steps"] == 1 and j["value"] > 0
    assert j["cpu_baseline"]["kind"] in ("port", "reference") and j["cpu_baseline"]["cores"] >= 1
    assert j["e2e"]["h2d_bytes_per_step"] == 0 and j["e2e"]["d2h_bytes_per_step"] == 0
    assert j["e2e"]["value"] == j["value"]


def test_reference_arm_nonzero_ranks_do_no_work():
    r = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"], env={"RANK": "1", "WORLD_SIZE": "2"})
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_b200_arm_fails_loudly_without_gpu():
    r = _run(["--steps", "1", "--warmup", "1", "--no-e2e", "--no-cpu-baseline"])
    assert r.returncode != 0
    assert "{\"metric\"" not in r.stdout
