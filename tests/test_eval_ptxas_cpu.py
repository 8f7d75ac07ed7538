"""The evaluation pass compiles for sm_90a with no spills in any kernel instantiation (ptxas -v, the library's flags)."""
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark_rapids_ml_b200", "csrc")


def _nvcc():
    home = os.environ.get("CUDA_HOME", "")
    for cand in (os.path.join(home, "bin", "nvcc") if home else "", shutil.which("nvcc") or "",
                 "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    pytest.fail("nvcc not found: the library cannot be built without it")


def test_eval_kernels_have_no_spills(tmp_path):
    res = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
                          "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "b2k_eval.cu"), "-o",
                          str(tmp_path / "b2k_eval.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    entries = {}
    current = None
    for line in res.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            entries[current] = tuple(int(v) for v in m.groups())
            current = None
    kernels = {k: v for k, v in entries.items() if "k_eval_" in k}
    # linear and forest x {vector, scalar staging} x {classification, regression}, two folds, the label check
    assert sum("k_eval_linear" in k for k in kernels) == 4 and sum("k_eval_forest" in k for k in kernels) == 4
    assert len(kernels) >= 11, sorted(kernels)
    spilled = {k: v for k, v in kernels.items() if v[1] or v[2]}
    assert not spilled, spilled
