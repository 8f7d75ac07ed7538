"""The search passes that IVF-Flat shares with exact k-NN (b2k_knn.cu: the wgmma and generic scans, the refine, the
merge, the prep), IVF-Flat's own kernels (b2k_ivf.cu) and DBSCAN's count and union passes (b2k_dbscan.cu, on the same
wgmma pipeline) compile for sm_90a with no spills (ptxas -v, the library's flags)."""
import os
import re
import subprocess

import pytest

from test_eval_ptxas_cpu import CSRC, _nvcc


def _entries(src, tmp_path):
    res = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
                          "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o",
                          str(tmp_path / (src + ".o"))], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    entries, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            entries[current] = tuple(int(v) for v in m.groups())
            current = None
    return entries


@pytest.mark.parametrize("src,names", [
    ("b2k_knn.cu", ["k_knn_wgILi1", "k_knn_wgILi2", "k_knn_wgILi4", "k_knn_generic", "k_knn_refine", "k_knn_merge",
                    "k_knn_prep", "k_knn_shift_q"]),
    ("b2k_ivf.cu", ["k_ivf_nonfinite", "k_ivf_train_rows", "k_ivf_offsets", "k_ivf_perm", "k_ivf_pairs", "k_ivf_slots",
                    "k_ivf_gather_q", "k_ivf_narrow"]),
    ("b2k_dbscan.cu", ["k_db_wgILi1ELb0", "k_db_wgILi2ELb0", "k_db_wgILi4ELb0", "k_db_wgILi1ELb1", "k_db_wgILi2ELb1",
                       "k_db_wgILi4ELb1", "k_db_generic"]),
])
def test_search_kernels_have_no_spills(tmp_path, src, names):
    entries = _entries(src, tmp_path)
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    spilled = {e: v for e, v in entries.items() if ("k_knn" in e or "k_ivf" in e or "k_db" in e) and (v[1] or v[2])}
    assert not spilled, spilled
