"""The binary evaluation's kernels, the score passes (b2k_eval.cu) and the curve pass (b2k_binary.cu), compile for
sm_90a with no spills (ptxas -v, the library's flags)."""
import pytest

from test_ann_ptxas_cpu import _entries


@pytest.mark.parametrize("src,names", [
    ("b2k_eval.cu", ["k_score_linearILb0", "k_score_linearILb1", "k_score_forestILb0", "k_score_forestILb1"]),
    ("b2k_binary.cu", ["k_bin_keys", "k_bin_flags", "k_bin_points", "k_bin_area", "k_bin_fold"]),
])
def test_binary_kernels_have_no_spills(tmp_path, src, names):
    entries = _entries(src, tmp_path)
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    mine = {e: v for e, v in entries.items() if "k_score_" in e or "k_bin_" in e}
    spilled = {e: v for e, v in mine.items() if v[0] or v[1] or v[2]}
    assert not spilled, spilled
