"""The bisecting k-means kernels (b2k_bisect.cu) compile for sm_90a with no spills and no stack frame (ptxas -v, the
library's flags): both split-pass instantiations (float4 and scalar rows), the fold, centre, partition and predict
passes.  The cluster sizes come from the shared label count of b2k_generic.cu (test_gram_ptxas_cpu.py)."""
from test_ann_ptxas_cpu import _entries


def test_bkm_kernels_have_no_spills_or_stack(tmp_path):
    entries = _entries("b2k_bisect.cu", tmp_path)
    names = ["k_bkm_splitILb0E", "k_bkm_splitILb1E", "k_bkm_fold", "k_bkm_centres", "k_bkm_count", "k_bkm_scan",
             "k_bkm_scatter", "k_bkm_iota", "k_bkm_predict"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if "k_bkm" in e and any(v)}
    assert not bad, bad
