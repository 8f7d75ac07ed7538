"""The Gaussian mixture kernels (b2k_gmm.cu) compile for sm_90a with no spills and no stack frame (ptxas -v, the
library's flags): the three wgmma E-pass instantiations, the generic E pass, the planes and the moments pass.  The
weighted Gram passes are the W = true instances of b2k_gram.cu (test_gram_ptxas_cpu.py)."""
from test_ann_ptxas_cpu import _entries


def test_gmm_kernels_have_no_spills_or_stack(tmp_path):
    entries = _entries("b2k_gmm.cu", tmp_path)
    names = ["k_gmm_e_wgILi1E", "k_gmm_e_wgILi2E", "k_gmm_e_wgILi4E", "k_gmm_e_generic", "k_gmm_planes", "k_gmm_mom"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if "k_gmm" in e and any(v)}
    assert not bad, bad
