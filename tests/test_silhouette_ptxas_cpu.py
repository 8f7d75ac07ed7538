"""The silhouette kernels (b2k_silhouette.cu) compile for sm_90a with no spills and no stack frame (ptxas -v, the
library's flags).  The wgmma pass shifts its tile in shared memory, so the shared pipeline of b2k_pair_wg.cuh, and with
it k_knn_wg and k_db_wg, is left as it was."""
from test_ann_ptxas_cpu import _entries


def test_silhouette_kernels_have_no_spills_or_stack(tmp_path):
    entries = _entries("b2k_silhouette.cu", tmp_path)
    names = ["k_sil_wgILi1ELb0", "k_sil_wgILi2ELb0", "k_sil_wgILi4ELb0", "k_sil_wgILi1ELb1", "k_sil_wgILi2ELb1",
             "k_sil_wgILi4ELb1", "k_sil_genericILb0", "k_sil_genericILb1", "k_sil_statsILb0", "k_sil_statsILb1",
             "k_sil_stats_fold", "k_sil_shift", "k_sil_means", "k_sil_cid"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if "k_sil" in e and any(v)}
    assert not bad, bad
