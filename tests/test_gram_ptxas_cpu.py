"""The shared fp64 reduction kernels compile for sm_90a with no spills and no stack frame (ptxas -v, the library's
flags): both instances (unweighted and weighted) of the wgmma and the generic Gram passes of b2k_gram.cu and their
folds and the unpack of a triangle, and the ordered span fold and the label count of b2k_generic.cu."""
import pytest

from test_ann_ptxas_cpu import _entries


@pytest.mark.parametrize("src,names", [
    ("b2k_gram.cu", ["k_gram_wgILb0E", "k_gram_wgILb1E", "k_gram_genericILb0E", "k_gram_genericILb1E",
                     "k_gram_fold_wg", "k_gram_fold_generic", "k_gram_unpack"]),
    ("b2k_generic.cu", ["k_fold_spans", "k_label_counts"]),
])
def test_shared_reduction_kernels_have_no_spills_or_stack(src, names, tmp_path):
    entries = _entries(src, tmp_path)
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if any(n in e for n in names) and any(v)}
    assert not bad, bad
