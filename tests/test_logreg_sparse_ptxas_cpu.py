"""The sparse logistic regression kernels (b2k_logreg_sparse.cu) and the CSR ingest kernel (b2k_ingest.cu) compile for
sm_90a with no spills and no stack frame (ptxas -v, the library's flags)."""
from test_ann_ptxas_cpu import _entries


def test_sparse_logreg_kernels_have_no_spills(tmp_path):
    entries = _entries("b2k_logreg_sparse.cu", tmp_path)
    names = ["k_csr_check", "k_csr_pack", "k_csc_passILi0", "k_csc_passILi1", "k_csc_passILi2", "k_csc_carry",
             "k_csr_rowsILb1", "k_csr_rowsILb0", "k_csr_rows_fold"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if any(v)}
    assert not bad, bad


def test_csr_ingest_kernel_has_no_spills(tmp_path):
    entries = _entries("b2k_ingest.cu", tmp_path)
    got = {e: v for e, v in entries.items() if "k_csr_ingest" in e}
    assert len(got) == 2, sorted(entries)
    assert not any(any(v) for v in got.values()), got
