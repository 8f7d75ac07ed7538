"""The multilayer perceptron kernels (b2k_mlp.cu) compile for sm_90a with no spills and no stack frame (ptxas -v, the
library's flags): every wgmma instantiation (row products and cross-Gram at NB = 16, 32, 64, 128), the two generic
fp64 instantiations, the softmax, loss, fold and predict passes."""
from test_ann_ptxas_cpu import _entries


def test_mlp_kernels_have_no_spills_or_stack(tmp_path):
    entries = _entries("b2k_mlp.cu", tmp_path)
    names = [f"k_mlp_wgILi{nb}ELb{g}E" for nb in (16, 32, 64, 128) for g in (0, 1)]
    names += ["k_mlp_simtIfdE", "k_mlp_simtIddE", "k_mlp_softmaxIfE", "k_mlp_softmaxIdE", "k_mlp_loss_units",
              "k_mlp_fold", "k_mlp_predict_rowsIfE", "k_mlp_predict_rowsIdE"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if "k_mlp" in e and any(v)}
    assert not bad, bad
