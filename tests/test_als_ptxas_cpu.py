"""The ALS kernels (b2k_als.cu) compile for sm_90a with no spills and no stack frame (ptxas -v, the library's flags):
the eight normal-equation instantiations (ranks up to 16, 32, 64 and 128, explicit and implicit), the solve, start,
predict and recommend passes and the setup passes."""
from test_ann_ptxas_cpu import _entries


def test_als_kernels_have_no_spills_or_stack(tmp_path):
    entries = _entries("b2k_als.cu", tmp_path)
    names = [f"k_als_normalILi{nt}ELi{mt}ELi{rp}ELb{b}E" for nt, mt, rp in ((64, 1, 16), (64, 1, 32), (160, 1, 64),
                                                                            (192, 3, 128)) for b in (0, 1)]
    names += ["k_als_solve", "k_als_start", "k_als_predict", "k_als_recommend", "k_als_check", "k_als_dense",
              "k_als_pack", "k_als_own", "k_als_keys", "k_als_unpack", "k_als_ptr", "k_als_count"]
    for n in names:
        assert any(n in e for e in entries), (n, sorted(entries))
    bad = {e: v for e, v in entries.items() if "k_als" in e and any(v)}
    assert not bad, bad
