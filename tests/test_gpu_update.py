"""The per-cluster update of the 3xTF32 Lloyd pass (csrc/b2k_wg.cuh, UPD) on every instantiation the library compiles
(b2k_fused_tc.cu kInst: KP in {16, 32, 64, 128}, DP in {32, 64, 128}) and on the label patterns that stress its
counting sort and run split: one cluster for every row (one 128-row run per tile), k = 128 with runs of length 1, a
ragged last tile and an empty cluster.

One Lloyd step must equal the fp64 sums implied by the device's own labels (1e-5 relative), and two runs must give
bitwise-equal centres."""
import pytest

pytestmark = pytest.mark.gpu
STEP_RTOL = 1e-5


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    c.set_option("kernel_path", 2)       # fused kernel or fail: never a silent generic fallback
    yield c
    c.close()


def _one_step(ctx, X, C):
    from _fullsize import check_one_step

    labels, _ = ctx.kmeans_assign(X, C)
    before = ctx.stats()["fused_tc_launches"]
    rel, same = check_one_step(ctx, X, C, labels)
    st = ctx.stats()
    assert st["last_path"] == 2 and st["fused_tc_launches"] > before
    assert rel <= STEP_RTOL, rel
    assert same, "two runs of one Lloyd step differ"
    return labels


# (k, d) -> (KP, DP): every 3xTF32 instantiation; n = 20011 leaves a ragged last tile
@pytest.mark.parametrize("k,d", [(5, 20), (16, 64), (12, 128), (32, 32), (24, 60), (32, 128), (48, 32), (64, 64),
                                 (64, 128), (100, 64), (128, 128)])
def test_update_every_instantiation(ctx, k, d):
    from _fullsize import make_blobs

    X, C = make_blobs(20011, d, k, seed=k * 1000 + d)
    _one_step(ctx, X, C)


def test_update_one_cluster(ctx):
    """every row in cluster 0: each tile is one run of 128 rows, summed by one warp"""
    from _fullsize import make_blobs

    X, C = make_blobs(20011, 128, 64, seed=3)
    C[0] = X.mean(0)
    C[1:] = C[1:] + 1000.0
    labels = _one_step(ctx, X, C)
    assert int(labels.max()) == 0 and int(labels.min()) == 0


def test_update_run_length_one(ctx):
    """k = 128 and row i near centre i % 128: every tile holds each label once (128 runs of one row)"""
    import torch

    k, d, n = 128, 128, 128 * 160
    g = torch.Generator(device="cuda").manual_seed(9)
    ctr = torch.rand((k, d), generator=g, device="cuda") * 20 - 10
    z = torch.arange(n, device="cuda") % k
    X = (ctr[z] + 0.1 * torch.randn((n, d), generator=g, device="cuda")).contiguous()
    labels = _one_step(ctx, X, ctr.contiguous())
    assert torch.equal(labels.long(), z)


def test_update_empty_cluster(ctx):
    """a centre no row chooses keeps its value exactly"""
    import torch

    from _fullsize import make_blobs

    X, C = make_blobs(20011, 64, 32, seed=4)
    C[5] = C[5] + 1000.0
    labels = _one_step(ctx, X, C)
    assert int((labels == 5).sum()) == 0
    C1 = C.clone()
    ctx.kmeans_lloyd(X, C1, 1, 0.0)
    assert torch.equal(C1[5], C[5])
