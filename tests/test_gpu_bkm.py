"""b2k_bkm_fit / b2k_bkm_predict on the device against the fp64 oracle (tests/bkm_oracle.py): exact trees on data far
from any tie, a self-consistent tree on data with no cluster structure, the hand-derived known answers, k > n, an
empty child, offset data, a non-finite value, bitwise repeats, and a steady state in which each split CTA runs many
units over several levels."""
import json
import os

import numpy as np
import pytest

import bkm_oracle as bo

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bkm_known_answers.json")


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200._native import Context

    c = Context(0)
    yield c
    c.close()


def _dev(X):
    import torch

    return torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).cuda()


def _blobs(n, d, nb, seed, scale=10.0, spread=0.05, shift=0.0):
    rng = np.random.default_rng(seed)
    means = rng.uniform(-scale, scale, size=(nb, d))
    z = rng.integers(0, nb, size=n)
    return (means[z] + spread * rng.normal(size=(n, d)) + shift).astype(np.float32)


def _oracle_nodes(out):
    return {int(i): (int(s), c, float(q)) for i, c, s, q in
            zip(out["node_index"], out["centers"], out["sizes"], out["costs"])}


def _match(out, ref, X, ctx):
    nodes = ref["nodes"]
    order = bo.dfs(nodes)
    assert list(out["node_index"]) == order
    assert list(out["sizes"]) == [nodes[i][0] for i in order]
    scale = float(np.abs(X).max())
    np.testing.assert_allclose(out["centers"], np.stack([nodes[i][1] for i in order]), rtol=0, atol=1e-10 * scale)
    want = np.array([nodes[i][2] for i in order])
    np.testing.assert_allclose(out["costs"], want, rtol=1e-9, atol=1e-9 * want.max())
    assert out["training_cost"] == pytest.approx(bo.training_cost(nodes), rel=1e-9, abs=1e-9 * want.max())
    lab_ref, cost_ref = bo.predict(X, nodes)
    lab, cost = ctx.bkm_predict(_dev(X), out["node_index"], out["centers"], with_cost=True)
    np.testing.assert_array_equal(lab.cpu().numpy(), lab_ref)
    np.testing.assert_allclose(cost.cpu().numpy(), cost_ref, rtol=1e-9, atol=1e-9 * want.max())
    np.testing.assert_array_equal(out["cluster_sizes"], np.bincount(lab_ref, minlength=len(ref["leaves"])))


# (d, k, min_divisible, blobs): both forms of minDivisibleClusterSize, d across the float4 / scalar split paths
EXACT = [(1, 7, 1.0, 9), (3, 64, 0.01, 80), (4, 7, 5.0, 12), (4, 2, 1.0, 3), (128, 64, 1.0, 80), (129, 7, 0.05, 12),
         (1000, 2, 1.0, 4), (1000, 7, 3.0, 10)]


@pytest.mark.parametrize("d,k,md,nb", EXACT)
def test_exact_on_tie_free_data(ctx, d, k, md, nb):
    X = _blobs(3000, d, nb, seed=d * 100 + k)
    ref = bo.fit(X, k, max_iter=20, min_divisible=md, seed=5)
    assert ref["margin"] > 1e-11, ref["margin"]   # every side decision of the oracle is far from a tie
    out = ctx.bkm_fit(_dev(X), k, max_iter=20, min_divisible=md, seed=5)
    _match(out, ref, X, ctx)
    assert out["n_levels"] == len(ref["levels"])


def _descend(X, nodes):
    """Leaf by descent in fp64 and the smallest relative margin of any of the row's decisions."""
    X = X.astype(np.float64)
    lv = {i: j for j, i in enumerate(bo.leaves(nodes))}
    lab = np.empty(len(X), np.int32)
    marg = np.full(len(X), np.inf)
    for r, x in enumerate(X):
        i = 1
        while i not in lv:
            a, b = 2 * i, 2 * i + 1
            if a in nodes and b in nodes:
                da, db = ((x - nodes[a][1]) ** 2).sum(), ((x - nodes[b][1]) ** 2).sum()
                marg[r] = min(marg[r], abs(da - db) / max(da + db, 1e-300))
                i = a if da <= db else b
            else:
                i = a if a in nodes else b
        lab[r] = lv[i]
    return lab, marg


def test_general_data_tree_is_self_consistent(ctx):
    rng = np.random.default_rng(3)
    X = rng.normal(size=(4000, 16)).astype(np.float32)
    out = ctx.bkm_fit(_dev(X), 12, max_iter=10, seed=1)
    nodes = _oracle_nodes(out)
    # (a parent's stored size is its last iteration's count, so its children's sizes need not add up to it)
    assert len(bo.leaves(nodes)) == 12 and len(out["cluster_sizes"]) == 12
    assert out["cluster_sizes"].sum() == 4000
    lab, _ = ctx.bkm_predict(_dev(X), out["node_index"], out["centers"])
    lab = lab.cpu().numpy()
    ref, marg = _descend(X, nodes)
    clear = marg > 1e-12
    assert clear.mean() > 0.99
    np.testing.assert_array_equal(lab[clear], ref[clear])
    np.testing.assert_array_equal(out["cluster_sizes"], np.bincount(lab, minlength=12))
    assert out["training_cost"] == pytest.approx(sum(nodes[i][2] for i in bo.leaves(nodes)), rel=1e-12)


@pytest.mark.parametrize("case", json.load(open(GOLDEN)), ids=lambda c: c["name"])
def test_known_answers(ctx, case):
    X = np.asarray(case["X"], dtype=np.float32)
    out = ctx.bkm_fit(_dev(X), case["k"], max_iter=case["max_iter"], min_divisible=case["min_divisible"], seed=11)
    assert list(out["node_index"]) == case["node_index"]
    assert list(out["sizes"]) == case["sizes"]
    np.testing.assert_allclose(out["centers"], case["centers"], atol=1e-12)
    np.testing.assert_allclose(out["costs"], case["costs"], atol=1e-12)
    assert out["training_cost"] == pytest.approx(case["training_cost"], abs=1e-12)
    assert list(out["cluster_sizes"]) == case["cluster_sizes"]
    lab, _ = ctx.bkm_predict(_dev(X), out["node_index"], out["centers"])
    assert list(lab.cpu().numpy()) == case["labels"]


def test_k_above_n(ctx):
    X = _blobs(5, 3, 5, seed=2)
    ref = bo.fit(X, 10, seed=4)
    out = ctx.bkm_fit(_dev(X), 10, seed=4)
    _match(out, ref, X, ctx)
    assert len(out["cluster_sizes"]) <= 5


def test_empty_child_mid_level(ctx):
    # integer rows whose centres are exact: level 1 splits the pattern at the origin from the one at (64, 64); at
    # level 2 the origin node's centre is 0, both its children start there, every row ties left and the right child
    # drops out, while (64, 64) splits properly beside it; need drops by two, leaving 3 leaves for k = 4
    P = np.array([[1, 2], [-1, -2], [3, -1], [-3, 1]], dtype=np.float32)
    X = np.concatenate([P, P + 64])
    ref = bo.fit(X, 4, max_iter=6, seed=2)
    assert ref["levels"] == [[1], [2, 3]] and 4 in ref["nodes"] and 5 not in ref["nodes"]
    assert len(ref["leaves"]) == 3
    out = ctx.bkm_fit(_dev(X), 4, max_iter=6, seed=2)
    _match(out, ref, X, ctx)


def test_offset_data(ctx):
    X = _blobs(3000, 8, 6, seed=21, scale=1.0, spread=0.01, shift=1e3)
    ref = bo.fit(X, 6, seed=3)
    assert ref["margin"] > 1e-11, ref["margin"]
    out = ctx.bkm_fit(_dev(X), 6, seed=3)
    _match(out, ref, X, ctx)
    assert min(out["costs"]) > 0.0


def test_non_finite_fails(ctx):
    from spark_rapids_ml_b200._native import B2KError

    X = _blobs(100, 4, 2, seed=1)
    X[17, 2] = np.nan
    with pytest.raises(B2KError, match="NaN or an infinity"):
        ctx.bkm_fit(_dev(X), 3)
    X[17, 2] = np.inf
    with pytest.raises(B2KError, match="NaN or an infinity"):
        ctx.bkm_fit(_dev(X), 3)


@pytest.mark.parametrize("kw,msg", [({"k": 1}, "k must be"), ({"max_iter": 0}, "maxIter"),
                                    ({"min_divisible": 0.0}, "minDivisibleClusterSize")])
def test_argument_errors(ctx, kw, msg):
    from spark_rapids_ml_b200._native import B2KError

    args = {"k": 3, "max_iter": 5, "min_divisible": 1.0}
    args.update(kw)
    k = args.pop("k")
    with pytest.raises(B2KError, match=msg):
        ctx.bkm_fit(_dev(_blobs(50, 4, 2, seed=1)), k, **args)


def test_unsupported_width(ctx):
    from spark_rapids_ml_b200._native import B2KError

    with pytest.raises(B2KError, match="supports d <= 4096"):
        ctx.bkm_fit(_dev(np.zeros((4, 4097), np.float32)), 2)


def _same(a, b):
    for key in ("node_index", "centers", "sizes", "costs", "cluster_sizes"):
        np.testing.assert_array_equal(a[key], b[key])
    assert a["training_cost"] == b["training_cost"]


def test_bitwise_repeat_and_steady_state(ctx):
    # 200 k rows: units of 256 rows, so a level has hundreds of units; with two split CTAs each runs many of them at
    # every level, and the result must be the bits of the full grid
    X = _blobs(200_000, 32, 40, seed=8, spread=1.0)
    a = ctx.bkm_fit(_dev(X), 16, max_iter=8, seed=7)
    b = ctx.bkm_fit(_dev(X), 16, max_iter=8, seed=7)
    _same(a, b)
    assert a["n_levels"] >= 4
    ctx.set_option("grid_limit", 2)
    try:
        c = ctx.bkm_fit(_dev(X), 16, max_iter=8, seed=7)
    finally:
        ctx.set_option("grid_limit", 0)
    _same(a, c)


def test_time_kernels_fills_stats(ctx):
    X = _blobs(20_000, 16, 8, seed=4)
    ctx.set_option("time_kernels", 1)
    try:
        out = ctx.bkm_fit(_dev(X), 8, seed=1)
        st = ctx.stats()
    finally:
        ctx.set_option("time_kernels", 0)
    assert st["last_n_iter"] == out["n_levels"] >= 3
    assert st["last_fused_ms"] > 0 and st["last_reduce_ms"] > 0 and st["last_loop_ms"] > 0
    assert len(out["level_ms"]) == out["n_levels"] and np.all(out["level_ms"] > 0)
