"""Exact k-NN at its edges: b2k_knn_search on data far from the origin, on integer data where every step is exact, at
every DP width and tile boundary, at the largest split count, under a persistent schedule squeezed onto few CTAs, at
large k, with misaligned queries and with non-finite rows.  Every comparison with floating-point data uses the parity
rule of tests/knn_oracle.py; the integer cases compare bits."""
import numpy as np
import pytest

import knn_oracle as ko

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200 import _native  # noqa: E402

# tile and split constants of the planner in csrc/b2k_knn.cu
KW_TM, KW_N, KW_SMAX = 128, 128, 256   # wgmma path: queries per tile, items per block, most index splits
GQ, GN = 16, 64                        # generic path: queries per CTA, items per tile


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


def _search(ctx, X, Q, k, path=0, grid=0):
    """(dist, idx, last_path); X and Q are numpy arrays or CUDA tensors."""
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid)
    try:
        Xd = X if torch.is_tensor(X) else torch.from_numpy(X).cuda()
        Qd = Q if torch.is_tensor(Q) else torch.from_numpy(Q).cuda()
        dist, idx = ctx.knn_search(Xd, Qd, k)
        return dist.cpu().numpy(), idx.cpu().numpy(), ctx.stats()["last_path"]
    finally:
        ctx.set_option("kernel_path", 0)
        ctx.set_option("grid_limit", 0)


def _normal(n, nq, d, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) + offset).astype(np.float32)
    Q = (rng.normal(size=(nq, d)) + offset).astype(np.float32)
    return X, Q


def _planned_splits(nq, item_tiles, q_tile):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    ntiles = -(-nq // q_tile)
    return max(1, min(-(-2 * sm // ntiles), item_tiles, KW_SMAX))


def _paths(d, k):
    return [2, 1] if d % 4 == 0 and 4 <= d <= 128 and k <= 64 else [1]


# ---- 1. data far from the origin ----
@pytest.mark.parametrize("path", [2, 1])
@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4])
@pytest.mark.parametrize("k", [8, 64])
def test_offsets(ctx, path, d, offset, k):
    # An fp32 screen ||x||^2 - 2 q.x loses the gaps between neighbours when ||x||^2 is large; the wgmma pass screens in
    # a frame shifted by an item row, so the returned set does not depend on where the data sits.
    X, Q = _normal(4000, 200, d, seed=int(d + k + np.log10(offset + 1)), offset=offset)
    Q[:10] = X[:10]
    dist, idx, p = _search(ctx, X, Q, k, path=path)
    assert p == path
    assert np.all(dist[:10, 0] == 0.0)
    bad = ko.compare(X, Q, k, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


# ---- 2. integer data: every partial sum is an integer below 2^24, so screen, refine and sqrtf are exact ----
def _int_data(n, nq, d, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-3, 4, size=(n, d)).astype(np.int64), rng.integers(-3, 4, size=(nq, d)).astype(np.int64)


def _int_oracle(Xi, Qi, k):
    """Exact squared distances in int64; the k smallest by (distance, row); distances as float32 sqrt of the sum."""
    d2 = (Qi * Qi).sum(1)[:, None] + (Xi * Xi).sum(1)[None, :] - 2 * (Qi @ Xi.T)
    key = d2 * Xi.shape[0] + np.arange(Xi.shape[0])[None, :]
    idx = np.argsort(key, axis=1, kind="stable")[:, :k]
    return np.sqrt(np.take_along_axis(d2, idx, 1).astype(np.float32)), idx


def _check_int(ctx, Xi, Qi, k, path):
    ref_d, ref_i = _int_oracle(Xi, Qi, k)
    out = []
    for off in (0.0, 1024.0):
        X = (Xi.astype(np.float32) + np.float32(off))
        Q = (Qi.astype(np.float32) + np.float32(off))
        dist, idx, p = _search(ctx, X, Q, k, path=path)
        assert p == path
        np.testing.assert_array_equal(idx, ref_i, err_msg=f"offset {off}")
        np.testing.assert_array_equal(dist.view(np.uint32), ref_d.view(np.uint32), err_msg=f"offset {off}")
        out.append((dist, idx))
    np.testing.assert_array_equal(out[0][0].view(np.uint32), out[1][0].view(np.uint32))
    np.testing.assert_array_equal(out[0][1], out[1][1])


@pytest.mark.parametrize("d,path", [(4, 2), (16, 2), (64, 2), (128, 2), (3, 1), (130, 1)])
def test_integer_data_exact(ctx, d, path):
    Xi, Qi = _int_data(3000, 100, d, seed=d)
    _check_int(ctx, Xi, Qi, 16, path)


@pytest.mark.parametrize("path", [2, 1])
def test_integer_tie_group_across_splits(ctx, path):
    # ten copies of one row spread over the index (different blocks and splits); queries at distance 0 and 1 from it,
    # k = 6 cuts inside the tie group, which must give its lowest rows
    d = 64
    Xi, Qi = _int_data(3000, 100, d, seed=11)
    dup = [123, 401, 777, 1100, 1499, 1800, 2222, 2500, 2801, 2999]
    Xi[dup] = Xi[dup[0]]
    Qi[0] = Xi[dup[0]]
    Qi[1] = Xi[dup[0]]
    Qi[1, 0] += 1 if Qi[1, 0] < 3 else -1
    nq, n = Qi.shape[0], Xi.shape[0]
    S = _planned_splits(nq, -(-n // KW_N) if path == 2 else -(-n // GN), KW_TM if path == 2 else GQ)
    assert S >= 8   # the copies lie in different splits
    _check_int(ctx, Xi, Qi, 6, path)
    _, idx = _int_oracle(Xi, Qi, 6)
    assert idx[0].tolist() == dup[:6]


# ---- 3. shape edges of the wgmma path: every DP width and both sides of each boundary ----
SHAPES = [  # (d, n_items, k, n_queries)
    (4, 1, 1, 1), (8, 2, 2, 127), (28, 63, 63, 128), (32, 64, 64, 129),
    (36, 127, 1, 257), (60, 128, 2, 1), (64, 129, 63, 127), (68, 300, 64, 128),
    (100, 127, 64, 129), (124, 128, 63, 257), (128, 129, 1, 1), (128, 300, 2, 127),
    (4, 300, 64, 257), (68, 64, 64, 1), (100, 2, 2, 129), (124, 1, 1, 128),
]


@pytest.mark.parametrize("d,n,k,nq", SHAPES)
def test_shape_edges_fused(ctx, d, n, k, nq):
    X, Q = _normal(n, nq, d, seed=d * 1000 + n + k)
    dist, idx, p = _search(ctx, X, Q, k, path=2)
    assert p == 2
    assert np.all(idx >= 0)
    if k == n:   # every item exactly once
        assert np.all(np.sort(idx, axis=1) == np.arange(n)[None, :])
    bad = ko.compare(X, Q, k, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


# ---- 4. splits: the largest split count, and splits holding fewer items than k ----
@pytest.mark.parametrize("path,n,nq,d,k", [(2, 40000, 128, 128, 64), (1, 20000, 16, 20, 64)])
def test_largest_split_count(ctx, path, n, nq, d, k):
    item_tiles = -(-n // KW_N) if path == 2 else -(-n // GN)
    assert _planned_splits(nq, item_tiles, KW_TM if path == 2 else GQ) == KW_SMAX   # all 8 list heads per lane
    X, Q = _normal(n, nq, d, seed=n + d)
    dist, idx, p = _search(ctx, X, Q, k, path=path)
    assert p == path
    bad = ko.compare(X, Q, k, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


@pytest.mark.parametrize("path", [2, 1])
def test_splits_shorter_than_k(ctx, path):
    # 300 items, k = 64: the last block (wgmma) or tile (generic) holds 44 items, so its split's list ends in padding
    X, Q = _normal(300, 5, 64, seed=300)
    item_tiles = 3 if path == 2 else 5
    assert _planned_splits(5, item_tiles, KW_TM if path == 2 else GQ) == item_tiles
    dist, idx, p = _search(ctx, X, Q, 64, path=path)
    assert p == path and np.all(idx >= 0)
    bad = ko.compare(X, Q, 64, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


# ---- 5. persistent schedule: the global top-k by (screen, row) does not depend on the split count ----
@pytest.mark.parametrize("d", [32, 64, 128])
def test_persistent_grid_invariance(ctx, d):
    X, Q = _normal(20011, 1000, d, seed=d + 5)   # 8 query tiles
    Xd, Qd = torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda()
    ref = _search(ctx, Xd, Qd, 10, path=2)
    bad = ko.compare(X, Q, 10, ref[0], ref[1])
    assert bad["n_outside_margin"] == 0, bad
    for grid in (1, 3, 7):   # grid 1: one CTA runs every unit, the query-tile barrier turns 8 x S times
        dist, idx, _ = _search(ctx, Xd, Qd, 10, path=2, grid=grid)
        np.testing.assert_array_equal(idx, ref[1], err_msg=f"grid {grid}")
        np.testing.assert_array_equal(dist.view(np.uint32), ref[0].view(np.uint32), err_msg=f"grid {grid}")


# ---- 6. generic path at large k ----
@pytest.mark.parametrize("d", [1, 3, 33, 129, 300, 1000])
@pytest.mark.parametrize("k", [200, 1024])
def test_generic_large_k(ctx, d, k):
    X, Q = _normal(3000, 40, d, seed=d * 7 + k)
    Xd, Qd = torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda()
    d1, i1, p = _search(ctx, Xd, Qd, k)
    d2, i2, _ = _search(ctx, Xd, Qd, k)
    assert p == 1
    np.testing.assert_array_equal(i1, i2)
    np.testing.assert_array_equal(d1.view(np.uint32), d2.view(np.uint32))
    bad = ko.compare(X, Q, k, d1, i1)
    assert bad["n_outside_margin"] == 0, bad


def test_generic_k_equals_n_total(ctx):
    X, Q = _normal(1024, 20, 3, seed=1024)
    dist, idx, p = _search(ctx, X, Q, 1024)
    assert p == 1
    assert np.all(np.sort(idx, axis=1) == np.arange(1024)[None, :])
    bad = ko.compare(X, Q, 1024, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


# ---- 7. queries that are not 16-byte aligned ----
def test_misaligned_queries(ctx):
    X, Q = _normal(3000, 50, 128, seed=77)
    Xd = torch.from_numpy(X).cuda()
    buf = torch.empty(Q.size + 1, dtype=torch.float32, device="cuda")
    Qv = buf[1:].view(Q.shape)   # starts 4 bytes into the buffer
    Qv.copy_(torch.from_numpy(Q))
    assert Qv.data_ptr() % 16 != 0 and Qv.is_contiguous()
    dm, im, p = _search(ctx, Xd, Qv, 16)
    assert p == 1   # the wgmma path needs aligned queries
    da, ia, _ = _search(ctx, Xd, torch.from_numpy(Q).cuda(), 16, path=1)
    np.testing.assert_array_equal(im, ia)
    np.testing.assert_array_equal(dm, da)
    assert ko.compare(X, Q, 16, dm, im)["n_outside_margin"] == 0
    with pytest.raises(_native.B2KError):
        _search(ctx, Xd, Qv, 16, path=2)


# ---- 8. non-finite rows ----
@pytest.mark.parametrize("path,d", [(2, 128), (2, 32), (1, 128), (1, 20)])
def test_non_finite_rows(ctx, path, d):
    # NaN in item row 0 (the row the wgmma screen shifts by) and +inf in another item; a NaN query among finite ones
    X, Q = _normal(3000, 60, d, seed=d + path)
    X[0, 3] = np.nan
    X[777, 0] = np.inf
    Q[17, 5] = np.nan
    k = 16
    dist, idx, p = _search(ctx, X, Q, k, path=path)
    assert p == path
    finite = np.array([r for r in range(X.shape[0]) if r not in (0, 777)])
    keep = np.array([i for i in range(Q.shape[0]) if i != 17])
    bad = ko.compare(X[finite], Q[keep], k, dist[keep], idx[keep], ids=finite)
    assert bad["n_outside_margin"] == 0, bad
    # the NaN query finds nothing (DESIGN 11.1) and leaves every other query's result as it was
    assert np.all(np.isinf(dist[17])) and np.all(idx[17] == -1)
    Q2 = Q.copy()
    Q2[17] = 0.0
    dist2, idx2, _ = _search(ctx, X, Q2, k, path=path)
    np.testing.assert_array_equal(idx[keep], idx2[keep])
    np.testing.assert_array_equal(dist[keep].view(np.uint32), dist2[keep].view(np.uint32))
