"""IVF-Flat search (b2k_ivf_search) through the C ABI on both scan paths, checked step by step against tests/ann_oracle.py:
the item lists, the probes and the result over the probed lists, with injected and trained centres, at its edges (an
empty list, fewer than k items, a NaN query, a non-finite item, data far from the origin), bitwise against the exact
search when every list is probed, bitwise repeatable, and in a steady state of many units per CTA over two query
chunks."""
import numpy as np
import pytest

import ann_oracle as ao
import knn_oracle as ko

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200 import _native  # noqa: E402


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


def _ivf(ctx, X, Q, k, nlist, nprobe, C=None, path=0, grid=0, **kw):
    """numpy (dist, idx, centers, lists, probes), last_path"""
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid)
    try:
        Cd = None if C is None else torch.from_numpy(np.ascontiguousarray(C, np.float32)).cuda()
        out = ctx.ivf_search(torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda(), k, nlist, nprobe, centers=Cd,
                             return_lists=True, **kw)
        return [o.cpu().numpy() for o in out], ctx.stats()["last_path"]
    finally:
        ctx.set_option("kernel_path", 0)
        ctx.set_option("grid_limit", 0)


def _paths(d, k):
    return [2, 1] if d % 4 == 0 and 4 <= d <= 128 and k <= 64 else [1]


def _blobs(n, nq, d, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(16, d)) * 4
    X = (mu[rng.integers(0, 16, n)] + rng.normal(size=(n, d)) + offset).astype(np.float32)
    Q = (mu[rng.integers(0, 16, nq)] + rng.normal(size=(nq, d)) + offset).astype(np.float32)
    return X, Q


def _check_all(X, Q, k, out, squared=False):
    dist, idx, C, lists, probes = out
    assert ao.check_lists(X, C, lists) == 0
    assert ao.check_probes(C, Q, probes) == 0
    bad = ao.check_result(X, Q, k, lists, probes, dist, idx, squared=squared)
    assert bad == {"n_outside_margin": 0, "n_fill": 0}, bad


LIST_CASES = [(1, 1), (7, 3), (64, 3), (7, 7), (64, 64)]


@pytest.mark.parametrize("d", [2, 3, 32, 100, 128, 132])
@pytest.mark.parametrize("k", [1, 5, 64, 65])
def test_injected_centres_match_oracle(ctx, d, k):
    X, Q = _blobs(1500, 80, d, seed=d * 100 + k)
    nlist, nprobe = LIST_CASES[(d + k) % len(LIST_CASES)]
    C = X[np.random.default_rng(k).choice(X.shape[0], nlist, replace=False)]
    for path in _paths(d, k):
        out, last = _ivf(ctx, X, Q, k, nlist, nprobe, C=C, path=path)
        assert last == (2 if path == 2 else 1)
        np.testing.assert_array_equal(out[2], C)
        _check_all(X, Q, k, out)


@pytest.mark.parametrize("d,k,nlist,nprobe", [(32, 5, 7, 3), (100, 10, 64, 3), (128, 64, 64, 64), (3, 65, 7, 1)])
def test_trained_centres_match_oracle(ctx, d, k, nlist, nprobe):
    X, Q = _blobs(3000, 100, d, seed=7 + d)
    for path in _paths(d, k):
        out, _ = _ivf(ctx, X, Q, k, nlist, nprobe, path=path, n_iters=10)
        _check_all(X, Q, k, out)


@pytest.mark.parametrize("d,k", [(32, 10), (128, 64), (100, 5), (3, 65)])
def test_all_lists_probed_is_exact_search(ctx, d, k):
    rng = np.random.default_rng(d + k)
    Xi = rng.integers(-8, 9, size=(2000, d)).astype(np.float32)
    Qi = rng.integers(-8, 9, size=(150, d)).astype(np.float32)
    Xf, Qf = _blobs(2000, 150, d, seed=3)
    C = Xf[:9]
    for path in _paths(d, k):
        ctx.set_option("kernel_path", path)
        try:
            de, ie = [t.cpu().numpy() for t in ctx.knn_search(torch.from_numpy(Xi).cuda(), torch.from_numpy(Qi).cuda(), k)]
        finally:
            ctx.set_option("kernel_path", 0)
        (dist, idx, *_), _ = _ivf(ctx, Xi, Qi, k, 9, 9, C=Xi[:9], path=path)
        np.testing.assert_array_equal(dist.view(np.int32), de.view(np.int32))
        np.testing.assert_array_equal(idx, ie)
        (dist, idx, *_), _ = _ivf(ctx, Xf, Qf, k, 9, 50, C=C, path=path)   # nprobe clamps to nlist
        assert ko.compare(Xf, Qf, k, dist, idx)["n_outside_margin"] == 0


@pytest.mark.parametrize("d", [32, 128])
def test_offset_data(ctx, d):
    X, Q = _blobs(2000, 100, d, seed=11, offset=1e3)
    for path in _paths(d, 10):
        out, _ = _ivf(ctx, X, Q, 10, 16, 4, path=path)
        _check_all(X, Q, 10, out)


def test_empty_list_fewer_than_k_and_nan_query(ctx):
    X, Q = _blobs(600, 40, 32, seed=5)
    C = np.concatenate([X[:6], np.full((1, 32), 1e4, np.float32)])   # list 6 holds no item
    Q[3, 7] = np.nan
    Q[4] = 1e4   # probes the empty list first
    for path in (2, 1):
        out, _ = _ivf(ctx, X, Q, 64, 7, 1, C=C, path=path)
        dist, idx, _, lists, probes = out
        assert not np.any(lists == 6)
        assert np.all(probes[3] == -1) and np.all(np.isinf(dist[3])) and np.all(idx[3] == ao.INT64_MAX)
        assert probes[4, 0] == 6 and np.all(np.isinf(dist[4])) and np.all(idx[4] == ao.INT64_MAX)
        _check_all(X, Q, 64, out)
        # a small list: fewer than k items, the rest filled with the first id and +inf
        small = np.bincount(lists, minlength=7)[:6].argmin()
        q = np.nonzero(probes[:, 0] == small)[0]
        if q.size and np.bincount(lists, minlength=7)[small] < 64:
            i = q[0]
            n = np.bincount(lists, minlength=7)[small]
            assert np.all(np.isfinite(dist[i, :n])) and np.all(np.isinf(dist[i, n:]))
            assert np.all(idx[i, n:] == idx[i, 0])


def test_sqeuclidean(ctx):
    X, Q = _blobs(1500, 60, 64, seed=9)
    (de, ie, *_), _ = _ivf(ctx, X, Q, 8, 16, 5, C=X[:16])
    out, _ = _ivf(ctx, X, Q, 8, 16, 5, C=X[:16], metric="sqeuclidean")
    np.testing.assert_array_equal(out[1], ie)
    np.testing.assert_allclose(out[0], de.astype(np.float64) ** 2, rtol=3e-7)
    _check_all(X, Q, 8, out, squared=True)


def test_non_finite_item_fails(ctx):
    X, Q = _blobs(300, 10, 16, seed=1)
    X[17, 3] = np.inf
    with pytest.raises(RuntimeError, match="non-finite"):
        ctx.ivf_search(torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda(), 5, 4, 2)


def test_bad_arguments_fail(ctx):
    X, Q = _blobs(300, 10, 16, seed=1)
    Xd, Qd = torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda()
    with pytest.raises(RuntimeError, match="training rows"):
        ctx.ivf_search(Xd, Qd, 5, 200, 2)   # 150 training rows at the default fraction
    with pytest.raises(RuntimeError, match="exceeds 256"):
        ctx.ivf_search(Xd, Qd, 5, 290, 280, centers=Xd[:290].contiguous())
    with pytest.raises(RuntimeError, match="k = 301"):
        ctx.ivf_search(Xd, Qd, 301, 4, 2)


def test_repeatable(ctx):
    X, Q = _blobs(5000, 300, 64, seed=2)
    a, _ = _ivf(ctx, X, Q, 10, 32, 4)
    b, _ = _ivf(ctx, X, Q, 10, 32, 4)
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u.view(np.uint8), v.view(np.uint8))


@pytest.mark.parametrize("path", [2, 1])
def test_steady_state_two_chunks(ctx, path):
    # 40 k queries x 20 probes at d = 128, k = 10: the gathered queries need two chunks of at most 256 MB; four CTAs run
    # thousands of units each
    X, Q = _blobs(100_000, 40_000, 128, seed=4)
    out, _ = _ivf(ctx, X, Q, 10, 256, 20, path=path, grid=4 if path == 2 else 0, n_iters=5)
    dist, idx, C, lists, probes = out
    sel = np.r_[0:150, 26_100:26_300, 39_850:40_000]
    assert ao.check_lists(X[:5000], C, lists[:5000]) == 0
    assert ao.check_probes(C, Q[sel], probes[sel]) == 0
    bad = ao.check_result(X, Q[sel], 10, lists, probes[sel], dist[sel], idx[sel])
    assert bad == {"n_outside_margin": 0, "n_fill": 0}, bad
