"""b2k_silhouette_multi on one H100: every model's value has exactly the bits of its own b2k_silhouette call, across
widths (both passes), both distance measures, model counts past one chunk of B2K_SILHOUETTE_MULTI_CHUNK with cluster
counts whose segments straddle blocks, offset data, grid_limit and forced kernel paths; each value within beta of the
fp64 oracle; one silhouette pass per (shift group, chunk); errors name the first failing model; repeatable bits."""
import math

import numpy as np
import pytest

import silhouette_oracle as so

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

MC = 16   # B2K_SILHOUETTE_MULTI_CHUNK (include/b2kmeans.h)
KS = [2, 3, 64, 129, 1000]


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _models(n, d, Ks, seed, offset=0.0):
    """Rows around 8 blob centres and one labelling per K: model m's ids are a hash of the row's blob and index, so the
    models' clusters differ and every cluster is present."""
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(8, d)) * 2
    blob = rng.integers(0, 8, n)
    X = (mu[blob] + rng.normal(size=(n, d)) + offset).astype(np.float32)
    ids = []
    for m, K in enumerate(Ks):
        lab = (blob * 131 + np.arange(n) * (m + 3)) % K
        lab[:K] = np.arange(K)
        ids.append((5 * lab - 2 + m).astype(np.int64))
    return X, ids


def _set(ctx, path, grid_limit):
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid_limit)


def _both(ctx, X, ids, metric, path=0, grid_limit=0):
    """(multi values, its stats, per-model single values) under the same options."""
    Xd = torch.from_numpy(X).cuda()
    idd = [torch.from_numpy(i).cuda() for i in ids]
    _set(ctx, path, grid_limit)
    try:
        before = ctx.stats()
        multi = ctx.silhouette_multi(Xd, idd, metric)
        after = ctx.stats()
        single = [ctx.silhouette(Xd, i, metric) for i in idd]
    finally:
        _set(ctx, 0, 0)
    launches = {k: after[k] - before[k] for k in ("fused_tc_launches", "generic_launches")}
    return multi, after["last_path"], launches, single


def _bits(v):
    return [np.float64(x).tobytes() for x in v]


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("d", [1, 3, 4, 100, 128, 132, 256])
def test_bits_equal_single_calls_across_widths(ctx, d, metric):
    X, ids = _models(1500, d, [2, 64, 3, 129], seed=d)
    multi, path, launches, single = _both(ctx, X, ids, metric)
    assert _bits(multi) == _bits(single), (multi, single)
    wg = d % 4 == 0 and 4 <= d <= 128
    assert path == (2 if wg else 1)
    assert launches == ({"fused_tc_launches": 1, "generic_launches": 0} if wg else
                        {"fused_tc_launches": 0, "generic_launches": 1}), launches


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("M", [1, 2, 12, 33])
@pytest.mark.parametrize("path", [0, 1])
def test_bits_and_launches_across_model_counts(ctx, M, path, metric):
    Ks = [KS[(3 * m + 1) % len(KS)] for m in range(M)]
    X, ids = _models(2000 + 37 * M, 64, Ks, seed=M)
    multi, got_path, launches, single = _both(ctx, X, ids, metric, path=path)
    assert _bits(multi) == _bits(single)
    assert got_path == (2 if path == 0 else 1)
    # one shift group (the ids differ, the rows and so their mean do not, unless a model's cluster-order sums round m
    # differently): at least ceil(M / MC) passes, at most one per model; a loop over b2k_silhouette would make M
    key = "fused_tc_launches" if path == 0 else "generic_launches"
    chunks = math.ceil(M / MC)
    assert chunks <= launches[key] <= M
    if M > 1:
        assert launches[key] < M, launches


def test_launches_equal_groups_times_chunks(ctx):
    """Rows on a lattice of small integers: every model's fp64 sums are exact, so all shifts agree (one group), and 33
    models take exactly ceil(33 / MC) passes."""
    rng = np.random.default_rng(3)
    X = rng.integers(-4, 5, size=(3000, 32)).astype(np.float32)
    ids = [rng.integers(0, K, 3000).astype(np.int64) for K in [KS[m % len(KS)] for m in range(33)]]
    for i, K in zip(ids, [KS[m % len(KS)] for m in range(33)]):
        i[:K] = np.arange(K)
    for path, key in ((0, "fused_tc_launches"), (1, "generic_launches")):
        multi, _, launches, single = _both(ctx, X, ids, "squaredEuclidean", path=path)
        assert _bits(multi) == _bits(single)
        assert launches[key] == math.ceil(33 / MC), launches


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("d", [32, 130])
def test_offset_data(ctx, d, metric):
    X, ids = _models(1800, d, [3, 10, 64], seed=7, offset=1e3)
    multi, _, _, single = _both(ctx, X, ids, metric)
    assert _bits(multi) == _bits(single)
    for v, i in zip(multi, ids):
        assert abs(v - so.closed_form(X, i, metric)) <= so.beta(X, i, metric)


@pytest.mark.parametrize("path", [0, 1, 2])
@pytest.mark.parametrize("grid_limit", [1, 3, 0])
def test_grid_limit_and_paths(ctx, grid_limit, path):
    X, ids = _models(128 * 30 + 77, 64, [2, 129, 20, 64, 3], seed=11)
    multi, got, _, single = _both(ctx, X, ids, "squaredEuclidean", path=path, grid_limit=grid_limit)
    assert _bits(multi) == _bits(single)
    assert got == (1 if path == 1 else 2)


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
def test_within_beta_of_oracle(ctx, metric):
    X, ids = _models(2500, 128, [2, 3, 64, 129, 1000], seed=5)
    multi, _, _, _ = _both(ctx, X, ids, metric)
    for v, i in zip(multi, ids):
        ref, beta = so.closed_form(X, i, metric), so.beta(X, i, metric)
        assert abs(v - ref) <= beta, (v, ref, beta)


@pytest.mark.parametrize("path", [0, 1])
def test_two_calls_same_bits(ctx, path):
    X, ids = _models(20000, 96, [37, 5, 200], seed=5)
    a, _, _, _ = _both(ctx, X, ids, "squaredEuclidean", path=path)
    b, _, _, _ = _both(ctx, X, ids, "squaredEuclidean", path=path)
    assert _bits(a) == _bits(b)


def _err(ctx, X, ids, metric="squaredEuclidean"):
    from spark_rapids_ml_b200 import _native

    with pytest.raises(_native.B2KError) as e:
        ctx.silhouette_multi(torch.from_numpy(X).cuda(), [torch.from_numpy(i).cuda() for i in ids], metric)
    return e.value


def test_errors_name_the_first_failing_model(ctx):
    from spark_rapids_ml_b200 import _native

    X, ids = _models(600, 8, [4, 5, 6, 7], seed=1)
    bad = list(ids)
    bad[3] = np.zeros_like(ids[3])
    bad[2] = np.full_like(ids[2], 9)
    e = _err(ctx, X, bad)
    assert "model 2: Number of clusters must be greater than one." in str(e), str(e)
    c = np.arange(65537)
    P = np.stack([c % 256, c // 256, (c * 7) % 13, np.zeros(65537)], axis=1).astype(np.float32)
    many = [np.zeros(65537, np.int64), c.astype(np.int64)]
    many[0][1] = 1
    e = _err(ctx, P, many)
    assert e.code == 4 and "model 1: " in str(e) and "65536 distinct cluster ids" in str(e), str(e)
    Xz = X.copy()
    Xz[5] = 0.0
    e = _err(ctx, Xz, ids, "cosine")
    assert "model 0: " in str(e) and "zero row" in str(e), str(e)
    with pytest.raises((ValueError, _native.B2KError)):
        ctx.silhouette_multi(torch.from_numpy(X).cuda(), [], "squaredEuclidean")
