"""b2k_silhouette on one H100: both passes within the bound beta of the fp64 oracle (tests/silhouette_oracle.py) across
widths, cluster counts (several blocks of 128 means past K = 128), both distance measures, offset data, many tiles per
CTA with a ragged last tile; the passes within 2 beta of each other; bitwise repeatability; the cluster-id limit; every
error; and ClusteringEvaluator end to end on KMeansModel and DBSCANModel output against scikit-learn."""
import numpy as np
import pytest

import silhouette_oracle as so

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _data(n, d, K, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(K, d)) * 2
    lab = rng.integers(0, K, n)
    lab[:K] = np.arange(K)   # every cluster present
    X = (mu[lab] + rng.normal(size=(n, d)) + offset).astype(np.float32)
    ids = (3 * lab - 1).astype(np.int64)   # non-contiguous, -1 included
    return X, ids


def _run(ctx, X, ids, metric, path=0, grid_limit=0):
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid_limit)
    try:
        v = ctx.silhouette(torch.from_numpy(X).cuda(), torch.from_numpy(ids).cuda(), metric)
        return v, ctx.stats()["last_path"]
    finally:
        ctx.set_option("kernel_path", 0)
        ctx.set_option("grid_limit", 0)


def _check(ctx, X, ids, metric, wg_expected):
    ref, beta = so.closed_form(X, ids, metric), so.beta(X, ids, metric)
    v_auto, p_auto = _run(ctx, X, ids, metric)
    v_gen, p_gen = _run(ctx, X, ids, metric, path=1)
    assert p_auto == (2 if wg_expected else 1) and p_gen == 1
    assert abs(v_auto - ref) <= beta, (v_auto, ref, beta)
    assert abs(v_gen - ref) <= beta, (v_gen, ref, beta)
    assert abs(v_auto - v_gen) <= 2 * beta


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("d", [1, 3, 4, 100, 128, 132, 256])
def test_widths(ctx, d, metric):
    X, ids = _data(2000, d, 64, seed=d)
    _check(ctx, X, ids, metric, wg_expected=d % 4 == 0 and 4 <= d <= 128)


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("K", [2, 3, 64, 129, 1000])
def test_cluster_counts(ctx, K, metric):
    X, ids = _data(3000, 128, K, seed=K)
    _check(ctx, X, ids, metric, wg_expected=True)


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("d", [32, 128, 130])
def test_offset_data(ctx, d, metric):
    X, ids = _data(2500, d, 10, seed=7, offset=1e3)
    _check(ctx, X, ids, metric, wg_expected=d != 130)


@pytest.mark.parametrize("path", [0, 1])
@pytest.mark.parametrize("grid_limit", [1, 3, 0])
def test_many_tiles_per_cta_ragged(ctx, grid_limit, path):
    X, ids = _data(128 * 40 + 77, 64, 20, seed=11)
    ref, beta = so.closed_form(X, ids, "squaredEuclidean"), so.beta(X, ids, "squaredEuclidean")
    v, p = _run(ctx, X, ids, "squaredEuclidean", path=path, grid_limit=grid_limit)
    assert p == (2 if path == 0 else 1)
    assert abs(v - ref) <= beta, (v, ref, beta)


@pytest.mark.parametrize("path", [0, 1])
def test_two_calls_same_bits(ctx, path):
    X, ids = _data(20000, 96, 37, seed=5)
    a, _ = _run(ctx, X, ids, "squaredEuclidean", path=path)
    b, _ = _run(ctx, X, ids, "squaredEuclidean", path=path)
    assert np.float64(a).tobytes() == np.float64(b).tobytes()


def _pairs(K):
    """K clusters of two equal rows each at distinct points: every s_i is 1 (a = 0 < b)."""
    c = np.arange(K)
    P = np.stack([c % 256, c // 256, (c * 7) % 13, np.zeros(K)], axis=1).astype(np.float32)
    return np.repeat(P, 2, axis=0), np.repeat(c.astype(np.int64) * 5 - 3, 2)


def test_id_limit(ctx):
    from spark_rapids_ml_b200 import _native

    X, ids = _pairs(65536)
    v, _ = _run(ctx, X, ids, "squaredEuclidean", path=1)   # fp64: a is 0 up to the rounding of Psi
    assert abs(v - 1.0) < 1e-9, v
    v, _ = _run(ctx, X, ids, "squaredEuclidean")   # 3xTF32: a is within the bound of 0, b is 1
    assert abs(v - 1.0) < 1e-2, v
    X, ids = _pairs(65537)
    with pytest.raises(_native.B2KError) as e:
        _run(ctx, X, ids, "squaredEuclidean")
    assert e.value.code == 4 and "65536 distinct cluster ids" in str(e.value)


def _err(ctx, X, ids, metric="squaredEuclidean", path=0):
    from spark_rapids_ml_b200 import _native

    with pytest.raises(_native.B2KError) as e:
        _run(ctx, X, ids, metric, path=path)
    return e.value


def test_errors(ctx):
    X, ids = _data(500, 8, 4, seed=1)
    for bad in (np.nan, np.inf):
        Xb = X.copy()
        Xb[17, 3] = bad
        assert "NaN or infinity" in str(_err(ctx, Xb, ids))
    Xz = X.copy()
    Xz[5] = 0.0
    assert "zero row" in str(_err(ctx, Xz, ids, "cosine"))
    _run(ctx, Xz, ids, "squaredEuclidean")   # a zero row is fine under squaredEuclidean
    assert "Number of clusters must be greater than one." in str(_err(ctx, X, np.zeros_like(ids)))
    assert "no rows" in str(_err(ctx, X[:0], ids[:0]))
    e = _err(ctx, _data(300, 3, 4, seed=2)[0], _data(300, 3, 4, seed=2)[1], path=2)
    assert e.code == 4 and "kernel_path=2" in str(e)
    from spark_rapids_ml_b200 import _native

    ctx.set_option("kernel_path", 2)
    try:   # a view one float in: X is not 16-byte aligned
        big = torch.from_numpy(np.ascontiguousarray(np.concatenate([np.zeros(1, np.float32), X.reshape(-1)]))).cuda()
        with pytest.raises(_native.B2KError) as ee:
            ctx.silhouette(big[1:].view(500, 8), torch.from_numpy(ids).cuda())
        assert ee.value.code == 4
    finally:
        ctx.set_option("kernel_path", 0)
    with pytest.raises(ValueError):
        ctx.silhouette(torch.from_numpy(X).cuda(), torch.from_numpy(ids).cuda(), "euclidean")


def _frame(X, cols=None):
    from spark_rapids_ml_b200.sparkshim import get_session

    s = get_session()
    if cols is None:
        return s.createDataFrame([(list(map(float, r)),) for r in X], ["features"])
    return s.createDataFrame([tuple(map(float, r)) for r in X], cols)


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("metric,sk", [("squaredEuclidean", "sqeuclidean"), ("cosine", "cosine")])
def test_evaluator_on_kmeans_output(multi, metric, sk):
    from sklearn.metrics import silhouette_score

    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    X, _ = _data(600, 6, 4, seed=21)
    cols = [f"f{i}" for i in range(6)] if multi else None
    df = _frame(X, cols)
    feats = cols if multi else "features"
    out = KMeans(k=4, seed=1, featuresCol=feats).fit(df).transform(df)
    labels = np.asarray(out.toPandas()["prediction"], dtype=np.int64)
    v = ClusteringEvaluator(featuresCol=feats, distanceMeasure=metric).evaluate(out)
    ref = silhouette_score(X.astype(np.float64), labels, metric=sk)
    assert abs(v - ref) <= so.beta(X, labels, metric), (v, ref)


def test_evaluator_on_dbscan_output_with_noise():
    from sklearn.metrics import silhouette_score

    from spark_rapids_ml_b200.clustering import DBSCAN
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    rng = np.random.default_rng(4)
    X = np.concatenate([rng.normal(size=(200, 3)) * 0.3, rng.normal(size=(200, 3)) * 0.3 + 4,
                        rng.uniform(-8, 12, size=(20, 3))]).astype(np.float32)
    df = _frame(X)
    out = DBSCAN(eps=0.6, min_samples=5).fit(df).transform(df)
    labels = np.asarray(out.toPandas()["prediction"], dtype=np.int64)
    assert (labels == -1).any() and len(set(labels)) >= 3
    v = ClusteringEvaluator().evaluate(out)
    ref = silhouette_score(X.astype(np.float64), labels, metric="sqeuclidean")
    assert abs(v - ref) <= so.beta(X, labels), (v, ref)
