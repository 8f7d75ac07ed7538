"""CPU checks of KMeans tuning with ClusteringEvaluator: which (estimator, evaluator) pairs CrossValidator takes, the
features-column check of KMeansModel._transformEvaluate, _combine, which param grids fitMultiple fits from one ingest,
and the fp64 oracle per model (the reference of the GPU tests)."""
import numpy as np
import pytest

import silhouette_oracle as so


def _cv(est, ev):
    from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder

    return CrossValidator(estimator=est, estimatorParamMaps=ParamGridBuilder().addGrid(est.k, [2, 3]).build()
                          if hasattr(est, "k") else [{}], evaluator=ev)


def test_supported_pairs_for_kmeans():
    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import (BinaryClassificationEvaluator, ClusteringEvaluator,
                                                 MulticlassClassificationEvaluator, RegressionEvaluator)

    km = KMeans()
    for dist in ("squaredEuclidean", "cosine"):
        assert km._supportsTransformEvaluate(ClusteringEvaluator(distanceMeasure=dist))
        _cv(km, ClusteringEvaluator(distanceMeasure=dist))._check()
    for ev in (MulticlassClassificationEvaluator(), BinaryClassificationEvaluator(), RegressionEvaluator()):
        assert not km._supportsTransformEvaluate(ev)
        with pytest.raises(NotImplementedError, match="KMeans"):
            _cv(km, ev)._check()


def test_features_column_must_match():
    from spark_rapids_ml_b200.clustering import KMeansModel
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator
    from spark_rapids_ml_b200.sparkshim import get_session

    m = KMeansModel(cluster_centers_=[[0.0, 0.0], [1.0, 1.0]], n_cols=2, dtype="float32")
    m.setFeaturesCol("x")
    df = get_session().createDataFrame([([0.0, 0.0],), ([1.0, 1.0],)], ["x"])
    with pytest.raises(NotImplementedError, match="'features'.*'x'"):
        m._transformEvaluate(df, ClusteringEvaluator())
    m.setFeaturesCol(["a", "b"])
    with pytest.raises(NotImplementedError, match=r"\['a', 'b'\]"):
        m._transformEvaluate(df, ClusteringEvaluator(featuresCol="x"))


def test_combine_keeps_every_centre_set():
    from spark_rapids_ml_b200.clustering import KMeansModel

    a = KMeansModel(cluster_centers_=[[0.0, 1.0], [2.0, 3.0]], n_cols=2, dtype="float32")
    b = KMeansModel(cluster_centers_=[[0.0, 1.0], [2.0, 3.0], [4.0, 5.0]], n_cols=2, dtype="float32")
    a.setFeaturesCol("v")
    c = KMeansModel._combine([a, b])
    assert c._center_sets() == [a.cluster_centers_, b.cluster_centers_]
    assert a._center_sets() == [a.cluster_centers_]
    assert c.getFeaturesCol() == "v" and c.n_cols == 2


def test_fit_multiple_map_classification():
    from spark_rapids_ml_b200.clustering import KMeans, _kmeans_grid_shares_ingest
    from spark_rapids_ml_b200.tuning import ParamGridBuilder

    km = KMeans()
    shared = (ParamGridBuilder().addGrid(km.k, [2, 3]).addGrid(km.maxIter, [5, 9]).addGrid(km.tol, [1e-4])
              .addGrid(km.seed, [1, 2]).addGrid(km.initMode, ["random", "k-means||"]).build())
    assert _kmeans_grid_shares_ingest(shared)
    assert not _kmeans_grid_shares_ingest([])
    assert not _kmeans_grid_shares_ingest(ParamGridBuilder().addGrid(km.k, [2]).addGrid(km.featuresCol, ["x"]).build())
    assert not _kmeans_grid_shares_ingest(ParamGridBuilder().addGrid(km.predictionCol, ["p"]).build())


def test_oracle_per_model():
    """Each model's closed form equals the pairwise definition on a small frame, and beta is positive and small."""
    rng = np.random.default_rng(0)
    X = rng.normal(size=(60, 3)).astype(np.float32)
    for K in (2, 3, 5):
        ids = rng.integers(0, K, 60).astype(np.int64)
        ids[:K] = np.arange(K)
        Y = X.astype(np.float64)
        D = ((Y[:, None, :] - Y[None, :, :]) ** 2).sum(-1)
        s = []
        for i in range(60):
            own = ids == ids[i]
            na = own.sum()
            if na == 1:
                s.append(0.0)
                continue
            a = D[i, own].sum() / (na - 1)
            b = min(D[i, ids == c].mean() for c in set(ids.tolist()) if c != ids[i])
            s.append((b - a) / max(a, b))
        assert abs(so.closed_form(X, ids, "squaredEuclidean") - np.mean(s)) < 1e-9
        assert 0 < so.beta(X, ids, "squaredEuclidean") < 1e-3
