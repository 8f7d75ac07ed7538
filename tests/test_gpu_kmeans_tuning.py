"""CrossValidator(KMeans, ClusteringEvaluator) on one H100: fitMultiple's models equal separate fits bit for bit;
_transformEvaluate equals, per model, ClusteringEvaluator().evaluate(model.transform(valid)) bit for bit (both distance
measures, array and list-of-columns features); avgMetrics / stdMetrics equal the hand loop over k_fold's folds; the best
model has the expected k on well-separated blobs; the metric agrees with scikit-learn within beta."""
import numpy as np
import pytest

import silhouette_oracle as so

pytestmark = pytest.mark.gpu

pytest.importorskip("torch")


def _blobs(n, d, k, seed, spread=12.0):
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(k, d)) * spread
    lab = rng.integers(0, k, n)
    return (mu[lab] + rng.normal(size=(n, d))).astype(np.float32), lab


def _frame(X, cols=None):
    from spark_rapids_ml_b200.sparkshim import get_session

    s = get_session()
    if cols is None:
        return s.createDataFrame([(list(map(float, r)),) for r in X], ["features"])
    return s.createDataFrame([tuple(map(float, r)) for r in X], cols)


def _grid(km, ks):
    from spark_rapids_ml_b200.tuning import ParamGridBuilder

    return ParamGridBuilder().addGrid(km.k, ks).addGrid(km.maxIter, [7]).build()


def test_fit_multiple_equals_separate_fits():
    from spark_rapids_ml_b200.clustering import KMeans

    X, _ = _blobs(1200, 8, 5, seed=1)
    df = _frame(X)
    km = KMeans(seed=3)
    maps = _grid(km, [2, 3, 5, 9])
    got = sorted(km.fitMultiple(df, maps), key=lambda t: t[0])
    for (i, m), pm in zip(got, maps):
        ref = km.copy(pm).fit(df)
        assert np.asarray(m.cluster_centers_).tobytes() == np.asarray(ref.cluster_centers_).tobytes()
        assert m.getK() == ref.getK() and m.cuml_params["n_clusters"] == ref.cuml_params["n_clusters"]


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
def test_transform_evaluate_equals_evaluate_of_transform(multi, metric):
    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    X, _ = _blobs(1500, 6, 4, seed=2, spread=3.0)
    cols = [f"f{i}" for i in range(6)] if multi else None
    feats = cols if multi else "features"
    df = _frame(X, cols)
    km = KMeans(seed=5, featuresCol=feats)
    models = [m for _, m in sorted(km.fitMultiple(df, _grid(km, [2, 3, 4, 7, 12])), key=lambda t: t[0])]
    ev = ClusteringEvaluator(featuresCol=feats, distanceMeasure=metric)
    got = models[0]._combine(models)._transformEvaluate(df, ev)
    ref = [ev.evaluate(m.transform(df)) for m in models]
    assert [np.float64(v).tobytes() for v in got] == [np.float64(v).tobytes() for v in ref], (got, ref)


def test_cross_validator_equals_hand_loop_and_picks_k():
    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator
    from spark_rapids_ml_b200.tuning import CrossValidator, k_fold

    X, _ = _blobs(2000, 5, 4, seed=4)
    df = _frame(X)
    km = KMeans(seed=7)
    maps = _grid(km, [2, 3, 4, 6, 8])
    ev = ClusteringEvaluator()
    cv = CrossValidator(estimator=km, estimatorParamMaps=maps, evaluator=ev, numFolds=3, seed=11)
    model = cv.fit(df)
    parts = int(km.num_workers)
    hand = []
    for train, valid in k_fold(df, 3, 11, None, parts):
        hand.append([ev.evaluate(km.copy(pm).fit(train).transform(valid)) for pm in maps])
    assert model.avgMetrics == [float(v) for v in np.mean(hand, axis=0)]
    assert model.stdMetrics == [float(v) for v in np.std(hand, axis=0)]
    assert model.bestModel.getK() == 4
    assert len(model.bestModel.clusterCenters()) == 4


@pytest.mark.parametrize("metric,sk", [("squaredEuclidean", "sqeuclidean"), ("cosine", "cosine")])
def test_metric_agrees_with_sklearn(metric, sk):
    from sklearn.metrics import silhouette_score

    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    X, _ = _blobs(900, 4, 3, seed=9, spread=4.0)
    df = _frame(X)
    km = KMeans(seed=1)
    models = [m for _, m in sorted(km.fitMultiple(df, _grid(km, [2, 3, 5])), key=lambda t: t[0])]
    got = models[0]._combine(models)._transformEvaluate(df, ClusteringEvaluator(distanceMeasure=metric))
    for v, m in zip(got, models):
        labels = np.asarray(m.transform(df).toPandas()["prediction"], dtype=np.int64)
        ref = silhouette_score(X.astype(np.float64), labels, metric=sk)
        assert abs(v - ref) <= so.beta(X, labels, metric), (v, ref)
