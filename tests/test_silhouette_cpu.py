"""The silhouette oracle against the definition and scikit-learn, at its edges (singletons, duplicate rows, a == b,
two clusters, ids -1 and non-contiguous, offset data where Spark's expanded form loses digits), and ClusteringEvaluator's
params, defaults, validation, copy(), weightCol and pyspark-frame errors — none of which needs a GPU."""
import numpy as np
import pytest
from sklearn.metrics import silhouette_score

import silhouette_oracle as so
from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

SK = {"squaredEuclidean": "sqeuclidean", "cosine": "cosine"}


def _blobs(n, d, K, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, K, n)
    lab[:K] = np.arange(K)
    return (rng.normal(size=(K, d))[lab] * 3 + rng.normal(size=(n, d)) + offset).astype(np.float32), lab


CASES = {
    "blobs": _blobs(240, 5, 4, 0),
    "two_clusters": _blobs(100, 3, 2, 1),
    "singletons": (np.concatenate([_blobs(60, 4, 3, 2)[0], [[9, 9, 9, 9], [-9, 3, 1, 2]]]).astype(np.float32),
                   np.concatenate([_blobs(60, 4, 3, 2)[1], [7, 8]])),
    "duplicates": (np.repeat(_blobs(40, 3, 3, 3)[0], 3, axis=0), np.repeat(_blobs(40, 3, 3, 3)[1], 3)),
    "noncontiguous_ids": (_blobs(150, 6, 5, 4)[0], np.array([-1, 7, 1000, 3, 42])[_blobs(150, 6, 5, 4)[1]]),
}


@pytest.mark.parametrize("metric", ["squaredEuclidean", "cosine"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_closed_form_equals_definition_and_sklearn(name, metric):
    X, ids = CASES[name]
    cf, bf = so.closed_form(X, ids, metric), so.brute_force(X, ids, metric)
    assert abs(cf - bf) <= 1e-12
    assert abs(bf - silhouette_score(X.astype(np.float64), ids, metric=SK[metric])) <= 1e-12


def test_a_equals_b_gives_zero():
    # 1-D: A = {0, 2}, B = {-2, 2}.  Row 0: a = 4 = b, so s = 0; the others give 0.5, -0.375 and -0.875
    X = np.array([[0], [2], [-2], [2]], np.float32)
    ids = np.array([0, 0, 1, 1])
    assert so.brute_force(X, ids) == -0.1875
    assert abs(so.closed_form(X, ids) + 0.1875) <= 1e-12
    assert abs(silhouette_score(X.astype(np.float64), ids, metric="sqeuclidean") + 0.1875) <= 1e-12


def test_offset_data_spark_form_loses_digits():
    X, ids = _blobs(300, 8, 3, 5, offset=1e6)
    bf = so.brute_force(X, ids)
    assert abs(so.closed_form(X, ids) - bf) <= 1e-12
    assert abs(so.spark_expanded(X, ids) - bf) > 1e-9


def test_beta_bounds_the_half_widths():
    X, ids = CASES["blobs"]
    b = so.beta(X, ids)
    assert 0 < b < 1e-3
    assert so.beta(X, np.zeros_like(ids) + np.arange(len(ids))) < 1e-12   # all singletons: s = 0 exactly


def test_fewer_than_two_clusters():
    X, _ = CASES["blobs"]
    with pytest.raises(ValueError, match="Number of clusters must be greater than one."):
        so.closed_form(X, np.zeros(len(X), np.int64))


def test_params_and_defaults():
    e = ClusteringEvaluator()
    assert (e.getFeaturesCol(), e.getPredictionCol(), e.getMetricName(), e.getDistanceMeasure()) == \
        ("features", "prediction", "silhouette", "squaredEuclidean")
    assert e.isLargerBetter()
    e2 = ClusteringEvaluator(featuresCol=["a", "b"], predictionCol="p", distanceMeasure="cosine")
    assert e2.getFeaturesCol() == ["a", "b"] and e2.getPredictionCol() == "p" and e2.getDistanceMeasure() == "cosine"
    e.setDistanceMeasure("cosine").setPredictionCol("q").setFeaturesCol("v")
    assert (e.getDistanceMeasure(), e.getPredictionCol(), e.getFeaturesCol()) == ("cosine", "q", "v")


def test_copy():
    e = ClusteringEvaluator()
    c = e.copy({e.distanceMeasure: "cosine"})
    assert isinstance(c, ClusteringEvaluator)
    assert c.getDistanceMeasure() == "cosine" and e.getDistanceMeasure() == "squaredEuclidean"


def test_validation_messages():
    with pytest.raises(ValueError, match=r"parameter metricName given invalid value foo\."):
        ClusteringEvaluator(metricName="foo")
    with pytest.raises(ValueError, match=r"parameter distanceMeasure given invalid value euclidean\."):
        ClusteringEvaluator().setDistanceMeasure("euclidean")


def _frame(pred):
    from spark_rapids_ml_b200.sparkshim import get_session

    return get_session().createDataFrame([([1.0, 2.0], p) for p in pred], ["features", "prediction"])


@pytest.mark.parametrize("pred", [[0.0, 0.5], [0.0, float("nan")], [0.0, 1e19]])
def test_prediction_must_hold_integers(pred):
    with pytest.raises(ValueError, match="predictionCol 'prediction'"):
        ClusteringEvaluator().evaluate(_frame(pred))


def test_weight_col_and_empty_frame():
    with pytest.raises(NotImplementedError, match="weightCol"):
        ClusteringEvaluator(weightCol="w").evaluate(_frame([0, 1]))
    from spark_rapids_ml_b200.sparkshim import get_session

    empty = get_session().createDataFrame([([1.0, 2.0], 0)], ["features", "prediction"]).repartition(1)
    empty = empty._derive([[b.slice(0, 0) for b in p] for p in empty._parts])
    with pytest.raises(ValueError, match="no rows"):
        ClusteringEvaluator().evaluate(empty)


def test_pyspark_frame_is_refused(monkeypatch):
    import spark_rapids_ml_b200.evaluation as ev
    from spark_rapids_ml_b200 import spark_binding

    monkeypatch.setattr(ev, "HAVE_PYSPARK", True)
    monkeypatch.setattr(spark_binding, "is_spark_dataframe", lambda obj: True)
    with pytest.raises(NotImplementedError, match=r"evaluate\(\) of a pyspark DataFrame is not supported"):
        ClusteringEvaluator().evaluate(object())
