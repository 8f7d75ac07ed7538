"""Metrics, evaluators, folds and CrossValidator params without a GPU."""
import re

import numpy as np
import pandas as pd
import pytest
from sklearn import metrics as skm

from spark_rapids_ml_b200 import metrics
from spark_rapids_ml_b200.sparkshim import LocalSession
from spark_rapids_ml_b200.sparkshim.evaluation import MulticlassClassificationEvaluator, RegressionEvaluator
from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder, fold_ids, k_fold

import tuning_oracle as oracle


def _cls_data(n=500, C=4, seed=0):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, C, n).astype(np.float64)
    p = np.where(rng.random(n) < 0.6, y, rng.integers(0, C + 1, n)).astype(np.float64)
    probs = rng.random((n, C))
    probs[np.arange(n), (y % C).astype(int)] += 1.0
    probs /= probs.sum(1, keepdims=True)
    probs[:5, :] = 0.0   # p_y = 0: clipped at eps
    return y, p, probs


@pytest.mark.parametrize("metric", metrics.MULTICLASS_METRICS)
@pytest.mark.parametrize("label,beta,eps", [(0.0, 1.0, 1e-15), (2.0, 0.5, 1e-6)])
def test_multiclass_metrics_match_oracle(metric, label, beta, eps):
    y, p, probs = _cls_data()
    acc = metrics.class_accumulators(y, p, probs, eps)
    got = metrics.multiclass_metric(acc, metric, label, beta)
    assert got == pytest.approx(oracle.multiclass(y, p, probs, metric, label, beta, eps), rel=1e-12)
    ses = LocalSession()
    df = ses.createDataFrame(pd.DataFrame({"label": y, "prediction": p, "probability": list(probs)}), num_partitions=2)
    ev = MulticlassClassificationEvaluator(metricName=metric, metricLabel=label, beta=beta, eps=eps)
    assert ev.evaluate(df) == got


def test_multiclass_against_sklearn():
    y, p, probs = _cls_data()
    acc = metrics.class_accumulators(y, p, probs, 1e-15)
    m = lambda name: metrics.multiclass_metric(acc, name)   # noqa: E731
    labels = sorted(set(y))
    assert m("accuracy") == pytest.approx(skm.accuracy_score(y, p), rel=1e-12)
    assert m("weightedPrecision") == pytest.approx(skm.precision_score(y, p, labels=labels, average="weighted",
                                                                       zero_division=0), rel=1e-12)
    assert m("weightedRecall") == pytest.approx(skm.recall_score(y, p, labels=labels, average="weighted"), rel=1e-12)
    assert m("f1") == pytest.approx(skm.f1_score(y, p, labels=labels, average="weighted", zero_division=0), rel=1e-12)
    ll = -np.log(np.maximum(probs[np.arange(y.size), y.astype(int)], 1e-15)).mean()
    assert m("logLoss") == pytest.approx(ll, rel=1e-12)


def test_multiclass_known_answers():
    y = np.array([0, 0, 1, 1, 2, 2], dtype=float)
    p = np.array([0, 1, 1, 1, 0, 2], dtype=float)
    acc = metrics.class_accumulators(y, p, None, 1e-15)
    assert metrics.multiclass_metric(acc, "hammingLoss") == pytest.approx(2 / 6)
    assert metrics.multiclass_metric(acc, "precisionByLabel", 1.0) == pytest.approx(2 / 3)
    assert metrics.multiclass_metric(acc, "recallByLabel", 0.0) == pytest.approx(1 / 2)
    assert metrics.multiclass_metric(acc, "falsePositiveRateByLabel", 0.0) == pytest.approx(1 / 4)
    # weighted FPR: label 0: 1/4, label 1: 1/4, label 2: 0/4, each weighted 1/3
    assert metrics.multiclass_metric(acc, "weightedFalsePositiveRate") == pytest.approx(1 / 6)
    with pytest.raises(ValueError):
        metrics.multiclass_metric(acc, "recallByLabel", 7.0)


@pytest.mark.parametrize("metric", metrics.REGRESSION_METRICS)
@pytest.mark.parametrize("through_origin", [False, True])
def test_regression_metrics(metric, through_origin):
    rng = np.random.default_rng(1)
    y = rng.normal(3, 2, 400)
    p = y + rng.normal(0, 0.5, 400)
    acc = metrics.reg_accumulators(y, p)
    got = metrics.regression_metric(acc, metric, through_origin)
    assert got == pytest.approx(oracle.regression(y, p, metric, through_origin), rel=1e-12)
    if metric in ("mse", "mae") or (metric == "r2" and not through_origin):
        sk = {"mse": skm.mean_squared_error, "mae": skm.mean_absolute_error, "r2": skm.r2_score}[metric]
        assert got == pytest.approx(sk(y, p), rel=1e-12)
    df = LocalSession().createDataFrame(pd.DataFrame({"label": y, "prediction": p}), num_partitions=3)
    assert RegressionEvaluator(metricName=metric, throughOrigin=through_origin).evaluate(df) == got


def test_regression_var_known_answer():
    acc = metrics.reg_accumulators(np.array([1.0, 2.0, 3.0]), np.array([1.0, 1.0, 4.0]))
    # sum p^2 / n + ybar^2 - 2 ybar pbar = 18/3 + 4 - 2*2*2 = 2
    assert metrics.regression_metric(acc, "var") == pytest.approx(2.0)


def test_merge_equals_unsplit():
    y, p, probs = _cls_data(n=301)
    whole = metrics.class_accumulators(y, p, probs, 1e-15)
    parts = [metrics.class_accumulators(y[a:b], p[a:b], probs[a:b], 1e-15) for a, b in ((0, 100), (100, 101), (101, 301))]
    merged = metrics.merge_all(parts, True)
    for k in ("label_count", "tp", "fp"):
        np.testing.assert_array_equal(merged[k], whole[k])
    assert merged["loss"] == pytest.approx(whole["loss"], rel=1e-13)
    yr = np.random.default_rng(2).normal(size=301)
    pr = yr * 0.5
    wr = metrics.reg_accumulators(yr, pr)
    mr = metrics.merge_all([metrics.reg_accumulators(yr[a:b], pr[a:b]) for a, b in ((0, 7), (7, 301))], False)
    np.testing.assert_allclose(mr["reg"], wr["reg"], rtol=1e-12, atol=1e-12)


def test_chan_merge_keeps_precision_at_a_large_offset():
    rng = np.random.default_rng(3)
    y = 1e6 + rng.normal(size=10000)
    p = y - rng.normal(size=10000)
    parts = [metrics.reg_accumulators(y[i:i + 256], p[i:i + 256]) for i in range(0, y.size, 256)]
    m = metrics.merge_all(parts, False)
    two_pass = float(np.sum((y - y.mean()) ** 2))
    assert m["reg"][0][2] == pytest.approx(two_pass, rel=1e-12)


def _frame(n=200, parts=2, fold=None):
    data = {"features": list(np.random.default_rng(0).random((n, 3)).astype(np.float32)), "label": np.zeros(n)}
    if fold is not None:
        data["fold"] = fold
    return LocalSession().createDataFrame(pd.DataFrame(data), num_partitions=parts)


def test_folds_disjoint_cover_and_reproducible():
    df = _frame()
    a, b = fold_ids(df, 3, 7), fold_ids(df, 3, 7)
    np.testing.assert_array_equal(a, b)
    assert set(a.tolist()) == {0, 1, 2}
    u = np.random.default_rng(7).random(200)
    np.testing.assert_array_equal(a, np.floor(3 * u).astype(int))
    folds = k_fold(df, 3, 7, None, 2)
    assert sum(v.count() for _, v in folds) == 200
    for (t, v) in folds:
        assert t.count() + v.count() == 200 and t.getNumPartitions() == 2


def test_fold_col():
    f = np.arange(90) % 3
    df = _frame(90, fold=f.astype(np.int32))
    np.testing.assert_array_equal(fold_ids(df, 3, 0, "fold"), f)
    assert "fold" not in k_fold(df, 3, 0, "fold", 1)[0][0].columns
    with pytest.raises(ValueError, match=re.escape("range [0, 2)")):
        fold_ids(df, 2, 0, "fold")


def test_param_grid_order_first_grid_slowest():
    from spark_rapids_ml_b200.classification import LogisticRegression

    lr = LogisticRegression()
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.1, 0.2]).addGrid(lr.elasticNetParam, [0.0, 0.5, 1.0]).build()
    assert [(g[lr.regParam], g[lr.elasticNetParam]) for g in grid] == [
        (0.1, 0.0), (0.1, 0.5), (0.1, 1.0), (0.2, 0.0), (0.2, 0.5), (0.2, 1.0)]


def test_cv_param_validation():
    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.clustering import KMeans

    lr = LogisticRegression()
    ev = MulticlassClassificationEvaluator()
    assert CrossValidator().getNumFolds() == 3
    with pytest.raises(ValueError, match="numFolds"):
        CrossValidator(estimator=lr, estimatorParamMaps=[{}], evaluator=ev, numFolds=1).fit(_frame())
    with pytest.raises(NotImplementedError, match="KMeans"):
        CrossValidator(estimator=KMeans(), estimatorParamMaps=[{}], evaluator=ev).fit(_frame())
    with pytest.raises(NotImplementedError, match="RegressionEvaluator"):
        CrossValidator(estimator=lr, estimatorParamMaps=[{}], evaluator=RegressionEvaluator()).fit(_frame())
    assert ev.isLargerBetter() and not MulticlassClassificationEvaluator(metricName="logLoss").isLargerBetter()
    assert not RegressionEvaluator().isLargerBetter() and RegressionEvaluator(metricName="r2").isLargerBetter()


def test_weight_col_raises():
    df = LocalSession().createDataFrame(pd.DataFrame({"label": np.zeros(3), "prediction": np.zeros(3)}))
    with pytest.raises(NotImplementedError):
        RegressionEvaluator(weightCol="w").evaluate(df)
