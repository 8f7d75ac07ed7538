"""BinaryClassificationEvaluator without a GPU: params, the fp64 oracle on hand-computed curves and against
scikit-learn, the host metric and the local evaluator against the oracle."""
import math

import numpy as np
import pandas as pd
import pytest
from sklearn import metrics as skm

from spark_rapids_ml_b200 import metrics
from spark_rapids_ml_b200.core import _eval_metric_info, _supports_transform_evaluate
from spark_rapids_ml_b200.sparkshim import LocalSession
from spark_rapids_ml_b200.sparkshim.evaluation import BinaryClassificationEvaluator

import binary_oracle as oracle

NAMES = ("areaUnderROC", "areaUnderPR")


def test_params_and_defaults():
    ev = BinaryClassificationEvaluator()
    assert (ev.getMetricName(), ev.getRawPredictionCol(), ev.getLabelCol(), ev.getNumBins()) == \
        ("areaUnderROC", "rawPrediction", "label", 1000)
    assert ev.isLargerBetter() and ev.setMetricName("areaUnderPR").isLargerBetter()
    ev = BinaryClassificationEvaluator(rawPredictionCol="r", labelCol="y", metricName="areaUnderPR", numBins=0)
    assert (ev.getMetricName(), ev.getRawPredictionCol(), ev.getLabelCol(), ev.getNumBins()) == \
        ("areaUnderPR", "r", "y", 0)
    c = ev.copy({ev.numBins: 7})
    assert c.getNumBins() == 7 and ev.getNumBins() == 0 and c.getRawPredictionCol() == "r" and c.uid == ev.uid
    assert ev.setNumBins(3).getNumBins() == 3 and ev.setRawPredictionCol("q").getRawPredictionCol() == "q"


def test_errors():
    with pytest.raises(ValueError, match="numBins must be >= 0"):
        BinaryClassificationEvaluator(numBins=-1)
    ev = BinaryClassificationEvaluator(numBins=5)
    with pytest.raises(ValueError, match="numBins must be >= 0"):
        ev.setNumBins(-2)
    assert ev.getNumBins() == 5
    df = _frame([0.1, 0.9], [0.0, 1.0])
    with pytest.raises(ValueError, match="Unsupported metric name, found auc"):
        BinaryClassificationEvaluator(metricName="auc").evaluate(df)
    with pytest.raises(NotImplementedError, match="weightCol"):
        BinaryClassificationEvaluator(weightCol="w").evaluate(df)
    with pytest.raises(NotImplementedError, match="weightCol"):
        _eval_metric_info(BinaryClassificationEvaluator(weightCol="w"))
    with pytest.raises(ValueError, match="fewer than 2"):
        BinaryClassificationEvaluator().evaluate(_frame([[0.5], [0.2]], [0.0, 1.0]))
    with pytest.raises(ValueError, match="at least one row"):
        metrics.binary_metric([], [], "areaUnderROC", 0)


def test_single_pass_accepts_binary_classifiers_only():
    for name in NAMES:
        ev = BinaryClassificationEvaluator(metricName=name, numBins=17)
        assert _supports_transform_evaluate(True, ev) and not _supports_transform_evaluate(False, ev)
        info = _eval_metric_info(ev)
        assert info["binary"] and info["classification"] and info["numBins"] == 17 and info["metric"] == name
    assert not _supports_transform_evaluate(True, BinaryClassificationEvaluator(metricName="areaUnderXY"))


# ---- the oracle on hand-computed curves ----
@pytest.mark.parametrize("scores,labels,bins,roc,pr", [
    # heavy ties: 0.9 -> (1 pos, 1 neg), 0.5 -> (2, 0), 0.1 -> (0, 1)
    ([0.9, 0.9, 0.5, 0.5, 0.1], [1, 0, 1, 1, 0], 0, 7 / 12, 7 / 12),
    # all scores equal: one point
    ([0.3] * 4, [1, 0, 0, 1], 1000, 0.5, 0.5),
    # 5 distinct scores, numBins 2: g = 2, points {5, 4}, {3, 2}, {1} (a short last run)
    ([5, 4, 3, 2, 1], [1, 0, 1, 0, 0], 2, 2 / 3, 1 / 2),
    # numBins 3: g = 1, no down-sampling
    ([5, 4, 3, 2, 1], [1, 0, 1, 0, 0], 3, 5 / 6, 0.5 * (1.0 + 1.0) / 2 + 0.5 * (0.5 + 2 / 3) / 2),
    # NaN sorts above +inf and is one value
    ([math.nan, 2.0, 1.0, math.nan], [0, 1, 0, 1], 0, 0.625, 0.5 * (0.5 + 0.5) / 2 + 0.5 * (0.5 + 2 / 3) / 2),
    ([math.inf, math.nan, -math.inf], [1, 0, 1], 0, 0.0, None),   # the negative NaN ranks first
    # +0.0 above -0.0
    ([-0.0, 0.0], [0, 1], 0, 1.0, 1.0),
    # single class: guards give 0 (all negative) and 1 (all positive)
    ([3.0, 2.0, 1.0], [0, 0, 0], 0, 0.0, 0.0),
    ([3.0, 2.0, 1.0], [1, 1, 1], 0, 1.0, 1.0),
    ([1.0, 1.0], [0.7, 0.2], 0, 0.5, 0.5),   # label > 0.5 is positive
])
def test_oracle_hand_computed(scores, labels, bins, roc, pr):
    assert oracle.metric(scores, labels, "areaUnderROC", bins) == pytest.approx(roc, abs=1e-15)
    if pr is not None:
        assert oracle.metric(scores, labels, "areaUnderPR", bins) == pytest.approx(pr, abs=1e-15)
    for name, want in (("areaUnderROC", roc), ("areaUnderPR", pr)):
        if want is not None:
            assert metrics.binary_metric(scores, labels, name, bins) == pytest.approx(want, abs=1e-15)


def test_grouped_points_hand_computed():
    pts = oracle.down_sample(oracle.distinct_counts([5, 4, 3, 2, 1], [1, 0, 1, 0, 0]), 2)
    assert pts == [(1, 1), (1, 1), (0, 1)]
    assert oracle.roc_curve([5, 4, 3, 2, 1], [1, 0, 1, 0, 0], 2) == \
        [(0.0, 0.0), (1 / 3, 0.5), (2 / 3, 1.0), (1.0, 1.0), (1.0, 1.0)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_sklearn_without_ties(seed):
    rng = np.random.default_rng(seed)
    n = 2000
    y = (rng.random(n) < 0.3).astype(np.float64)
    s = rng.normal(size=n) + y
    assert len(set(s)) == n
    roc = oracle.metric(list(s), list(y), "areaUnderROC", 0)
    assert abs(roc - skm.roc_auc_score(y, s)) <= 1e-12
    p, r, _ = skm.precision_recall_curve(y, s)
    p, r = p[:-1][::-1], r[:-1][::-1]   # without sklearn's closing (recall 0, precision 1), in descending scores
    want = skm.auc(np.r_[0.0, r], np.r_[p[0], p])
    assert abs(oracle.metric(list(s), list(y), "areaUnderPR", 0) - want) <= 1e-12


@pytest.mark.parametrize("bins", [0, 1, 7, 50, 1000])
@pytest.mark.parametrize("name", NAMES)
def test_host_metric_matches_oracle(bins, name):
    rng = np.random.default_rng(bins)
    n = 3000
    y = rng.integers(0, 2, n).astype(np.float64)
    s = np.round(rng.normal(size=n) + y, 2)   # a few hundred distinct values, many ties
    s[:7] = np.nan
    s[7:9] = [-0.0, 0.0]
    want = oracle.metric(list(s), list(y), name, bins)
    assert abs(metrics.binary_metric(s, y, name, bins) - want) <= 1e-12 * abs(want)


def _frame(raw, labels, parts=2):
    ses = LocalSession()
    return ses.createDataFrame(pd.DataFrame({"rawPrediction": list(raw), "label": labels}), num_partitions=parts)


@pytest.mark.parametrize("name", NAMES)
def test_local_evaluate_matches_oracle(name):
    rng = np.random.default_rng(5)
    n = 500
    y = rng.integers(0, 2, n).astype(np.float64)
    s = np.round(rng.normal(size=n) + y, 1)
    raw = [np.array([-v, v]) for v in s]
    for bins in (0, 3, 1000):
        want = oracle.metric(list(s), list(y), name, bins)
        ev = BinaryClassificationEvaluator(metricName=name, numBins=bins)
        assert abs(ev.evaluate(_frame(raw, y)) - want) <= 1e-12 * abs(want)
        assert abs(ev.evaluate(_frame(list(s), y)) - want) <= 1e-12 * abs(want)   # a double column
    three = [np.array([0.2, v, 0.1]) for v in s]   # K classes: element 1 is the score
    assert BinaryClassificationEvaluator(metricName=name).evaluate(_frame(three, y)) == \
        pytest.approx(oracle.metric(list(s), list(y), name, 1000), rel=1e-12)
