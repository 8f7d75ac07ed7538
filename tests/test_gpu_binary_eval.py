"""Binary evaluation on the device: the score passes against transform()'s rawPrediction, the curve pass against the
fp64 oracle, the grouped single-pass evaluation against transform() + evaluate(), and CrossValidator end to end."""
import math

import numpy as np
import pandas as pd
import pytest
import torch

from spark_rapids_ml_b200 import _native, core
from spark_rapids_ml_b200.classification import LogisticRegression, RandomForestClassifier
from spark_rapids_ml_b200.evaluation import BinaryClassificationEvaluator
from spark_rapids_ml_b200.sparkshim import LocalSession
from spark_rapids_ml_b200.tree import json_to_forest
from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder, k_fold

import binary_oracle as oracle

pytestmark = pytest.mark.gpu
NAMES = ("areaUnderROC", "areaUnderPR")


def _data(n, d, C=2, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    s = X @ rng.normal(size=d)
    y = np.digitize(s + rng.normal(scale=0.7, size=n), np.quantile(s, np.linspace(0, 1, C + 1)[1:-1]))
    return X, y.astype(np.float32)


def _frame(X, y, parts=2, batch=10000):
    ses = LocalSession(conf={"spark.sql.execution.arrow.maxRecordsPerBatch": batch})
    return ses.createDataFrame(pd.DataFrame({"features": list(X), "label": y}), num_partitions=parts)


def _raw1(model, df):
    raw = model.transform(df).select("rawPrediction").toPandas()["rawPrediction"]
    return np.array([v[1] for v in raw], dtype=np.float64)


def _fit_all(est, maps, df):
    return [m for _, m in sorted(est.fitMultiple(df, maps), key=lambda t: t[0])]


def _device_scores(ctx, X, y, linear=None, forests=None):
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    m = len(linear or forests)
    scores, pos = ctx.binary_buffers(m, X.shape[0])
    if linear is not None:
        ctx.binary_scores_linear(Xd, yd, linear, scores, pos)
    else:
        ctx.binary_scores_forest(Xd, yd, forests, scores, pos)
    return scores, pos


@pytest.mark.parametrize("d", [3, 16, 130])
def test_scores_bitwise_equal_transform(d):
    X, y2 = _data(1500, d, 2, seed=d)
    _, y3 = _data(1500, d, 3, seed=d)
    df2, df3 = _frame(X, y2), _frame(X, y3)
    lr = LogisticRegression(maxIter=10)
    binomial = _fit_all(lr, [{lr.regParam: 0.0}, {lr.regParam: 0.1}], df2)
    softmax = _fit_all(lr, [{lr.family: "multinomial"}], df2) + _fit_all(lr, [{lr.regParam: 0.01}], df3)
    assert softmax[1].coefficientMatrix.shape[0] == 3
    models = binomial + softmax   # mixed kinds in one pass
    with _native.Context(0) as ctx:
        linear = [md for m in models for md in m._eval_models()]
        scores, pos = _device_scores(ctx, X, y2, linear=linear)
        for i, m in enumerate(models):
            want = _raw1(m, df2)
            assert np.array_equal(scores[i].cpu().numpy().view(np.uint64), want.view(np.uint64)), i
        assert np.array_equal(pos.cpu().numpy(), (y2 > 0.5).astype(np.uint8))
        rf = RandomForestClassifier(numTrees=4, seed=1)
        forests = _fit_all(rf, [{rf.maxDepth: 2}, {rf.maxDepth: 5, rf.maxBins: 16}], df3)
        scores, _ = _device_scores(ctx, X, y3, forests=[json_to_forest(m._model_json, m._num_classes) for m in forests])
        for i, m in enumerate(forests):
            assert np.array_equal(scores[i].cpu().numpy().view(np.uint64), _raw1(m, df3).view(np.uint64)), i


@pytest.mark.parametrize("bins", [0, 1000, 7])
def test_curve_matches_oracle_on_device_scores(bins):
    X, y = _data(3000, 8, 2, seed=4)
    df = _frame(X, y)
    lr, rf = LogisticRegression(maxIter=10), RandomForestClassifier(numTrees=3, maxDepth=3, seed=2)
    with _native.Context(0) as ctx:
        lin = [md for m in _fit_all(lr, [{lr.regParam: 0.0}, {lr.regParam: 1.0}], df) for md in m._eval_models()]
        sl, pl = _device_scores(ctx, X, y, linear=lin)
        fo = _fit_all(rf, [{rf.maxDepth: 3}], df)[0]
        sf, pf = _device_scores(ctx, X, y, forests=[json_to_forest(fo._model_json, fo._num_classes)])
        for scores, pos in ((sl, pl), (sf, pf)):
            s = scores.cpu().numpy()
            for name in NAMES:
                got = ctx.eval_binary(scores, pos, bins, name)
                for i in range(s.shape[0]):
                    want = oracle.metric(list(s[i]), list(y), name, bins)
                    assert abs(got[i] - want) <= 1e-12 * abs(want), (name, i, got[i], want)
                assert np.array_equal(got, ctx.eval_binary(scores, pos, bins, name))   # repeatable bits


def test_curve_edge_scores():
    rng = np.random.default_rng(3)
    n = 4000
    s = np.round(rng.normal(size=(3, n)), 1)
    s[0, :50] = np.nan
    s[0, 50:60] = np.inf
    s[0, 60:70] = -np.inf
    s[0, 70:90] = -0.0
    s[0, 90:100] = 0.0
    s[1] = 0.25                                   # all scores equal
    s[2, ::2] = np.nan                            # half NaN
    y = rng.integers(0, 2, n).astype(np.float64)
    with _native.Context(0) as ctx:
        scores = torch.from_numpy(s).cuda()
        pos = torch.from_numpy((y > 0.5).astype(np.uint8)).cuda()
        for name in NAMES:
            for bins in (0, 3, 1000):
                got = ctx.eval_binary(scores, pos, bins, name)
                for i in range(3):
                    want = oracle.metric(list(s[i]), list(y), name, bins)
                    assert abs(got[i] - want) <= 1e-12 * abs(want), (name, bins, i)
        # single-class sets: 0 when all negative, 1 when all positive
        for lab, want in ((0, 0.0), (1, 1.0)):
            p1 = torch.full((n,), lab, dtype=torch.uint8, device="cuda")
            for name in NAMES:
                assert ctx.eval_binary(scores, p1, 0, name) == pytest.approx([want] * 3, rel=1e-12, abs=1e-15)
                assert oracle.metric(list(s[0]), [lab] * n, name, 0) == pytest.approx(want, rel=1e-12, abs=1e-15)


def test_transform_evaluate_matches_hand_loop_and_groups(monkeypatch):
    X, y = _data(2500, 12, 2, seed=6)
    Xt, yt = _data(1200, 12, 2, seed=7)
    valid, train = _frame(X, y, parts=3, batch=300), _frame(Xt, yt)
    lr = LogisticRegression(maxIter=10)
    lmods = _fit_all(lr, [{lr.regParam: r, lr.family: f} for r in (0.0, 0.2) for f in ("binomial", "multinomial")],
                     train)
    rf = RandomForestClassifier(numTrees=4, seed=3)
    fmods = _fit_all(rf, [{rf.maxDepth: 2}, {rf.maxDepth: 4}], train)
    for models in (lmods, fmods):
        comb = models[0]._combine(models)
        for name in NAMES:
            for bins in (0, 1000, 5):
                ev = BinaryClassificationEvaluator(metricName=name, numBins=bins)
                got = comb._transformEvaluate(valid, ev)
                assert got == comb._transformEvaluate(valid, ev)
                want = [ev.evaluate(m.transform(valid)) for m in models]
                np.testing.assert_allclose(got, want, rtol=1e-12, err_msg=f"{name} {bins}")
                monkeypatch.setattr(core, "TRANSFORM_GROUP_ROWS", 97)   # many small groups: the same bits
                assert comb._transformEvaluate(valid, ev) == got
                monkeypatch.undo()


@pytest.mark.parametrize("which", ["logistic", "forest"])
def test_cross_validator(which):
    X, y = _data(1500, 6, 2, seed=11)
    df = _frame(X, y)
    if which == "logistic":
        est = LogisticRegression(maxIter=10)
        grid = ParamGridBuilder().addGrid(est.regParam, [0.0, 0.3, 3.0]).build()
    else:
        est = RandomForestClassifier(numTrees=3, seed=5)
        grid = ParamGridBuilder().addGrid(est.maxDepth, [1, 4]).addGrid(est.maxBins, [4, 32]).build()
    for name in NAMES:
        ev = BinaryClassificationEvaluator(metricName=name)
        m = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2).fit(df)
        hand = np.mean([[ev.evaluate(est.fit(t, pm).transform(v)) for pm in grid] for t, v in k_fold(df, 3, 2, None, 2)],
                       axis=0)
        np.testing.assert_allclose(m.avgMetrics, hand, rtol=1e-12)
        best = int(np.argmax(m.avgMetrics))
        assert best == int(np.argmax(hand))
        ref = est.fit(df, grid[best])
        got = m.bestModel
        if which == "logistic":
            assert got.coef_ == ref.coef_ and got.intercept_ == ref.intercept_
        else:
            assert got._model_json == ref._model_json


def test_errors_fail_cleanly(monkeypatch):
    X, y = _data(600, 4, 2, seed=8)
    train = _frame(X, y)
    lr = LogisticRegression(maxIter=5)
    comb = _fit_all(lr, [{lr.regParam: 0.0}], train)[0]
    ev = BinaryClassificationEvaluator()
    bad = y.copy()
    bad[17] = np.nan
    with pytest.raises(_native.B2KError, match="NaN or an infinity"):
        comb._transformEvaluate(_frame(X, bad), ev)
    bad[17] = np.inf
    with pytest.raises(_native.B2KError, match="NaN or an infinity"):
        comb._transformEvaluate(_frame(X, bad), ev)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (600 * 9 - 1, 80 << 30))
    with pytest.raises(MemoryError, match="need 5400 bytes of device memory"):
        comb._transformEvaluate(train, ev)
    monkeypatch.undo()
    assert math.isfinite(comb._transformEvaluate(train, ev)[0])
