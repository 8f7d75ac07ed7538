"""The single-pass evaluation against the hand loop of transform() + evaluate(), and CrossValidator end to end."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from spark_rapids_ml_b200 import metrics
from spark_rapids_ml_b200.classification import LogisticRegression, RandomForestClassifier
from spark_rapids_ml_b200.evaluation import MulticlassClassificationEvaluator, RegressionEvaluator
from spark_rapids_ml_b200.regression import LinearRegression, RandomForestRegressor
from spark_rapids_ml_b200.sparkshim import LocalSession
from spark_rapids_ml_b200.tuning import CrossValidator, CrossValidatorModel, ParamGridBuilder, k_fold

pytestmark = pytest.mark.gpu
COUNT_METRICS = [m for m in metrics.MULTICLASS_METRICS if m != "logLoss"]


def _frame(n, d, C=None, parts=2, seed=0, offset=0.0, batch=10000, label_dtype=np.float32):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    w = rng.normal(size=d)
    s = X @ w
    if C is None:
        y = (offset + s + rng.normal(size=n)).astype(np.float32)
    else:
        y = np.digitize(s + rng.normal(scale=0.5, size=n), np.quantile(s, np.linspace(0, 1, C + 1)[1:-1])).astype(np.float32)
    ses = LocalSession(conf={"spark.sql.execution.arrow.maxRecordsPerBatch": batch})
    return ses.createDataFrame(pd.DataFrame({"features": list(X), "label": y.astype(label_dtype)}),
                               num_partitions=parts)


def _check(est, maps, valid, train, evs, exact):
    models = [m for _, m in sorted(est.fitMultiple(train, maps), key=lambda t: t[0])]
    comb = models[0]._combine(models)
    for ev in evs:
        got = comb._transformEvaluate(valid, ev)
        again = comb._transformEvaluate(valid, ev)
        assert got == again or all(np.isnan(got))
        want = [ev.evaluate(m.transform(valid)) for m in models]
        if exact(ev.getMetricName()):
            assert got == want, ev.getMetricName()
        elif ev.getMetricName() == "r2":   # 1 - SSerr / SStot: the ratio holds 1e-12, r2 near 0 magnifies it
            np.testing.assert_allclose(1 - np.array(got), 1 - np.array(want), rtol=1e-12, err_msg="r2")
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, err_msg=ev.getMetricName())


def _cls_evs(label=1.0):
    return [MulticlassClassificationEvaluator(metricName=m, metricLabel=label) for m in metrics.MULTICLASS_METRICS]


def _reg_evs(var=True):
    return [RegressionEvaluator(metricName=m) for m in metrics.REGRESSION_METRICS if var or m != "var"]


@pytest.mark.parametrize("d", [1, 3, 127, 128, 513])
def test_logistic_binomial_and_multinomial(d):
    train, valid = _frame(600, d, C=3, seed=1), _frame(333, d, C=3, seed=2)
    lr = LogisticRegression(maxIter=20)
    maps = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.1]).addGrid(lr.family, ["binomial", "multinomial"]).build()
    tr2, va2 = _frame(600, d, C=2, seed=1), _frame(333, d, C=3, seed=2)   # label 2 absent from the training fold
    _check(lr, maps[:1] + maps[2:3], va2, tr2, _cls_evs(), lambda m: m != "logLoss")
    _check(lr, [maps[1], maps[3]], valid, train, _cls_evs(), lambda m: m != "logLoss")


def test_logistic_mixed_kinds_and_chunking():
    train, valid = _frame(400, 16, C=2, seed=3), _frame(1000, 16, C=2, seed=4)
    lr = LogisticRegression(maxIter=5)
    maps = [{lr.regParam: 0.01 * i, lr.family: "binomial" if i % 2 else "multinomial"} for i in range(33)]
    _check(lr, maps, valid, train, _cls_evs(0.0)[:3] + _cls_evs()[-1:], lambda m: m != "logLoss")


def test_linear_regression_large_offset():
    train, valid = _frame(500, 8, seed=5, offset=1e6), _frame(700, 8, seed=6, offset=1e6, parts=3)
    lr = LinearRegression()
    _check(lr, ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.5]).build(), valid, train, _reg_evs(var=False),
           lambda m: False)
    train, valid = _frame(500, 3, seed=5), _frame(700, 3, seed=6)
    _check(lr, [{lr.regParam: 0.0}], valid, train, _reg_evs(), lambda m: False)


def test_forests():
    train, valid = _frame(800, 5, C=3, seed=7), _frame(500, 5, C=3, seed=8)
    rf = RandomForestClassifier(numTrees=5, seed=1)
    _check(rf, ParamGridBuilder().addGrid(rf.maxBins, [8, 32]).addGrid(rf.maxDepth, [2, 4]).build(), valid, train,
           _cls_evs(), lambda m: m != "logLoss")
    train, valid = _frame(800, 5, seed=7), _frame(500, 5, seed=8)
    rr = RandomForestRegressor(numTrees=4, seed=2)
    _check(rr, ParamGridBuilder().addGrid(rr.maxBins, [8, 16]).build(), valid, train, _reg_evs(), lambda m: False)


def test_empty_validation_partition():
    train = _frame(300, 4, C=2, seed=9)
    valid = _frame(50, 4, C=2, seed=10, parts=1)
    valid = valid._derive([[]] + valid._parts, valid.schema)
    lr = LogisticRegression(maxIter=5)
    _check(lr, [{lr.regParam: 0.0}], valid, train, _cls_evs(0.0)[:2], lambda m: True)


def test_cross_validator_logistic(tmp_path):
    df = _frame(900, 6, C=2, seed=11)
    lr = LogisticRegression(maxIter=10)
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.1, 0.3]).addGrid(lr.elasticNetParam, [0.0, 1.0]).build()
    for name in ("accuracy", "f1"):
        ev = MulticlassClassificationEvaluator(metricName=name)
        cv = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=5,
                            collectSubModels=True)
        m = cv.fit(df)
        hand = [[ev.evaluate(lr.fit(t, pm).transform(v)) for pm in grid] for t, v in k_fold(df, 3, 5, None, 2)]
        assert m.avgMetrics == [float(a) for a in np.mean(hand, axis=0)]
        best = int(np.argmax(m.avgMetrics))
        ref = lr.fit(df, grid[best])
        assert m.bestModel.coef_ == ref.coef_ and m.bestModel.intercept_ == ref.intercept_
        assert len(m.subModels) == 3 and len(m.subModels[0]) == 6
    path = str(tmp_path / "cv")
    m.write().save(path)
    back = CrossValidatorModel.load(path)
    assert back.avgMetrics == m.avgMetrics
    assert ev.evaluate(back.transform(df)) == ev.evaluate(m.transform(df))


def _hand_avg(est, grid, ev, df, k, seed, fold_col=None):
    hand = [[ev.evaluate(est.fit(t, pm).transform(v)) for pm in grid] for t, v in k_fold(df, k, seed, fold_col, 2)]
    return np.mean(hand, axis=0)


def test_cross_validator_regressors_and_fold_col():
    df = _frame(600, 4, seed=12)
    rr = RandomForestRegressor(numTrees=3, seed=3)
    grid = ParamGridBuilder().addGrid(rr.maxBins, [8, 16]).build()
    ev = RegressionEvaluator()
    m = CrossValidator(estimator=rr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=4).fit(df)
    np.testing.assert_allclose(m.avgMetrics, _hand_avg(rr, grid, ev, df, 2, 4), rtol=1e-12)
    t = df._table()
    df2 = LocalSession().createDataFrame(t.append_column("fold", pa.array(np.arange(t.num_rows, dtype=np.int32) % 3)),
                                         num_partitions=2)
    lr = LinearRegression()
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 1.0]).build()
    ev = RegressionEvaluator(metricName="mae")
    m2 = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=ev, foldCol="fold").fit(df2)
    np.testing.assert_allclose(m2.avgMetrics, _hand_avg(lr, grid, ev, df2, 3, 0, "fold"), rtol=1e-12)
    assert m2.bestModel.coef_ == lr.fit(df2.select("features", "label"), grid[int(np.argmin(m2.avgMetrics))]).coef_


@pytest.fixture
def grid_limit():
    from spark_rapids_ml_b200.core import _transform_context

    ctx = _transform_context(0)
    ctx.set_option("grid_limit", 3)
    yield
    ctx.set_option("grid_limit", 0)


def test_many_tiles_per_cta(grid_limit):
    """3 CTAs over hundreds of tiles: the grid-stride loop, tile reuse and the tile-to-tile merges."""
    lr = LogisticRegression(maxIter=10)
    train, valid = _frame(2000, 128, C=3, seed=20), _frame(20011, 128, C=3, seed=21)
    maps = [{lr.regParam: 0.01, lr.family: "multinomial"}, {lr.regParam: 0.1, lr.family: "multinomial"}]
    _check(lr, maps, valid, train, _cls_evs(), lambda m: m != "logLoss")
    train, valid = _frame(2000, 12, seed=22, offset=1e6), _frame(20011, 12, seed=23, offset=1e6)
    lin = LinearRegression()
    _check(lin, ParamGridBuilder().addGrid(lin.regParam, [0.0, 0.1]).build(), valid, train, _reg_evs(var=False),
           lambda m: False)
    train, valid = _frame(1500, 8, C=3, seed=24), _frame(9001, 8, C=3, seed=25)
    rf = RandomForestClassifier(numTrees=4, seed=5)
    _check(rf, ParamGridBuilder().addGrid(rf.maxDepth, [3, 5]).build(), valid, train, _cls_evs(),
           lambda m: m != "logLoss")


def test_several_batch_groups(monkeypatch):
    """Partitions of many Arrow batches cut into several device passes, merged on the host within each partition."""
    from spark_rapids_ml_b200 import core

    monkeypatch.setattr(core, "TRANSFORM_GROUP_ROWS", 700)
    lr = LogisticRegression(maxIter=10)
    train, valid = _frame(800, 16, C=2, seed=30), _frame(5003, 16, C=2, seed=31, batch=300)
    _check(lr, [{lr.regParam: 0.0}, {lr.regParam: 0.2}], valid, train, _cls_evs(0.0), lambda m: m != "logLoss")
    train, valid = _frame(800, 16, seed=32, offset=1e6), _frame(5003, 16, seed=33, batch=300, offset=1e6)
    lin = LinearRegression()
    _check(lin, [{lin.regParam: 0.0}], valid, train, _reg_evs(var=False), lambda m: False)


def test_single_class_training_fold():
    """All training labels 0: infinite intercepts; the validation fold holds labels 0 and 1."""
    X = np.random.default_rng(40).normal(size=(300, 6)).astype(np.float32)
    train = LocalSession().createDataFrame(pd.DataFrame({"features": list(X), "label": np.zeros(300, np.float32)}),
                                           num_partitions=2)
    valid = _frame(400, 6, C=2, seed=41)
    lr = LogisticRegression(maxIter=5)
    _check(lr, [{lr.regParam: 0.0}, {lr.regParam: 0.5}], valid, train, _cls_evs(0.0), lambda m: m != "logLoss")


@pytest.mark.parametrize("d", [8, 128])
def test_forests_vector_staging(d):
    """d % 4 == 0: the float4 staging path of both forest kernels."""
    train, valid = _frame(900, d, C=4, seed=50), _frame(700, d, C=4, seed=51)
    rf = RandomForestClassifier(numTrees=6, seed=7)
    _check(rf, ParamGridBuilder().addGrid(rf.maxBins, [8, 32]).addGrid(rf.maxDepth, [3, 6]).build(), valid, train,
           _cls_evs(), lambda m: m != "logLoss")
    train, valid = _frame(900, d, seed=52), _frame(700, d, seed=53)
    rr = RandomForestRegressor(numTrees=5, seed=8)
    _check(rr, ParamGridBuilder().addGrid(rr.maxDepth, [3, 6]).build(), valid, train, _reg_evs(), lambda m: False)


@pytest.mark.parametrize("kind", ["logistic", "softmax", "identity", "forest"])
def test_unaligned_x_matches_aligned(kind):
    """d % 4 == 0 with X 4 bytes off a 16-byte boundary: the scalar staging path gives the aligned path's bits."""
    import torch

    from spark_rapids_ml_b200.core import _transform_context

    ctx = _transform_context(0)
    n, d = 3001, 32
    rng = np.random.default_rng(60)
    Xh = rng.normal(size=(n, d)).astype(np.float32)
    buf = torch.empty(n * d + 1, dtype=torch.float32, device="cuda")
    Xu = buf[1:].view(n, d)
    Xu.copy_(torch.as_tensor(Xh))
    Xa = torch.as_tensor(Xh).cuda()
    assert Xu.data_ptr() % 16 != 0 and Xa.data_ptr() % 16 == 0
    if kind == "forest":
        y = torch.as_tensor(rng.integers(0, 3, n).astype(np.float32)).cuda()
        forests = [ctx.rf_fit(Xa, y, n_trees=4, max_depth=4, seed=s) for s in range(2)]
        run = lambda X: ctx.eval_forest(X, y, forests, True)   # noqa: E731
    else:
        K = {"logistic": 1, "softmax": 3, "identity": 1}[kind]
        y = torch.as_tensor((rng.integers(0, 3, n) if kind != "identity" else rng.normal(size=n)).astype(np.float32))
        y = y.cuda()
        models = [{"kind": kind, "W": rng.normal(size=(K, d)), "b": rng.normal(size=K),
                   "class_values": np.arange(max(K, 2), dtype=np.float64)} for _ in range(3)]
        run = lambda X: ctx.eval_linear(X, y, models)   # noqa: E731
    a, u = run(Xa), run(Xu)
    for key in a:
        np.testing.assert_array_equal(np.asarray(a[key]), np.asarray(u[key]), err_msg=key)


def test_float64_label_is_scored_at_its_float32_rounding():
    rng = np.random.default_rng(70)
    X = rng.normal(size=(500, 5)).astype(np.float32)
    y64 = 1e6 + rng.normal(size=500)
    ses = LocalSession()
    df64 = ses.createDataFrame(pd.DataFrame({"features": list(X), "label": y64}), num_partitions=2)
    df32 = ses.createDataFrame(pd.DataFrame({"features": list(X), "label": y64.astype(np.float32).astype(np.float64)}),
                               num_partitions=2)
    lin = LinearRegression()
    model = lin.fit(df64)
    ev = RegressionEvaluator(metricName="rmse")
    comb = model._combine([model])
    np.testing.assert_allclose(comb._transformEvaluate(df64, ev), [ev.evaluate(model.transform(df32))], rtol=1e-12)
