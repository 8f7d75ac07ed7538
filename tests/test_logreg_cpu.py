"""Logistic regression without a GPU: the fp64 oracle against scikit-learn, the library's host optimizer
(b2k_logreg_minimize, with the oracle as its objective) against scipy's optimum and MLlib's known answers, the
estimator/model params and errors, persistence, the estimator end to end on local frames and on the pyspark branch with
host stand-ins for the device pieces, and the install proxy."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import logreg_oracle as lo
from spark_rapids_ml_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FAKE = os.path.join(ROOT, "tests", "fake_pyspark")


def _known():
    return json.load(open(os.path.join(GOLD, "logreg_known_answers.json")))


def _case_rows(c):
    """A known-answer case's rows: inline, or a data fixture beside the answers."""
    if "data" in c:
        z = np.load(os.path.join(GOLD, c["data"]))
        return z["X"], z["y"]
    return np.array(c["X"], dtype=np.float32), np.array(c["y"], dtype=np.float32)


def _data(n, d, K, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) * (1.0 + np.arange(d)) + offset).astype(np.float32)
    W = rng.normal(size=(K, d)) / (1.0 + np.arange(d))
    M = (X.astype(np.float64) - offset) @ W.T + rng.gumbel(size=(n, K))
    return X, M.argmax(1).astype(np.float32)


def _minimize(P, max_iter=1000, tol=1e-12):
    return _native.logreg_minimize(P.smooth, P.start(), l1=P.l1 if np.any(P.l1 > 0) else None, max_iter=max_iter,
                                   tol=tol)


def test_oracle_matches_sklearn():
    from sklearn.linear_model import LogisticRegression as SkLR

    for K in (2, 4):
        X, y = _data(300, 4, K, seed=K)
        C = 2.0
        sk = SkLR(C=C, tol=1e-14, max_iter=100000, solver="newton-cg").fit(X.astype(np.float64), y)
        # sklearn: sum loss + |W|^2 / (2C), unscaled features, intercept unpenalised (binomial: one margin)
        P = lo.Problem(X, y, reg=1.0 / (C * X.shape[0]), standardization=False)
        P.pen = np.ones(P.d)   # sklearn penalises W itself: the scaled frame with sigma = 1
        P.sig, P.inv = np.ones(P.d), np.ones(P.d)
        th = P.solve_scipy()
        W, b = P.model(th)
        if K == 2:
            np.testing.assert_allclose(W[0], sk.coef_[0], rtol=0, atol=1e-8)
            np.testing.assert_allclose(b, sk.intercept_, rtol=0, atol=1e-8)
        else:   # sklearn's multinomial intercepts are not centred; its coefficients sum to 0 per feature under L2 too
            np.testing.assert_allclose(W, sk.coef_, rtol=0, atol=1e-8)
            np.testing.assert_allclose(b, sk.intercept_ - sk.intercept_.mean(), rtol=0, atol=1e-8)
        # the loss itself against sklearn's log loss at the same parameters, to 1e-8
        from sklearn.metrics import log_loss

        probs = lo.predict(X, W, b, np.arange(K))["prob"]
        loss, _, _ = lo.loss_grad(X, y.astype(int), W, b)
        assert abs(loss - log_loss(y, probs, labels=np.arange(K))) <= 1e-8


@pytest.mark.parametrize("family,K", [("auto", 2), ("multinomial", 3)])
@pytest.mark.parametrize("reg,a", [(0.0, 0.0), (0.05, 0.0), (0.05, 1.0), (0.05, 0.4)])
@pytest.mark.parametrize("fi,st", [(True, True), (False, True), (True, False)])
def test_minimize_reaches_the_optimum(family, K, reg, a, fi, st):
    X, y = _data(200, 4, K, seed=11 + K)
    P = lo.Problem(X, y, reg=reg, l1_ratio=a, fit_intercept=fi, standardization=st, family=family)
    x, iters, evals, _ = _minimize(P)
    assert P.residual(x) <= 1e-8, (P.residual(x), iters, evals)
    ref = P.solve_scipy()
    f_x = P.smooth(x)[0] + float(P.l1 @ np.abs(x))
    f_r = P.smooth(ref)[0] + float(P.l1 @ np.abs(ref))
    assert f_x <= f_r + 1e-12 * max(1.0, abs(f_r))
    if reg > 0:   # a unique optimum (multinomial intercepts up to a common shift, which model() centres away)
        for u, v in zip(P.model(x), P.model(ref)):
            np.testing.assert_allclose(u, v, atol=1e-6)


def test_minimize_stopping_rules_and_errors():
    P = lo.Problem(*_data(100, 3, 2, seed=3), reg=0.01)
    x0 = P.start()
    _, it, ev, _ = _native.logreg_minimize(P.smooth, x0, max_iter=0)
    assert it == 0 and ev == 1
    _, it, _, _ = _native.logreg_minimize(P.smooth, x0, max_iter=3, tol=0.0)
    assert it == 3
    _, it_loose, _, _ = _native.logreg_minimize(P.smooth, x0, max_iter=1000, tol=1e-2)
    _, it_tight, _, _ = _native.logreg_minimize(P.smooth, x0, max_iter=1000, tol=1e-10)
    assert it_loose < it_tight
    with pytest.raises(_native.B2KError, match="maxIter given invalid value -1"):
        _native.logreg_minimize(P.smooth, x0, max_iter=-1)
    with pytest.raises(_native.B2KError, match="tol given invalid value"):
        _native.logreg_minimize(P.smooth, x0, tol=-1.0)
    with pytest.raises(_native.B2KError, match="L1 weights"):
        _native.logreg_minimize(P.smooth, x0, l1=-np.ones(x0.size))

    def boom(x):
        raise KeyError("from the objective")

    with pytest.raises(KeyError):
        _native.logreg_minimize(boom, x0)


def test_two_minimizations_are_bitwise_equal():
    P = lo.Problem(*_data(150, 5, 3, seed=5), reg=0.02, l1_ratio=0.5)
    a, b = _minimize(P), _minimize(P)
    assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]


def test_stable_loss_at_large_margins():
    X = np.array([[1.0], [1.0], [-1.0]], dtype=np.float32)
    for yi in (np.array([1, 0, 0]), np.array([0, 1, 1])):
        for kp, W in ((1, np.array([[1e3]])), (2, np.array([[1e3], [-1e3]]))):
            loss, gW, gb = lo.loss_grad(X, yi, W, np.zeros(kp))
            assert np.isfinite(loss) and np.all(np.isfinite(gW)) and np.all(np.isfinite(gb))


def test_a_row_of_no_class_has_a_zero_one_hot():
    rng = np.random.default_rng(11)
    X = rng.normal(size=(6, 3))
    for kp in (1, 4):
        W, b = rng.normal(size=(kp, 3)), rng.normal(size=kp)
        yi = np.array([0, 1, -1, 1, -1, 0]) if kp == 1 else np.array([0, 3, -1, 2, -1, 1])
        loss, gW, gb = lo.loss_grad(X, yi, W, b)
        M = X @ W.T + b
        if kp == 1:   # a row of no class is a negative row
            P = 1.0 / (1.0 + np.exp(-M))
            L = np.log1p(np.exp(M[:, 0])) - (yi == 1) * M[:, 0]
            Y = (yi == 1).astype(float)[:, None]
        else:   # the loss is log-sum-exp alone and the residuals the softmax alone
            P = np.exp(M) / np.exp(M).sum(axis=1, keepdims=True)
            L = np.log(np.exp(M).sum(axis=1)) - np.where(yi >= 0, M[np.arange(6), np.maximum(yi, 0)], 0.0)
            Y = np.zeros((6, kp))
            Y[yi >= 0, yi[yi >= 0]] = 1.0
        np.testing.assert_allclose(loss, L.mean(), rtol=1e-14)
        np.testing.assert_allclose(gW, (P - Y).T @ X / 6, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(gb, (P - Y).sum(axis=0) / 6, rtol=1e-12, atol=1e-15)


def test_known_answers_of_mllib_through_the_host_optimizer():
    """MLlib's published answers (tests/golden), to 1e-4 (the reference holds itself to 1e-3).  They pin the sample
    (n - 1) standard deviation: with the population one the standardized binomial coefficient is 2.678, not 2.482."""
    for c in _known()["cases"]:
        X, y = _case_rows(c)
        P = lo.Problem(X, y, reg=c["regParam"], l1_ratio=c["elasticNetParam"], fit_intercept=c["fitIntercept"],
                       standardization=c["standardization"], family=c["family"])
        x, _, _, _ = _minimize(P, max_iter=100, tol=1e-6)
        W, b = P.model(x)
        np.testing.assert_allclose(W, c["coefficientMatrix"], atol=1e-4, err_msg=c["name"])
        np.testing.assert_allclose(b, c["interceptVector"], atol=1e-4, err_msg=c["name"])
        if "first_row_probability" in c:
            out = lo.predict(X[:1], W, b, P.classes)
            np.testing.assert_allclose(out["prob"][0], c["first_row_probability"], atol=1e-4)
            np.testing.assert_allclose(out["raw"][0], c["first_row_rawPrediction"], atol=1e-4)
            assert out["pred"][0] == c["first_row_prediction"]


def test_params_defaults_mapping_and_validation():
    from spark_rapids_ml_b200.classification import LogisticRegression, LogisticRegressionModel

    lr = LogisticRegression()
    assert lr.getRegParam() == 0.0 and lr.getMaxIter() == 100 and lr.getTol() == 1e-6 and lr.getFamily() == "auto"
    assert lr.getFitIntercept() and lr.getStandardization() and lr.getElasticNetParam() == 0.0
    assert lr.getProbabilityCol() == "probability" and lr.getRawPredictionCol() == "rawPrediction"
    assert lr.cuml_params["C"] == 0.0 and lr.cuml_params["penalty"] is None and lr.cuml_params["max_iter"] == 100
    lr.setRegParam(0.5).setElasticNetParam(1.0)
    assert lr.cuml_params["C"] == 2.0 and lr.cuml_params["penalty"] == "l1" and lr.cuml_params["l1_ratio"] == 1.0
    lr.setElasticNetParam(0.3)
    assert lr.cuml_params["penalty"] == "elasticnet"
    assert LogisticRegression._reg_params_value_mapping(0.1, 0.0) == ("l2", 10.0, 0.0)
    assert LogisticRegression._param_mapping()["regParam"] == "C"
    assert LogisticRegression._param_mapping()["threshold"] is None
    with pytest.raises(ValueError, match="C or regParam given an invalid or unsupported value -1.0"):
        LogisticRegression().setRegParam(-1.0)
    with pytest.raises(ValueError, match="maxIter given invalid value -1"):
        LogisticRegression(maxIter=-1)._validate_parameters()
    for call in (lambda: LogisticRegression().setWeightCol("w"), lambda: LogisticRegression().setThreshold(0.2),
                 lambda: LogisticRegression(thresholds=[0.5, 0.5]),
                 lambda: LogisticRegression(lowerBoundsOnIntercepts=[0.0]),
                 lambda: LogisticRegression(enable_sparse_data_optim=True)):
        with pytest.raises(ValueError):
            call()
    m = LogisticRegressionModel(coef_=[[1.0, 2.0]], intercept_=[0.5], classes_=[0.0, 1.0], n_cols=2,
                                dtype="float32", num_iters=3)
    with pytest.raises(ValueError):
        m.setThreshold(0.2)


def test_model_surface_and_persistence(tmp_path):
    from spark_rapids_ml_b200.classification import LogisticRegression, LogisticRegressionModel

    est = LogisticRegression(regParam=0.5, maxIter=5, featuresCol="feats", labelCol="t")
    est.save(str(tmp_path / "est"))
    e2 = LogisticRegression.load(str(tmp_path / "est"))
    assert e2.uid == est.uid and e2.getRegParam() == 0.5 and e2.getMaxIter() == 5 and e2.getLabelCol() == "t"
    assert e2.cuml_params["C"] == 2.0
    bm = LogisticRegressionModel(coef_=[[1.5, -2.0]], intercept_=[0.25], classes_=[0.0, 1.0], n_cols=2,
                                 dtype="float32", num_iters=7)
    est._copyValues(bm)
    assert np.array_equal(bm.coefficients, [1.5, -2.0]) and bm.intercept == 0.25 and bm.numClasses == 2
    assert np.array_equal(np.asarray(bm.coefficientMatrix), [[1.5, -2.0]]) and bm.numFeatures == 2
    assert np.array_equal(bm.interceptVector, [0.25]) and bm.num_iters == 7 and bm.hasSummary is False
    with pytest.raises(RuntimeError, match="No training summary available"):
        bm.summary
    for call in (bm.cpu, lambda: bm.predict([1.0, 2.0]), lambda: bm.predictRaw([1.0, 2.0]),
                 lambda: bm.predictProbability([1.0, 2.0]), lambda: bm.evaluate(None)):
        with pytest.raises(NotImplementedError):
            call()
    mm = LogisticRegressionModel(coef_=[[1.0, 0.0], [0.0, 1.0], [-1.0, -1.0]], intercept_=[0.0, 0.0, 0.0],
                                 classes_=[0.0, 1.0, 2.0], n_cols=2, dtype="float32", num_iters=2)
    with pytest.raises(Exception, match="Multinomial models contain a matrix of coefficients"):
        mm.coefficients
    with pytest.raises(Exception, match="Multinomial models contain a vector of intercepts"):
        mm.intercept
    assert np.array_equal(mm.interceptVector.toArray(), [0.0, 0.0, 0.0])   # sparse: 1.5 (0 + 1) < 3
    assert type(mm.interceptVector).__name__ != "ndarray"
    comb = LogisticRegressionModel._combine([bm, bm])
    assert comb.coef_ == [bm.coef_, bm.coef_] and comb._get_num_models() == 2
    with pytest.raises(Exception, match="multi-model"):
        comb.coefficients
    bm.write().overwrite().save(str(tmp_path / "model"))
    m2 = LogisticRegressionModel.load(str(tmp_path / "model"))
    assert m2.uid == bm.uid and m2.coef_ == bm.coef_ and m2.intercept_ == bm.intercept_ and m2.getLabelCol() == "t"
    data = json.loads(open(tmp_path / "model" / "data" / "part-00000").read())
    assert data == {"coef_": [[1.5, -2.0]], "intercept_": [0.25], "classes_": [0.0, 1.0], "num_iters": 7, "n_cols": 2,
                    "dtype": "float32"}


def test_one_label_without_intercept_is_an_error():
    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.sparkshim import Row

    row = Row({"coef_": [[0.0, 0.0]], "intercept_": [float("inf")], "classes_": [1.0], "n_cols": 2,
               "dtype": "float32", "num_iters": 0})
    with pytest.raises(ValueError, match="All labels belong to a single class and fitIntercept=false"):
        LogisticRegression(fitIntercept=False)._create_pyspark_model(row)
    m = LogisticRegression()._create_pyspark_model(row)
    assert m.intercept == float("inf") and np.array_equal(m.coefficients, [0.0, 0.0])


# Host stand-ins for the device pieces, so that the label plumbing and the fit function run on a CPU: the appender keeps
# rows in a torch CPU tensor; the context finds classes with NumPy and fits with the library's host optimizer over the
# fp64 oracle.
_STUBS = '''
import sys
sys.path.insert(0, "tests")
import numpy as np, pandas as pd, torch
import logreg_oracle as lo
import spark_rapids_ml_b200.core as core
import spark_rapids_ml_b200.utils as utils
import spark_rapids_ml_b200.common.cuml_context as cc
from spark_rapids_ml_b200 import _native

class HostAppender:
    def __init__(self, ctx, d, first_capacity=0):
        self.d, self.rows_ = d, []
    def append_values(self, values, offsets, n_b):
        lo_ = int(offsets[0]) if offsets is not None else 0
        self.rows_.append(np.asarray(values[lo_:lo_ + n_b * self.d], dtype=np.float32).reshape(n_b, self.d))
    def append_columns(self, cols):
        self.rows_.append(np.stack(cols, 1).astype(np.float32))
    def finish(self):
        return torch.from_numpy(np.concatenate(self.rows_))

CALLS = {"labels": 0, "fit": 0}
class HostHandle:
    device = torch.device("cpu")
    def logreg_labels(self, y):
        assert y.dtype == torch.float32
        CALLS["labels"] += 1
        c, n, _ = lo.classes_of(y.numpy())
        return c, n, int(y.shape[0])
    def logreg_fit(self, X, y, classes, counts, settings):
        CALLS["fit"] += 1
        out = []
        for s in settings:
            P = lo.Problem(X.numpy(), y.numpy(), s["reg"], s["l1_ratio"], s["fit_intercept"], s["standardization"],
                           s["family"])
            x, it, _, _ = _native.logreg_minimize(P.smooth, P.start(), P.l1 if np.any(P.l1 > 0) else None,
                                                  s["max_iter"], s["tol"])
            W, b = P.model(x)
            out.append((W, b, it))
        return out
    def logreg_predict(self, X, W, b, cls):
        o = lo.predict(X.numpy(), W, b, cls)
        return torch.from_numpy(o["raw"]), torch.from_numpy(o["prob"]), torch.from_numpy(o["pred"])

class HostContext:
    def __init__(self, *a, **k): self.handle, self._loop = HostHandle(), None
    def __enter__(self): return self
    def __exit__(self, *a): return None

core.DeviceRowAppender = utils.DeviceRowAppender = HostAppender
cc.CumlContext = HostContext
core._CumlCommon._set_gpu_device = staticmethod(lambda context, is_local, is_transform=False: 0)
core._transform_context = lambda gpu: HostHandle()
'''

_LOCAL = '''
import json
from spark_rapids_ml_b200.sparkshim.sql import LocalSession
from spark_rapids_ml_b200.classification import LogisticRegression
rng = np.random.default_rng(0)
X = rng.normal(size=(300, 3)).astype(np.float32)
y = (X.astype(np.float64) @ [2.0, -1.0, 0.5] + rng.normal(size=300) > 0).astype(np.float64)
y3 = np.where(X[:, 0] > 0.5, 2.0, y)
sess = LocalSession()
df = sess.createDataFrame([(X[i].tolist(), float(y[i]), float(y3[i])) for i in range(300)],
                          "features array<float>, target double, t3 double").repartition(3)
lr = LogisticRegression(labelCol="target", regParam=0.01, tol=1e-10, num_workers=1)
m = lr.fit(df)
P = lo.Problem(X, y.astype(np.float32), 0.01)
W, b = P.model(P.solve_scipy())
res = {"coef_err": float(np.abs(np.asarray(m.coefficients) - W[0]).max()), "b_err": abs(m.intercept - b[0])}
out = m.transform(df)
rows = out.collect()
o = lo.predict(X, W, b, P.classes)
res["prob_err"] = float(np.abs(np.array([r["probability"] for r in rows]) - o["prob"]).max())
res["raw_err"] = float(np.abs(np.array([r["rawPrediction"] for r in rows]) - o["raw"]).max())
res["pred_same"] = bool(np.array_equal(np.array([r["prediction"] for r in rows]), o["pred"]))
res["types"] = [str(dict(out.dtypes)[c]) for c in ("rawPrediction", "probability", "prediction")]
m3 = LogisticRegression(labelCol="t3", num_workers=1).fit(df)
res["multi"] = [m3.numClasses, len(m3.coef_), m3.classes_]
res["multi_pred"] = sorted(set(r["prediction"] for r in m3.transform(df).collect()))
CALLS.update(labels=0, fit=0)
maps = [{lr.regParam: r, lr.elasticNetParam: a} for r in (0.0, 0.1) for a in (0.0, 0.5)]
models = dict(lr.fitMultiple(df, maps))
res["single_pass_calls"] = dict(CALLS)
singles = [lr.copy(pm).fit(df) for pm in maps]
res["same_as_single_fits"] = all(models[i].coef_ == s.coef_ and models[i].intercept_ == s.intercept_
                                 and models[i].getRegParam() == s.getRegParam() for i, s in enumerate(singles))
res["same_cuml_params"] = [models[i].cuml_params == s.cuml_params for i, s in enumerate(singles)]
try:
    LogisticRegression(labelCol="nope").fit(df)
except ValueError as e:
    res["missing_label"] = str(e)
print("RESULT " + json.dumps(res))
'''


def _run(script: str, with_fake_pyspark: bool) -> dict:
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join(([FAKE] if with_fake_pyspark else []) + [ROOT, env.get("PYTHONPATH", "")])
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(script)], env=env, capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


def test_estimator_end_to_end_on_local_frames_with_core_context_stub():
    res = _run(_STUBS + _LOCAL, with_fake_pyspark=False)
    assert res["coef_err"] < 1e-6 and res["b_err"] < 1e-6, res
    assert res["prob_err"] < 1e-6 and res["raw_err"] < 1e-5 and res["pred_same"], res
    assert res["types"][2] == "double" and all("double" in t for t in res["types"]), res
    assert res["multi"][0] == 3 and res["multi"][1] == 3 and res["multi"][2] == [0.0, 1.0, 2.0], res
    assert set(res["multi_pred"]) <= {0.0, 1.0, 2.0}, res
    assert res["single_pass_calls"] == {"labels": 1, "fit": 1} and res["same_as_single_fits"], res
    assert all(res["same_cuml_params"]), res
    assert "label column 'nope' not found" in res["missing_label"], res


_PYSPARK = '''
import json
from pyspark import CALLS as SPARK_CALLS
from pyspark.sql import DataFrame
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
from spark_rapids_ml_b200.classification import LogisticRegression
rng = np.random.default_rng(1)
X = rng.normal(size=(300, 3))
y = (X @ np.array([1.0, -2.0, 3.0]) > 0).astype(np.float64)
local = shim.LocalSession().createDataFrame([(X[i].tolist(), float(y[i])) for i in range(300)],
                                            "features array<double>, label double")
df = DataFrame(local, vector_cols=("features",))
m = LogisticRegression(regParam=0.1, num_workers=1).fit(df)
P = lo.Problem(X.astype(np.float32), y.astype(np.float32), 0.1)
W, b = P.model(P.solve_scipy())
selects = [c[1] for c in SPARK_CALLS if c[0] == "select"]
print("RESULT " + json.dumps({"coef_err": float(np.abs(np.asarray(m.coefficients) - W[0]).max()),
                              "selects": selects}))
'''


def test_pyspark_branch_carries_the_label():
    res = _run(_STUBS + _PYSPARK, with_fake_pyspark=True)
    assert res["coef_err"] < 1e-5, res
    from spark_rapids_ml_b200.core import alias

    assert any(["label", alias.label, "float"] in [list(c) for c in sel] for sel in res["selects"]), res["selects"]


_PROXY = '''
import sys, json
import pyspark.ml.classification as stock_mod
StockLR = stock_mod.LogisticRegression
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
import spark_rapids_ml_b200.install as inst
from pyspark.ml.classification import LogisticRegression as L1, LogisticRegressionModel as M1
from spark_rapids_ml_b200.classification import LogisticRegression
import pyspark.ml, pyspark.ml.param
res = {
    "stock_classes_kept": L1 is StockLR and getattr(M1, "stock", False) is True,
    "estimator_and_model_types": issubclass(LogisticRegression, pyspark.ml.Estimator),
    "pyspark_params": isinstance(LogisticRegression().getParam("regParam"), pyspark.ml.param.Param),
}
print("RESULT " + json.dumps(res))
'''


def test_install_proxy_leaves_classification_to_pyspark():
    """LogisticRegressionModel.transform() of a pyspark DataFrame is not built, so the no-import-change mode keeps
    pyspark.ml.classification's own classes: code written for MLlib keeps working end to end."""
    res = _run(_PROXY, with_fake_pyspark=True)
    for key in ("stock_classes_kept", "estimator_and_model_types", "pyspark_params"):
        assert res[key] is True, (key, res)
