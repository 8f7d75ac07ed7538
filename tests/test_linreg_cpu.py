"""Linear regression without a GPU: the fp64 oracle against scikit-learn, the library's host solver (b2k_linreg_solve)
against the oracle and MLlib's known answers, the estimator/model params, persistence, the worker plumbing of the label
(local frames and the pyspark branch, with host stand-ins for the device pieces) and the install proxy."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import linreg_oracle as lo
from spark_rapids_ml_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FAKE = os.path.join(ROOT, "tests", "fake_pyspark")


def _known():
    return json.load(open(os.path.join(GOLD, "linreg_known_answers.json")))


def _data(n, d, seed, noise=0.1, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) * (1.0 + np.arange(d)) + offset).astype(np.float32)
    w = rng.normal(size=d)
    y = (X.astype(np.float64) @ w + 2.5 + noise * rng.normal(size=n)).astype(np.float32)
    return X, y


def _solve(X, y, reg=0.0, l1=0.0, fi=True, st=True, max_iter=100, tol=1e-6):
    n, m, M = lo.moments(X, y)
    return _native.linreg_solve(m, M, n, reg, l1, fi, st, max_iter, tol)


def test_oracle_matches_sklearn():
    from sklearn.linear_model import ElasticNet, Lasso, LinearRegression, Ridge

    X, y = _data(300, 6, 0)
    X64, y64 = X.astype(np.float64), y.astype(np.float64)
    n = len(y)
    for fi in (True, False):
        w, b, _ = lo.fit(X, y, 0.0, 0.0, fi, False)
        sk = LinearRegression(fit_intercept=fi).fit(X64, y64)
        np.testing.assert_allclose(w, sk.coef_, rtol=1e-10)
        assert abs(b - sk.intercept_) <= 1e-9 * max(1.0, abs(sk.intercept_))
        # ridge: (1/2n)|r|^2 + lam/2 |w|^2  ==  sklearn's |r|^2 + (lam n) |w|^2, up to a factor 2n
        w, b, _ = lo.fit(X, y, 0.7, 0.0, fi, False)
        sk = Ridge(alpha=0.7 * n, fit_intercept=fi, solver="cholesky").fit(X64, y64)
        np.testing.assert_allclose(w, sk.coef_, rtol=1e-9)
        for l1, cls in ((1.0, Lasso), (0.4, ElasticNet)):
            w, b, _ = lo.fit(X, y, 0.3, l1, fi, False)
            kw = {} if cls is Lasso else {"l1_ratio": l1}
            sk = cls(alpha=0.3, fit_intercept=fi, tol=1e-14, max_iter=100000, **kw).fit(X64, y64)
            np.testing.assert_allclose(w, sk.coef_, rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("fi", [True, False])
@pytest.mark.parametrize("st", [True, False])
@pytest.mark.parametrize("kind", ["ols", "ridge", "lasso", "elastic_net"])
def test_solver_matches_the_oracle(kind, fi, st):
    reg, l1 = {"ols": (0.0, 0.0), "ridge": (0.5, 0.0), "lasso": (0.2, 1.0), "elastic_net": (0.2, 0.5)}[kind]
    X, y = _data(500, 8, 1, offset=3.0)
    w, b, it = _solve(X, y, reg, l1, fi, st, max_iter=100000, tol=1e-12)
    w_ref, b_ref, f = lo.fit(X, y, reg, l1, fi, st)
    if l1 == 0.0 or reg == 0.0:
        assert it == 0
        np.testing.assert_allclose(w, w_ref, rtol=1e-12 * 100, atol=0)
        assert abs(b - b_ref) <= 1e-10 * max(1.0, abs(b_ref))
    else:
        lam = reg / f["sy"]
        v = lo.solver_frame_v(w, f)
        assert lo.kkt_residual(f["A"], f["c"], v, lam * l1, lam * (1 - l1)) <= 1e-10 * np.abs(f["c"]).max()
        assert np.array_equal(v == 0, lo.solver_frame_v(w_ref, f) == 0)
        if fi:
            assert abs(b - (f["muy"] - w @ f["mu"])) <= 1e-12 * max(1.0, abs(b))
        else:
            assert b == 0.0


def test_cd_stops_within_tol():
    X, y = _data(400, 10, 2)
    f = lo.frame(X, y)
    lam = 0.3 / f["sy"]
    for tol in (1e-3, 1e-6, 1e-9):
        w, _, it = _solve(X, y, 0.3, 0.5, tol=tol, max_iter=10000)
        v = lo.solver_frame_v(w, f)
        # after a sweep moved no coordinate by more than tol max|v|, the KKT slack is of that order
        assert lo.kkt_residual(f["A"], f["c"], v, lam * 0.5, lam * 0.5) <= 10 * tol * np.abs(f["A"]).max() * np.abs(v).sum()
    _, _, it = _solve(X, y, 0.3, 0.5, tol=0.0, max_iter=3)
    assert it == 3
    w, b, it = _solve(X, y, 0.3, 0.5, max_iter=0)
    assert it == 0 and not w.any() and b == pytest.approx(float(y.astype(np.float64).mean()), rel=1e-12)


def test_collinear_columns_give_the_minimum_norm_split():
    X, y = _data(300, 3, 3)
    Xd = np.c_[X, X[:, 1]]   # a duplicate of column 1
    for st in (True, False):
        w, b, _ = _solve(Xd, y, st=st)
        w_ref, b_ref, _ = lo.fit(Xd, y, standardization=st)
        np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-9 * np.abs(w_ref).max())
        assert w[1] == pytest.approx(w[3], rel=1e-9)
        w3, _, _ = _solve(X, y, st=st)
        assert w[1] + w[3] == pytest.approx(w3[1], rel=1e-9)
        assert b == pytest.approx(b_ref, rel=1e-9)


def test_zero_variance_feature_and_constant_label():
    X, y = _data(200, 4, 4)
    X[:, 2] = 7.0
    for st in (True, False):
        w, b, _ = _solve(X, y, st=st)
        w_ref, b_ref, _ = lo.fit(X, y, standardization=st)
        assert abs(w[2]) <= 1e-12 * np.abs(w).max()   # minimum norm: no weight on a constant column
        np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-12 * np.abs(w).max())
        assert b == pytest.approx(b_ref, rel=1e-9)
    yc = np.full(200, 3.0, dtype=np.float32)
    w, b, it = _solve(X, yc, 0.1, 0.5, fi=True, st=True)
    assert not w.any() and b == 3.0 and it == 0
    # no intercept and a non-zero constant label: s_y = |muy|
    w, b, _ = _solve(X, yc, 0.0, 0.0, fi=False, st=True)
    w_ref, _, _ = lo.fit(X, yc, 0.0, 0.0, False, True)
    np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-12)
    w, b, _ = _solve(X, np.zeros(200, np.float32), fi=False)
    assert not w.any() and b == 0.0


def test_d_equal_1_and_d_equal_1024():
    X, y = _data(100, 1, 5)
    for reg, l1 in ((0.0, 0.0), (0.5, 0.0), (0.5, 1.0)):
        w, b, _ = _solve(X, y, reg, l1, max_iter=1000, tol=1e-14)
        w_ref, b_ref, _ = lo.fit(X, y, reg, l1)
        np.testing.assert_allclose(w, w_ref, rtol=1e-11)
        assert b == pytest.approx(b_ref, rel=1e-10, abs=1e-12)
    X, y = _data(3000, 1024, 6)
    w, b, _ = _solve(X, y, 0.1, 0.0)
    w_ref, b_ref, _ = lo.fit(X, y, 0.1, 0.0)
    np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-11 * np.abs(w_ref).max())
    n, m, M = lo.moments(X[:, :4], y)
    with pytest.raises(_native.B2KError, match="d <= 1024"):
        _native.linreg_solve(np.zeros(1026), np.eye(1026), 10)


def test_known_answers_of_mllib_through_the_host_solver():
    k = _known()
    X, y = np.array(k["X"]), np.array(k["y"])
    for name, c in k["cases"].items():
        w, b, _ = _solve(X, y, c["regParam"], c["elasticNetParam"], max_iter=200)
        np.testing.assert_allclose(w, c["coefficients"], rtol=1e-6, err_msg=name)
        assert abs(b - c["intercept"]) <= c.get("intercept_atol", 1e-6 * abs(c["intercept"])), (name, b)
        if "first_prediction" in c:
            assert b + np.float32(X[0]).astype(np.float64) @ w == pytest.approx(c["first_prediction"], rel=1e-6)


def test_solver_errors():
    n, m, M = lo.moments(*_data(50, 3, 7))
    for kw, msg in (({"reg": -1.0}, "regParam given invalid value -1.0"),
                    ({"l1_ratio": 1.5}, "elasticNetParam given invalid value 1.5"),
                    ({"max_iter": -1}, "maxIter given invalid value -1"),
                    ({"tol": -0.1}, "tol given invalid value -0.1")):
        with pytest.raises(_native.B2KError, match=msg):
            _native.linreg_solve(m, M, n, **kw)
    bad = M.copy()
    bad[0, 1] = np.inf
    with pytest.raises(_native.B2KError, match="NaN or an infinity"):
        _native.linreg_solve(m, bad, n)
    with pytest.raises(_native.B2KError, match="at least 1 row"):
        _native.linreg_solve(m, M, 0)


def test_params_defaults_mapping_and_validation():
    from spark_rapids_ml_b200.regression import LinearRegression

    lr = LinearRegression()
    assert (lr.getMaxIter(), lr.getRegParam(), lr.getElasticNetParam(), lr.getTol()) == (100, 0.0, 0.0, 1e-6)
    assert lr.getFitIntercept() and lr.getStandardization() and lr.getSolver() == "auto"
    assert lr.getLoss() == "squaredError" and lr.getLabelCol() == "label" and lr.getFeaturesCol() == "features"
    assert lr.getPredictionCol() == "prediction"
    cp = lr.cuml_params
    assert (cp["alpha"], cp["l1_ratio"], cp["max_iter"], cp["tol"], cp["fit_intercept"], cp["normalize"]) == \
        (0.0, 0.0, 100, 1e-6, True, True)
    lr = LinearRegression(regParam=0.5, elasticNetParam=0.3, maxIter=7, tol=1e-4, fitIntercept=False,
                          standardization=False, solver="normal", featuresCol=["a", "b"], labelCol="t")
    cp = lr.cuml_params
    assert (cp["alpha"], cp["l1_ratio"], cp["max_iter"], cp["tol"], cp["fit_intercept"], cp["normalize"],
            cp["solver"]) == (0.5, 0.3, 7, 1e-4, False, False, "eig")
    assert lr.getFeaturesCol() == ["a", "b"] and lr._fit_label_col() == "t"
    lr.setRegParam(2.0).setElasticNetParam(1.0).setMaxIter(3).setTol(0.0).setFitIntercept(True)
    assert (lr.cuml_params["alpha"], lr.cuml_params["l1_ratio"], lr.cuml_params["max_iter"]) == (2.0, 1.0, 3)
    for kw, msg in (({"regParam": -1.0}, "regParam given invalid value -1.0"),
                    ({"elasticNetParam": 1.5}, "elasticNetParam given invalid value 1.5"),
                    ({"maxIter": -1}, "maxIter given invalid value -1"),
                    ({"tol": -1.0}, "tol given invalid value -1.0")):
        with pytest.raises(ValueError, match=msg):
            LinearRegression(**kw)._validate_parameters()
    with pytest.raises(ValueError, match="huber"):
        LinearRegression(loss="huber")
    with pytest.raises(ValueError, match="l-bfgs"):
        LinearRegression(solver="l-bfgs")
    with pytest.raises(ValueError, match="weightCol"):
        LinearRegression(weightCol="w")
    with pytest.raises(ValueError, match="weightCol"):
        LinearRegression().setWeightCol("w")
    c = lr.copy({lr.regParam: 0.25})
    assert c.cuml_params["alpha"] == 0.25 and lr.cuml_params["alpha"] == 2.0


def test_spark_confs():
    from spark_rapids_ml_b200.regression import LinearRegression
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    sess = LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()
    sess.conf.set("spark.rapids.ml.num_workers", "3")
    sess.conf.set("spark.rapids.ml.verbose", "true")
    try:
        lr = LinearRegression()
        assert lr._num_workers == 3 and lr.cuml_params["verbose"] is True
        assert LinearRegression(num_workers=2)._num_workers == 2
        sess.conf.set("spark.rapids.ml.num_workers", "zero")
        with pytest.raises(ValueError, match="spark.rapids.ml.num_workers"):
            LinearRegression()
    finally:
        sess.conf.unset("spark.rapids.ml.num_workers")
        sess.conf.unset("spark.rapids.ml.verbose")


def test_model_surface_and_persistence(tmp_path):
    from spark_rapids_ml_b200.regression import LinearRegression, LinearRegressionModel

    est = LinearRegression(regParam=0.5, maxIter=5, featuresCol="feats", labelCol="t")
    est.save(str(tmp_path / "est"))
    e2 = LinearRegression.load(str(tmp_path / "est"))
    assert e2.uid == est.uid and e2.getRegParam() == 0.5 and e2.getMaxIter() == 5 and e2.getLabelCol() == "t"
    assert e2.cuml_params["alpha"] == 0.5 and e2.getFeaturesCol() == "feats"
    m = LinearRegressionModel(coef_=[1.5, -2.0], intercept_=0.25, n_cols=2, dtype="float32")
    est._copyValues(m)
    assert np.array_equal(m.coefficients, [1.5, -2.0]) and m.intercept == 0.25 and m.scale == 1.0
    assert m.numFeatures == 2 and m.hasSummary is False and m.getRegParam() == 0.5
    assert m._out_schema(None) == "double" and m._output_col_name() == "prediction"
    for call in (m.cpu, lambda: m.predict([1.0, 2.0]), lambda: m.evaluate(None), lambda: m.summary):
        with pytest.raises(NotImplementedError):
            call()
    m.write().overwrite().save(str(tmp_path / "model"))
    m2 = LinearRegressionModel.load(str(tmp_path / "model"))
    assert m2.uid == m.uid and m2.coef_ == m.coef_ and m2.intercept_ == m.intercept_ and m2.getLabelCol() == "t"
    data = json.loads(open(tmp_path / "model" / "data" / "part-00000").read())
    assert data == {"coef_": [1.5, -2.0], "intercept_": 0.25, "n_cols": 2, "dtype": "float32"}


def test_directory_written_by_the_reference_loads_here(tmp_path):
    """The reference's _CumlModelWriter layout: metadata/part-00000 (DefaultParamsWriter JSON + the cuML params) and
    data/part-00000 = json.dumps(model attributes), with Hadoop _SUCCESS markers."""
    from spark_rapids_ml_b200.regression import LinearRegressionModel

    path = tmp_path / "ref_lr_model"
    meta = {"class": "spark_rapids_ml.regression.LinearRegressionModel", "timestamp": 1700000000000,
            "sparkVersion": "3.5.1", "uid": "LinearRegression_0c1d2e3f4a5b",
            "paramMap": {"regParam": 2.0, "elasticNetParam": 0.5, "maxIter": 200, "featuresCol": "features",
                         "labelCol": "label"},
            "defaultParamMap": {"tol": 1e-06, "fitIntercept": True, "standardization": True, "solver": "auto",
                                "loss": "squaredError", "predictionCol": "prediction"},
            "_cuml_params": {"algorithm": "auto", "fit_intercept": True, "copy_X": True, "normalize": True,
                             "verbose": False, "alpha": 2.0, "solver": "auto", "loss": "squared_loss",
                             "l1_ratio": 0.5, "max_iter": 200, "tol": 1e-06, "shuffle": True},
            "_num_workers": 2, "_float32_inputs": True}
    attrs = {"coef_": [91.9070094, 11.23076474], "intercept_": 3.138371491598421, "n_cols": 2, "dtype": "float32"}
    for sub, obj in (("metadata", meta), ("data", attrs)):
        os.makedirs(path / sub)
        (path / sub / "part-00000").write_text(json.dumps(obj) + "\n")
        (path / sub / "_SUCCESS").write_text("")
    m = LinearRegressionModel.load(str(path))
    assert m.uid == "LinearRegression_0c1d2e3f4a5b" and m.getRegParam() == 2.0 and m.getElasticNetParam() == 0.5
    assert m._num_workers == 2 and m.n_cols == 2 and m.coef_ == attrs["coef_"] and m.intercept == attrs["intercept_"]
    assert m.cuml_params["alpha"] == 2.0


# Host stand-ins for the device pieces, so that the label plumbing and the fit function run on a CPU: the appender keeps
# rows in a torch CPU tensor, the context forms the moments in NumPy, the host solver is the library's.
_STUBS = '''
import numpy as np, pandas as pd, torch
import spark_rapids_ml_b200.core as core
import spark_rapids_ml_b200.utils as utils
import spark_rapids_ml_b200.common.cuml_context as cc

class HostAppender:
    def __init__(self, ctx, d, first_capacity=0):
        self.d, self.rows_ = d, []
    def append_values(self, values, offsets, n_b):
        lo = int(offsets[0]) if offsets is not None else 0
        self.rows_.append(np.asarray(values[lo:lo + n_b * self.d], dtype=np.float32).reshape(n_b, self.d))
    def append_columns(self, cols):
        self.rows_.append(np.stack(cols, 1).astype(np.float32))
    def finish(self):
        return torch.from_numpy(np.concatenate(self.rows_))

CALLS_MOMENTS = []
class HostHandle:
    device = torch.device("cpu")
    def linreg_moments(self, X, y):
        assert y.dtype == torch.float32 and tuple(y.shape) == (X.shape[0],)
        CALLS_MOMENTS.append(int(X.shape[0]))
        V = np.c_[X.numpy().astype(np.float64), y.numpy().astype(np.float64)]
        m = V.mean(0)
        return V.shape[0], m, (V - m).T @ (V - m)
    def linreg_predict(self, X, w, b):
        return torch.from_numpy(b + X.numpy().astype(np.float64) @ w.numpy())

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
import sys, json
sys.path.insert(0, "tests")
import linreg_oracle as lo
from spark_rapids_ml_b200.sparkshim.sql import LocalSession
from spark_rapids_ml_b200.regression import LinearRegression
rng = np.random.default_rng(0)
X = rng.normal(size=(400, 5)).astype(np.float32)
y = (X.astype(np.float64) @ np.arange(1, 6) + 1.0 + 0.1 * rng.normal(size=400))
sess = LocalSession()
df = sess.createDataFrame([(X[i].tolist(), float(y[i])) for i in range(400)], "features array<float>, target double")
df = df.repartition(3)
lr = LinearRegression(labelCol="target", regParam=0.1, elasticNetParam=0.5, tol=1e-12, maxIter=10000, num_workers=1)
m = lr.fit(df)
w, b, _ = lo.fit(X, y.astype(np.float32), 0.1, 0.5)
res = {"coef_err": float(np.abs(np.asarray(m.coefficients) - w).max()), "b_err": abs(m.intercept - b)}
out = m.transform(df)
pred = np.array([r["prediction"] for r in out.collect()])
res["pred_err"] = float(np.abs(pred - (m.intercept + X.astype(np.float64) @ np.asarray(m.coef_))).max())
res["pred_is_double"] = str(dict(out.dtypes)["prediction"])
del CALLS_MOMENTS[:]
maps = [{lr.regParam: r, lr.elasticNetParam: a} for r in (0.0, 0.1) for a in (0.0, 0.5, 1.0)]
models = dict(lr.fitMultiple(df, maps))
res["single_pass_moments_calls"] = len(CALLS_MOMENTS)
singles = [lr.copy(pm).fit(df) for pm in maps]
res["same_as_single_fits"] = all(models[i].coef_ == s.coef_ and models[i].intercept_ == s.intercept_
                                 and models[i].getRegParam() == s.getRegParam() for i, s in enumerate(singles))
res["same_cuml_params"] = [models[i].cuml_params == s.cuml_params for i, s in enumerate(singles)]
del CALLS_MOMENTS[:]
models = dict(lr.fitMultiple(df, [{lr.labelCol: "target"}, {lr.maxIter: 3}]))
res["fallback_moments_calls"] = len(CALLS_MOMENTS)
try:
    LinearRegression(labelCol="nope").fit(df)
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


def test_local_frames_carry_the_label_and_fit_multiple_takes_one_pass_with_core_context_stub():
    res = _run(_STUBS + _LOCAL, with_fake_pyspark=False)
    assert res["coef_err"] < 1e-9 and res["b_err"] < 1e-9, res
    assert res["pred_err"] < 1e-9 and res["pred_is_double"] == "double", res
    assert res["single_pass_moments_calls"] == 1 and res["same_as_single_fits"], res
    assert all(res["same_cuml_params"]), res
    assert res["fallback_moments_calls"] == 2, res
    assert "label column 'nope' not found" in res["missing_label"], res


_PYSPARK = '''
import sys, json
from pyspark import CALLS
from pyspark.sql import DataFrame
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
from spark_rapids_ml_b200.regression import LinearRegression
rng = np.random.default_rng(1)
X = rng.normal(size=(300, 4))
y = X @ np.array([1.0, -2.0, 3.0, 0.5]) + 4.0
local = shim.LocalSession().createDataFrame([(X[i].tolist(), float(y[i])) for i in range(300)],
                                            "features array<double>, label double")
df = DataFrame(local, vector_cols=("features",))
m = LinearRegression(num_workers=1).fit(df)
selects = [c[1] for c in CALLS if c[0] == "select"]
print("RESULT " + json.dumps({"coef": list(map(float, m.coefficients)), "intercept": m.intercept,
                              "selects": selects}))
'''


def test_pyspark_branch_carries_the_label():
    res = _run(_STUBS + _PYSPARK, with_fake_pyspark=True)
    np.testing.assert_allclose(res["coef"], [1.0, -2.0, 3.0, 0.5], rtol=1e-5)
    assert res["intercept"] == pytest.approx(4.0, rel=1e-5)
    from spark_rapids_ml_b200.core import alias

    assert any(["label", alias.label, "float"] in [list(c) for c in sel] for sel in res["selects"]), res["selects"]


_PROXY = '''
import sys, json
import pyspark.ml.regression as stock_mod
StockLR = stock_mod.LinearRegression
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
import spark_rapids_ml_b200.install as inst
from spark_rapids_ml_b200.regression import LinearRegression, LinearRegressionModel
from pyspark.ml.regression import LinearRegression as L1, LinearRegressionModel as M1, RandomForestRegressor as R1
import pyspark.ml, pyspark.ml.param
res = {
    "user_import_is_accelerated": L1 is LinearRegression and M1 is LinearRegressionModel
                                  and pyspark.ml.regression.LinearRegression is LinearRegression,
    "other_names_untouched": getattr(R1, "stock", False) is True,
    "estimator_and_model_types": issubclass(LinearRegression, pyspark.ml.Estimator)
                                 and issubclass(LinearRegressionModel, pyspark.ml.Model),
    "pyspark_params": isinstance(LinearRegression().getParam("regParam"), pyspark.ml.param.Param),
}
inst.uninstall()
res["uninstall_restores"] = sys.modules["pyspark.ml.regression"].LinearRegression is StockLR
print("RESULT " + json.dumps(res))
'''


def test_install_proxy_for_regression():
    res = _run(_PROXY, with_fake_pyspark=True)
    for key in ("user_import_is_accelerated", "other_names_untouched", "estimator_and_model_types", "pyspark_params",
                "uninstall_restores"):
        assert res[key] is True, (key, res)
