"""MultilayerPerceptronClassifier / MultilayerPerceptronClassificationModel end to end on local frames over several
partitions: a fit learns a nonlinear problem, MulticlassClassificationEvaluator scores the transform within a few
points of scikit-learn's MLPClassifier (lbfgs, logistic) when it is installed, else of the oracle-driven fit, and the
model round-trips through save and load with the same transform."""
import numpy as np
import pytest

import mlp_oracle as mo
from spark_rapids_ml_b200.classification import (MultilayerPerceptronClassificationModel,
                                                 MultilayerPerceptronClassifier)

pytestmark = pytest.mark.gpu


@pytest.fixture()
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "500", "spark.rapids.ml.num_workers.local": "1"})


def _rings(n, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, 4))
    r = np.linalg.norm(X[:, :2], axis=1)
    y = np.digitize(r, [0.8, 1.5])   # three classes by radius: not linearly separable
    return X.astype(np.float32), y.astype(np.float64)


def test_fit_transform_evaluate_and_persistence(session, tmp_path):
    from spark_rapids_ml_b200.evaluation import MulticlassClassificationEvaluator

    X, y = _rings(6000, 0)
    Xt, yt = _rings(3000, 1)
    tr = session.from_numpy(X, num_partitions=3, extra={"label": y})
    te = session.from_numpy(Xt, num_partitions=2, extra={"label": yt})
    layers = [4, 16, 3]
    model = MultilayerPerceptronClassifier(layers=layers, maxIter=200, seed=7).fit(tr)
    assert model.numFeatures == 4 and model.numClasses == 3 and len(model.weights) == mo.n_weights(layers)
    s = model.summary()
    assert s.totalIterations == len(s.objectiveHistory) > 10
    out = model.transform(te)
    acc = MulticlassClassificationEvaluator(metricName="accuracy").evaluate(out)
    pdf = out.toPandas()
    raw = np.stack(pdf["rawPrediction"].to_numpy())
    z, p, pred = mo.predict(layers, np.asarray(model.weights_), Xt.astype(np.float64))
    np.testing.assert_allclose(raw, z, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.stack(pdf["probability"].to_numpy()), p, atol=1e-4)
    try:
        from sklearn.neural_network import MLPClassifier

        ref = MLPClassifier(hidden_layer_sizes=(16,), activation="logistic", solver="lbfgs", alpha=0.0,
                            max_iter=200, random_state=0).fit(X, y).score(Xt, yt)
    except ImportError:
        w, *_ = __import__("spark_rapids_ml_b200._native", fromlist=["logreg_minimize"]).logreg_minimize(
            lambda w: mo.eval_fg(layers, w, X.astype(np.float64), y), mo.init_weights(layers, 7), max_iter=200,
            tol=1e-6)
        ref = float((mo.predict(layers, w, Xt.astype(np.float64))[2] == yt).mean())
    assert acc > 0.9 and acc >= ref - 0.05, (acc, ref)

    model.write().overwrite().save(str(tmp_path / "mlp"))
    m2 = MultilayerPerceptronClassificationModel.load(str(tmp_path / "mlp"))
    assert m2.weights_ == model.weights_ and m2.layers_ == layers
    np.testing.assert_array_equal(m2.transform(te).toPandas()["prediction"].to_numpy(), pdf["prediction"].to_numpy())


def test_refusals(session):
    X, y = _rings(200, 2)
    df = session.from_numpy(X, extra={"label": y})
    with pytest.raises(ValueError, match="must equal the number of features"):
        MultilayerPerceptronClassifier(layers=[5, 3], maxIter=2).fit(df)
    with pytest.raises(ValueError, match="layers must be set"):
        MultilayerPerceptronClassifier(maxIter=2).fit(df)
