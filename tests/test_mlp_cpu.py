"""Multilayer perceptron without a GPU: the fp64 oracle (tests/mlp_oracle.py) against central differences and the
hand-derived known answers, the flat weight layout, the init rule, the gd update and stopping rule, the estimator's
params and Spark's messages, the model surface and persistence, and that the oracle's error bound holds for a CPU
emulation of the 3xTF32 wgmma path and rejects the same path with the lo half of the split dropped."""
import json
import os

import numpy as np
import pytest

import mlp_oracle as mo
from spark_rapids_ml_b200.classification import (MultilayerPerceptronClassificationModel,
                                                 MultilayerPerceptronClassifier)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mlp_known_answers.json")


@pytest.mark.parametrize("layers", [[3, 2], [3, 4, 2], [2, 5, 3, 4], [1, 1, 1, 2]])
def test_oracle_gradient_matches_central_differences(layers):
    rng = np.random.default_rng(len(layers))
    X = rng.normal(size=(9, layers[0]))
    y = rng.integers(0, layers[-1], size=9).astype(np.float64)
    w = rng.normal(size=mo.n_weights(layers))
    _, g = mo.eval_fg(layers, w, X, y)
    h = 1e-6
    fd = np.array([(mo.eval_fg(layers, w + h * e, X, y)[0] - mo.eval_fg(layers, w - h * e, X, y)[0]) / (2 * h)
                   for e in np.eye(w.size)])
    np.testing.assert_allclose(g, fd, atol=1e-8)


def test_known_answers():
    with open(GOLDEN) as f:
        cases = json.load(f)
    assert [c["name"] for c in cases] == ["zero_weights", "one_layer"]
    for c in cases:
        F, g = mo.eval_fg(c["layers"], np.array(c["w"]), np.array(c["X"]), np.array(c["y"], dtype=np.float64))
        assert F == pytest.approx(c["F"], rel=1e-14)
        np.testing.assert_allclose(g, c["grad"], rtol=1e-13, atol=1e-15)


def test_flat_layout_round_trip():
    layers = [3, 2, 4]
    w = np.arange(mo.n_weights(layers), dtype=np.float64)
    (W1, b1), (W2, b2) = mo.unpack(layers, w)
    # W_1 is 2 x 3 column-major: element (o, i) at i * 2 + o
    assert W1[1, 2] == 2 * 2 + 1 and W1[0, 1] == 2
    np.testing.assert_array_equal(b1, [6, 7])
    assert W2.shape == (4, 2) and W2[3, 1] == 8 + 1 * 4 + 3
    np.testing.assert_array_equal(b2, [16, 17, 18, 19])
    np.testing.assert_array_equal(mo.pack(mo.unpack(layers, w)), w)
    assert mo.n_weights(layers) == 20


def test_init_rule():
    w = mo.init_weights([4, 3, 2], seed=5)
    assert w.size == mo.n_weights([4, 3, 2])
    assert np.all(np.abs(w[:15]) <= 2.4 / 2.0) and np.all(np.abs(w[15:]) <= 2.4 / np.sqrt(3))
    np.testing.assert_array_equal(w, mo.init_weights([4, 3, 2], seed=5))
    assert not np.array_equal(w, mo.init_weights([4, 3, 2], seed=6))
    # counter-based: the first layer's values do not depend on the later layers
    np.testing.assert_array_equal(mo.init_weights([4, 3, 7], seed=5)[:15], w[:15])


def test_gd_update_and_stopping_rule():
    calls = []

    def fun(w):
        calls.append(w.copy())
        return float(w @ w), 2.0 * w

    w, hist = mo.gd(fun, np.array([1.0, -2.0]), max_iter=3, tol=0.0, step_size=0.1)
    np.testing.assert_allclose(calls[1], np.array([1.0, -2.0]) * (1 - 0.2))
    np.testing.assert_allclose(calls[2], calls[1] * (1 - 0.2 / np.sqrt(2)))
    assert len(hist) == 3 and hist[0] == 5.0
    # ||w_t - w_{t-1}|| = 0.2 / sqrt(t) ||w_{t-1}||; tol = 0.25 stops at t = 1 since 0.2 < 0.25 * 0.8
    _, h2 = mo.gd(fun, np.array([1.0, -2.0]), max_iter=10, tol=0.25, step_size=0.1)
    assert len(h2) == 1


def test_params_and_messages():
    est = MultilayerPerceptronClassifier(layers=[4, 5, 3])
    assert (est.getMaxIter(), est.getTol(), est.getBlockSize(), est.getSolver(), est.getStepSize()) == \
        (100, 1e-6, 128, "l-bfgs", 0.03)
    assert est.getRawPredictionCol() == "rawPrediction" and est.getProbabilityCol() == "probability"
    assert est.getLabelCol() == "label" and est.getInitialWeights() is None
    est._validate_parameters()
    bad = [({"layers": [4]}, "at least 2 entries"), ({"layers": [4, 0, 2]}, "every entry must be > 0"),
           ({"layers": [4, 2], "maxIter": -1}, "maxIter given invalid value -1"),
           ({"layers": [4, 2], "tol": -1.0}, "tol given invalid value"),
           ({"layers": [4, 2], "solver": "sgd"}, "solver given invalid value sgd"),
           ({"layers": [4, 2], "stepSize": 0.0}, "stepSize given invalid value"),
           ({"layers": [4, 2], "blockSize": 0}, "blockSize given invalid value"),
           ({"layers": [4, 2], "initialWeights": [0.0] * 3}, "initialWeights has 3 values")]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            MultilayerPerceptronClassifier(**kw)._validate_parameters()
    with pytest.raises(ValueError, match="layers must be set"):
        MultilayerPerceptronClassifier()._validate_parameters()
    with pytest.raises(ValueError, match="thresholds"):
        MultilayerPerceptronClassifier(layers=[2, 2], thresholds=[0.5, 0.5])
    with pytest.raises(ValueError, match="thresholds"):
        est.setThresholds([0.5, 0.5])
    e2 = est.setInitialWeights(np.zeros(mo.n_weights([4, 5, 3]))).setSolver("gd").setStepSize(0.5)
    assert e2.getInitialWeights() == [0.0] * 43 and e2.cuml_params["solver"] == "gd"
    assert e2.cuml_params["step_size"] == 0.5


def _model():
    layers = [2, 3, 2]
    w = list(np.linspace(-1, 1, mo.n_weights(layers)))
    return MultilayerPerceptronClassificationModel(weights_=w, layers_=layers, objective_history_=[0.7, 0.5, 0.4],
                                                   n_cols=2, dtype="float32")


def test_model_surface_and_persistence(tmp_path):
    m = _model()
    assert m.numFeatures == 2 and m.numClasses == 2 and m.getLayers() == [2, 3, 2]
    np.testing.assert_array_equal(np.asarray(m.weights), m.weights_)
    s = m.summary()
    assert s.objectiveHistory == [0.7, 0.5, 0.4] and s.totalIterations == 3
    assert m._transform_outputs() == [("rawPrediction", "array<double>"), ("probability", "array<double>"),
                                      ("prediction", "double")]
    for f in (lambda: m.predict([0.0, 0.0]), lambda: m.predictRaw([0.0, 0.0]),
              lambda: m.predictProbability([0.0, 0.0]), m.cpu):
        with pytest.raises(NotImplementedError):
            f()
    m.setProbabilityCol("p")
    m.write().overwrite().save(str(tmp_path / "model"))
    m2 = MultilayerPerceptronClassificationModel.load(str(tmp_path / "model"))
    assert m2.weights_ == m.weights_ and m2.layers_ == [2, 3, 2] and m2.summary().objectiveHistory == [0.7, 0.5, 0.4]
    assert m2.getProbabilityCol() == "p" and m2.numClasses == 2
    est = MultilayerPerceptronClassifier(layers=[2, 3, 2], solver="gd", maxIter=7)
    est.save(str(tmp_path / "est"))
    e2 = MultilayerPerceptronClassifier.load(str(tmp_path / "est"))
    assert e2.getLayers() == [2, 3, 2] and e2.getSolver() == "gd" and e2.getMaxIter() == 7
    assert e2.cuml_params["max_iter"] == 7


# the wgmma-path shapes of tests/test_gpu_mlp.py (d % 4 == 0), with its data rule
WG_CASES = [([64, 63, 10], 300, {}), ([128, 64, 65], 257, {}), ([128, 129, 63, 1, 10], 513, {}),
            ([784, 129, 10], 200, {}), ([4, 64, 64, 64, 65], 100, {}), ([128, 64, 32, 10], 3000, {}),
            ([16, 63, 65, 3], 700, {"shift": 20.0}), ([16, 63, 65, 3], 700, {"scale": 30.0})]


@pytest.mark.parametrize("layers,n,kw", WG_CASES)
def test_bound_holds_for_3xtf32_and_rejects_1xtf32(layers, n, kw):
    """A CPU emulation of the wgmma path stays well inside mo.eval_bound with the 3xTF32 split; with the lo half of the
    split dropped (hi.hi alone) it leaves the bound, on F or on some gradient entry."""
    rng = np.random.default_rng(n + len(layers))
    X = (rng.normal(size=(n, layers[0])) * kw.get("scale", 1.0) + kw.get("shift", 0.0)).astype(np.float32)
    y = rng.integers(0, layers[-1], size=n).astype(np.float64)
    w = rng.normal(size=mo.n_weights(layers)) * 0.5
    Fo, go = mo.eval_fg(layers, w, X.astype(np.float64), y)
    bF, bg = mo.eval_bound(layers, w, X.astype(np.float64), y)
    F3, g3 = mo.emulate_wgmma(layers, w, X, y, split=3)
    assert abs(F3 - Fo) <= 0.25 * bF and (np.abs(g3 - go) <= 0.25 * bg).all()
    F1, g1 = mo.emulate_wgmma(layers, w, X, y, split=1)
    assert abs(F1 - Fo) > bF or (np.abs(g1 - go) > 2 * bg).any()
    z, bz = mo.z_bound(layers, w, X.astype(np.float64))
    assert bz.shape == z.shape and (bz > 0).all()
