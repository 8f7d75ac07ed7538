"""RandomForestClassifier / RandomForestRegressor end to end on one H100: a fit on a local frame (one or two
partitions) must give the oracle's forest, transform() must append the oracle's predictions, fitMultiple must equal
the single fits, and a saved model must load and transform alike."""
import json

import numpy as np
import pytest

import rf_oracle as ro

pytestmark = pytest.mark.gpu

pytest.importorskip("torch")


def _df(X, y, parts):
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    return LocalSession().createDataFrame([(X[i].tolist(), float(y[i])) for i in range(len(y))],
                                          "features array<float>, label float").repartition(parts)


def _data(n, d, seed, regression):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    if regression:
        return X, (X[:, 0] * 3 - X[:, 1] ** 2 + 0.3 * rng.normal(size=n)).astype(np.float32)
    return X, ((X[:, 0] + X[:, 2] > 0.3).astype(int) + (X[:, 1] > 1.0)).astype(np.float32)


def _oracle(X, y, est, classification):
    s = est._settings()
    k = ro.features_per_node(s["strategy"], X.shape[1], s["n_trees"], classification)
    return ro.fit(X, y, n_trees=s["n_trees"], max_depth=s["max_depth"], max_bins=s["max_bins"],
                  min_instances=s["min_instances"], features_per_node=k, bootstrap=s["bootstrap"],
                  impurity_name=s["impurity"], min_info_gain=s["min_info_gain"], seed=s["seed"])


@pytest.mark.parametrize("parts", [1, 2])
def test_classifier_end_to_end(parts, tmp_path):
    from spark_rapids_ml_b200.classification import RandomForestClassificationModel, RandomForestClassifier
    from spark_rapids_ml_b200.tree import forest_to_json

    X, y = _data(3000, 10, 1, False)
    est = RandomForestClassifier(numTrees=12, maxDepth=6, seed=7, num_workers=1)
    m = est.fit(_df(X, y, parts))
    ref = _oracle(X, y, est, True)
    assert m._model_json == forest_to_json(ref, True)
    assert m.numClasses == 3 and m.numFeatures == 10 and m.getNumTrees == 12
    assert m.totalNumNodes == int(ref["tree_offsets"][-1]) and m.treeWeights == [1.0] * 12
    np.testing.assert_array_equal(np.asarray(m.featureImportances), ro.feature_importances(ref, 10))
    rows = m.transform(_df(X, y, parts)).collect()
    raw, prob, pred = ro.predict(X, ref, True)
    np.testing.assert_array_equal(np.array([r["rawPrediction"] for r in rows]), raw)
    np.testing.assert_array_equal(np.array([r["probability"] for r in rows]), prob)
    np.testing.assert_array_equal(np.array([r["prediction"] for r in rows]), pred)
    path = str(tmp_path / "rfc")
    m.write().overwrite().save(path)
    m2 = RandomForestClassificationModel.load(path)
    assert m2._model_json == m._model_json and m2.numClasses == 3
    rows2 = m2.transform(_df(X, y, 1)).collect()
    np.testing.assert_array_equal(np.array([r["prediction"] for r in rows2]), pred)


def test_regressor_end_to_end_and_fit_multiple(tmp_path):
    from spark_rapids_ml_b200.regression import RandomForestRegressionModel, RandomForestRegressor

    X, y = _data(4000, 8, 2, True)
    df = _df(X, y, 2)
    est = RandomForestRegressor(numTrees=10, maxDepth=5, seed=3, num_workers=1)
    maps = [{est.maxDepth: 3}, {est.maxDepth: 6, est.numTrees: 4}, {est.maxBins: 64}]
    models = dict(est.fitMultiple(df, maps))
    for i, pm in enumerate(maps):
        single = est.copy(pm)
        one = single.fit(df)
        assert models[i]._model_json == one._model_json and models[i].cuml_params == one.cuml_params
        ref = _oracle(X, y, single, False)
        rows = models[i].transform(df).collect()
        np.testing.assert_array_equal(np.array([r["prediction"] for r in rows]), ro.predict(X, ref, False)[2])
    path = str(tmp_path / "rfr")
    models[1].write().overwrite().save(path)
    m2 = RandomForestRegressionModel.load(path)
    assert json.loads(m2._model_json) == json.loads(models[1]._model_json)


def test_reference_layout_model_transforms():
    """A model written in the reference's layout (tests/golden/rf_reference_model) loads through its model_json, with
    its "<" splits read at the float32 below their thresholds."""
    import os

    from spark_rapids_ml_b200.classification import RandomForestClassificationModel

    here = os.path.dirname(os.path.abspath(__file__))
    m = RandomForestClassificationModel.load(os.path.join(here, "golden", "rf_reference_model"))
    X = np.array([[0.5, 2.0], [1.0, 2.0], [1.0, 3.0], [3.0, 0.0]], dtype=np.float32)
    rows = m.transform(_df(X, np.zeros(4), 1)).collect()
    assert [r["prediction"] for r in rows] == [0.0, 1.0, 0.0, 1.0]
