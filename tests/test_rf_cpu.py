"""Random forests without a GPU: the NumPy oracle (tests/rf_oracle.py) against scikit-learn's decision trees and
forests, the semantics' known answers (tests/golden/rf_known_answers.json, written by make_rf_known_answers.py), and
the estimator surface: params, value mappings, validation, Spark confs, persistence and model_json."""
import json
import os
import re

import numpy as np
import pytest

import rf_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "rf_known_answers.json")
SK = {"gini": "gini", "entropy": "entropy", "variance": "squared_error"}


def _tree_data(n, d, seed, impurity):
    if impurity == "variance":
        rng = np.random.default_rng(seed)
        # every feature has <= 32 distinct values, so every midpoint is a candidate (as in scikit-learn)
        X = (rng.integers(0, 25, size=(n, d)) * rng.uniform(0.5, 2.0, size=d)).astype(np.float32)
        y = X[:, 0] * 0.3 - X[:, 1] + rng.normal(size=n) * 3   # continuous labels: no gains tie
        return X, y.astype(np.float32)
    # class labels can tie two gains in a small node, where scikit-learn breaks the tie at random: seed 0 has no tie
    rng = np.random.default_rng(0)
    X = np.take_along_axis(rng.normal(size=(32, d)), rng.integers(0, 32, size=(n, d)), axis=0).astype(np.float32)
    y = ((X[:, 0] + X[:, 2 % d] + rng.normal(size=n)) > 0).astype(int) + (X[:, 1] > 1) * 2
    return X, y.astype(np.float32)


def _partition(labels):
    groups = {}
    for i, g in enumerate(labels):
        groups.setdefault(int(g), []).append(i)
    return sorted(tuple(v) for v in groups.values())


@pytest.mark.parametrize("impurity", ["gini", "entropy", "variance"])
@pytest.mark.parametrize("depth", [2, 5])
def test_oracle_tree_matches_sklearn(impurity, depth):
    tree = pytest.importorskip("sklearn.tree")
    X, y = _tree_data(700, 5, depth, impurity)
    F = ro.fit(X, y, n_trees=1, max_depth=depth, max_bins=32, bootstrap=False, impurity_name=impurity, seed=3)
    cls = tree.DecisionTreeRegressor if impurity == "variance" else tree.DecisionTreeClassifier
    sk = cls(criterion=SK[impurity], max_depth=depth, random_state=0).fit(X, y)
    lf = ro.leaves(X, F)[:, 0]
    assert _partition(lf) == _partition(sk.apply(X))
    _, prob, pred = ro.predict(X, F, impurity != "variance")
    if impurity == "variance":
        # labels are resolved to max|y| 2^-24 (the fixed-point grid)
        np.testing.assert_allclose(pred, sk.predict(X), rtol=0, atol=np.abs(y).max() * 2.0 ** -23)
    else:
        np.testing.assert_allclose(prob, sk.predict_proba(X), rtol=0, atol=1e-15)


@pytest.mark.parametrize("classification", [True, False])
def test_forest_accuracy_near_sklearn(classification):
    ens = pytest.importorskip("sklearn.ensemble")
    rng = np.random.default_rng(9)
    X = rng.normal(size=(4000, 10)).astype(np.float32)
    if classification:
        y = ((X[:, 0] + X[:, 1] * X[:, 2] + 0.5 * rng.normal(size=4000)) > 0).astype(np.float32)
    else:
        y = (np.sin(X[:, 0] * 2) + X[:, 1] ** 2 + 0.3 * rng.normal(size=4000)).astype(np.float32)
    tr, te = slice(0, 3000), slice(3000, None)
    k = ro.features_per_node("auto", 10, 20, classification)
    F = ro.fit(X[tr], y[tr], n_trees=20, max_depth=8, max_bins=32, features_per_node=k,
               impurity_name="gini" if classification else "variance", seed=1)
    pred = ro.predict(X[te], F, classification)[2]
    if classification:
        sk = ens.RandomForestClassifier(20, max_depth=8, max_features="sqrt", random_state=0).fit(X[tr], y[tr])
        ours, theirs = (pred == y[te]).mean(), (sk.predict(X[te]) == y[te]).mean()
        assert ours >= theirs - 0.03, (ours, theirs)   # held-out accuracy within 3 points
    else:
        sk = ens.RandomForestRegressor(20, max_depth=8, max_features=1 / 3, random_state=0).fit(X[tr], y[tr])
        ours = np.sqrt(((pred - y[te]) ** 2).mean())
        theirs = np.sqrt(((sk.predict(X[te]) - y[te]) ** 2).mean())
        assert ours <= theirs * 1.10, (ours, theirs)   # held-out RMSE within 10 %


def test_known_answers():
    g = json.load(open(GOLDEN))
    for c in g["hash"]:
        assert int(ro.rf_hash(c["seed"], c["stream"], c["tree"], [c["index"]])[0]) == c["h"]
    assert ro.POISSON_CDF.tolist() == g["poisson_cdf"]
    for c in g["poisson"]:
        assert int(ro.poisson([c["u"]])[0]) == c["w"]
    for c in g["subsets"]:
        assert ro.feature_subset(c["seed"], c["tree"], c["heap"], c["d"], c["k"]).tolist() == c["features"]
    for c in g["thresholds"]:
        t = ro.thresholds_of(np.array(c["col"], dtype=np.float32), c["max_bins"])
        assert t.tolist() == [float(np.float32(v)) for v in c["t"]]


def test_header_states_the_table_and_hash():
    """include/b2kmeans.h's Poisson table and hash constants are the oracle's."""
    h = open(os.path.join(HERE, "..", "include", "b2kmeans.h")).read()
    table = re.search(r"#define B2K_RF_POISSON_CDF\s*\\\s*\{([^}]*)\}", h).group(1).replace("\\", "")
    assert [int(v.strip().rstrip("u")) for v in table.split(",")] == ro.POISSON_CDF.tolist()
    for const in ("0xBF58476D1CE4E5B9", "0x94D049BB133111EB", "0x9E3779B97F4A7C15"):
        assert const in h


def test_bootstrap_weights_are_poisson_one():
    w = ro.weights(5, 0, 200000, True)
    assert abs(w.mean() - 1.0) < 0.01 and abs(w.var() - 1.0) < 0.02 and w.max() <= ro.POISSON_CAP
    assert ro.weights(5, 0, 10, False).tolist() == [1] * 10


def test_sample_fraction_and_thresholds():
    assert ro.sample_rows(1, 5000, 32).size == 5000            # M = 10000 >= n: every row
    rows = ro.sample_rows(1, 200000, 128)                       # M = 16384
    assert abs(rows.size - 16384) < 600
    t = ro.thresholds_of(np.array([1.0, 2.0, 2.0, np.nextafter(np.float32(2), np.float32(3))], dtype=np.float32), 32)
    assert t.tolist() == [1.5, 2.0]   # the midpoint of two adjacent floats rounds to the upper one: use the lower


@pytest.mark.parametrize("strategy, d, trees, cls, k", [
    ("auto", 100, 1, True, 100), ("auto", 100, 5, True, 10), ("auto", 100, 5, False, 34), ("all", 7, 3, True, 7),
    ("sqrt", 17, 3, True, 5), ("log2", 17, 3, True, 5), ("log2", 1, 3, True, 1), ("onethird", 10, 3, False, 4),
    ("3", 10, 3, True, 3), ("30", 10, 3, True, 10), ("0.25", 10, 3, True, 3), ("1.0", 10, 3, True, 10)])
def test_features_per_node(strategy, d, trees, cls, k):
    from spark_rapids_ml_b200.tree import features_per_node

    assert features_per_node(strategy, d, trees, cls) == k == ro.features_per_node(strategy, d, trees, cls)


def test_log2_is_close_to_numpy():
    p = np.linspace(1e-6, 1.0, 10001)
    np.testing.assert_allclose(ro.log2(p), np.log2(p), rtol=0, atol=4e-16 * np.abs(np.log2(p)).max())


# ---- the estimator surface ----
def test_defaults_and_mappings():
    from spark_rapids_ml_b200.classification import RandomForestClassifier
    from spark_rapids_ml_b200.regression import RandomForestRegressor

    for E, imp, crit in ((RandomForestClassifier, "gini", "gini"), (RandomForestRegressor, "variance", "mse")):
        est = E()
        assert (est.getMaxBins(), est.getMaxDepth(), est.getOrDefault("numTrees"), est.getBootstrap(),
                est.getFeatureSubsetStrategy(), est.getImpurity()) == (32, 5, 20, True, "auto", imp)
        cp = est.cuml_params
        assert (cp["n_bins"], cp["n_estimators"], cp["max_depth"], cp["bootstrap"], cp["max_features"],
                cp["split_criterion"], cp["n_streams"]) == (32, 20, 5, True, "auto", crit, 1)
        est = E(maxBins=17, maxDepth=9, numTrees=17, featureSubsetStrategy="onethird")
        assert (est.cuml_params["n_bins"], est.cuml_params["max_depth"], est.cuml_params["n_estimators"],
                est.cuml_params["max_features"]) == (17, 9, 17, 1 / 3.0)
    assert RandomForestClassifier(impurity="entropy").cuml_params["split_criterion"] == "entropy"


@pytest.mark.parametrize("spark, cuml", [
    ({"maxDepth": 51}, {"max_depth": 51}), ({"maxBins": 61}, {"n_bins": 61}),
    ({"minInstancesPerNode": 63}, {"min_samples_leaf": 63}), ({"numTrees": 56}, {"n_estimators": 56}),
    ({"featureSubsetStrategy": "onethird"}, {"max_features": 1.0 / 3.0}), ({"seed": 21}, {"random_state": 21}),
    ({"bootstrap": False}, {"bootstrap": False}), ({"n_streams": 2}, {"n_streams": 2}),
    ({"min_samples_split": 19}, {"min_samples_split": 19}), ({"max_samples": 0.77}, {"max_samples": 0.77}),
    ({"max_leaves": 72}, {"max_leaves": 72}), ({"min_impurity_decrease": 0.03}, {"min_impurity_decrease": 0.03}),
    ({"max_batch_size": 1025}, {"max_batch_size": 1025}), ({"verbose": True}, {"verbose": True})])
def test_rf_copy(spark, cuml):
    from spark_rapids_ml_b200.classification import RandomForestClassifier
    from spark_rapids_ml_b200.regression import RandomForestRegressor

    for E in (RandomForestClassifier, RandomForestRegressor):
        est = E(**spark)
        for k, v in cuml.items():
            assert est.cuml_params[k] == v
        base = E()
        params = {base.getParam(k): v for k, v in spark.items() if base.hasParam(k)}
        if params:
            c = base.copy(params)
            for k, v in cuml.items():
                assert c.cuml_params[k] == v
            assert base.cuml_params == E().cuml_params


@pytest.mark.parametrize("kw, msg", [
    ({"maxDepth": -1}, "maxDepth given invalid value -1"), ({"maxBins": -1}, "maxBins given invalid value -1"),
    ({"maxBins": 300}, "maxBins given invalid value 300"), ({"maxDepth": 17}, "maxDepth given invalid value 17"),
    ({"numTrees": 0}, "numTrees given invalid value 0"), ({"featureSubsetStrategy": "bogus"}, "featureSubsetStrategy"),
    ({"impurity": "variance"}, "impurity given invalid value")])
def test_validation_messages(kw, msg):
    from spark_rapids_ml_b200.classification import RandomForestClassifier

    with pytest.raises(ValueError, match=msg):
        RandomForestClassifier(**kw)._validate_parameters()


def test_unsupported_params():
    from spark_rapids_ml_b200.classification import RandomForestClassifier
    from spark_rapids_ml_b200.regression import RandomForestRegressor

    for E in (RandomForestClassifier, RandomForestRegressor):
        with pytest.raises(ValueError, match="'weightCol' is not supported"):
            E().setWeightCol("w")
        with pytest.raises(ValueError, match="'leafCol' is not supported"):
            E().setLeafCol("leaf")
        with pytest.raises(ValueError, match="'weightCol' is not supported"):
            E(weightCol="w")
        with pytest.raises(ValueError, match="32-bit"):
            E().setSeed(2 ** 40)


def test_features_cols_and_spark_confs():
    from spark_rapids_ml_b200.classification import RandomForestClassifier
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    est = RandomForestClassifier().setFeaturesCols(["a", "b"])
    assert est.getFeaturesCol() == ["a", "b"] and est._get_input_columns() == (None, ["a", "b"])
    assert RandomForestClassifier(featuresCol=["a", "b"]).getFeaturesCol() == ["a", "b"]
    sess = LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()
    sess.conf.set("spark.rapids.ml.num_workers", "3")
    sess.conf.set("spark.rapids.ml.verbose", "5")
    try:
        est = RandomForestClassifier()
        assert est._input_kwargs["num_workers"] == 3 and est._input_kwargs["verbose"] == 5
        assert RandomForestClassifier(num_workers=2)._num_workers == 2
    finally:
        for k in ("num_workers", "verbose"):
            sess.conf.unset(f"spark.rapids.ml.{k}")


def test_estimator_persistence(tmp_path):
    from spark_rapids_ml_b200.regression import RandomForestRegressor

    est = RandomForestRegressor(maxBins=17, maxDepth=9, numTrees=17, featureSubsetStrategy="onethird", seed=4)
    est.write().overwrite().save(str(tmp_path / "est"))
    e2 = RandomForestRegressor.load(str(tmp_path / "est"))
    assert e2.cuml_params == est.cuml_params and e2.getMaxDepth() == 9 and e2.getSeed() == 4


def test_model_json_round_trip_and_persistence(tmp_path):
    from spark_rapids_ml_b200.classification import RandomForestClassificationModel
    from spark_rapids_ml_b200.tree import forest_to_json, json_to_forest

    X, y = _tree_data(500, 4, 1, "gini")
    F = ro.fit(X, y, n_trees=3, max_depth=4, max_bins=16, features_per_node=2, seed=2)
    text = forest_to_json(F, True)
    G = json_to_forest(text, F["n_values"])
    for k in ("tree_offsets", "feature", "children", "count"):
        np.testing.assert_array_equal(G[k], F[k])
    np.testing.assert_array_equal(G["threshold"].view(np.uint32), F["threshold"].view(np.uint32))
    leaf = F["feature"] < 0
    np.testing.assert_array_equal(G["value"][leaf], F["value"][leaf])
    np.testing.assert_array_equal(G["gain"], F["gain"])
    m = RandomForestClassificationModel(n_cols=4, dtype="float32", model_json=text, num_classes=F["n_values"])
    assert m.getNumTrees == 3 and m.totalNumNodes == F["tree_offsets"][-1] and m.treeWeights == [1.0] * 3
    np.testing.assert_array_equal(np.asarray(m.featureImportances), ro.feature_importances(F, 4))
    m.write().overwrite().save(str(tmp_path / "m"))
    m2 = RandomForestClassificationModel.load(str(tmp_path / "m"))
    assert m2._model_json == text and m2.numClasses == F["n_values"] and m2.numFeatures == 4
    assert not os.path.exists(os.path.join(str(tmp_path / "m"), "data", "treelite_model"))
    assert "treelite_model" not in json.loads(open(tmp_path / "m" / "data" / "part-00000").read())


def test_reference_layout_model_loads():
    from spark_rapids_ml_b200.classification import RandomForestClassificationModel
    from spark_rapids_ml_b200.tree import json_to_forest

    m = RandomForestClassificationModel.load(os.path.join(HERE, "golden", "rf_reference_model"))
    assert m.numClasses == 2 and m.numFeatures == 2 and m.getNumTrees == 1 and m.totalNumNodes == 5
    f = m._flat()
    assert f["threshold"][0] == np.nextafter(np.float32(1.0), np.float32(0.0))   # "<" 1.0 read as "<=" below it
    assert f["threshold"][2] == np.float32(2.0) and f["children"][0].tolist() == [1, 2]
    lf = ro.leaves(np.array([[0.5, 2.0], [1.0, 2.0], [1.0, 3.0]], dtype=np.float32), f)[:, 0]
    assert lf.tolist() == [1, 3, 4]
    bad = json.dumps({"trees": [{"num_nodes": 1, "nodes": [{"node_id": 0, "split_feature_id": 0, "comparison_op": ">",
                                                            "threshold": 1.0, "left_child": 1, "right_child": 2}]}]})
    with pytest.raises(ValueError, match="unsupported comparison_op"):
        json_to_forest(bad, 2)


def test_unsupported_model_calls():
    from spark_rapids_ml_b200.regression import RandomForestRegressionModel

    m = RandomForestRegressionModel(n_cols=1, dtype="float32",
                                    model_json=json.dumps({"trees": [{"num_nodes": 1, "nodes": [
                                        {"node_id": 0, "leaf_value": 2.0, "instance_count": 3}]}]}))
    assert m.getNumTrees == 1 and np.asarray(m.featureImportances).tolist() == [0.0]
    for call in (m.cpu, lambda: m.trees, lambda: m.toDebugString, lambda: m.predict([1.0]),
                 lambda: m.predictLeaf([1.0])):
        with pytest.raises(NotImplementedError):
            call()
