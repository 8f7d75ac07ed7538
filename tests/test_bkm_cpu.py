"""BisectingKMeans without a GPU: the fp64 oracle's own rules (minSize, the choice of the dividing nodes, `need`
dropping past an empty child, depth-first leaf order, predict by descent rather than by the nearest leaf), the
hand-derived known answers of tests/golden/bkm_known_answers.json, and the estimator / model surface (params,
defaults, validation, copy, persistence)."""
import json
import os

import numpy as np
import pytest

import bkm_oracle as bo
from spark_rapids_ml_b200.clustering import BisectingKMeans, BisectingKMeansModel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bkm_known_answers.json")


def test_min_size_rule():
    assert bo.min_size(1.0, 1000) == 1
    assert bo.min_size(2.5, 1000) == 3
    assert bo.min_size(0.5, 7) == 4          # ceil(3.5)
    assert bo.min_size(0.01, 1000) == 10
    assert bo.min_size(0.001, 10) == 1       # ceil(0.01)


def test_choose_keeps_the_largest_ties_to_the_lower_index():
    div = [(5, 10), (2, 30), (7, 30), (4, 10), (6, 20)]
    assert bo.choose(div, 10) == [2, 4, 5, 6, 7]
    assert bo.choose(div, 2) == [2, 7]
    assert bo.choose(div, 3) == [2, 6, 7]
    assert bo.choose(div, 4) == [2, 4, 6, 7]   # 4 and 5 tie at n = 10: the lower index wins


def test_need_drops_even_when_a_child_is_empty():
    # symmetric about the origin: every split sends all rows left, so each level adds one node and uses up one of need
    X = np.array([[1, 2], [-1, -2], [3, -1], [-3, 1]], dtype=np.float32)
    r = bo.fit(X, 3, max_iter=4)
    assert r["levels"] == [[1], [2]]
    assert sorted(r["nodes"]) == [1, 2, 4] and r["leaves"] == [4]
    assert r["nodes"][4][0] == 4


def test_split_noise_is_counter_based():
    u = bo.split_noise(7, 3, 5)
    assert u.shape == (5,) and np.all((u >= 0) & (u < 1))
    np.testing.assert_array_equal(u[:3], bo.split_noise(7, 3, 3))
    assert not np.array_equal(u, bo.split_noise(7, 2, 5)) and not np.array_equal(u, bo.split_noise(8, 3, 5))


def test_depth_first_leaf_order():
    c = np.zeros(2)
    nodes = {i: (1, c, 0.0) for i in (1, 2, 3, 6, 7, 12, 13)}
    assert bo.dfs(nodes) == [1, 2, 3, 6, 12, 13, 7]
    assert bo.leaves(nodes) == [2, 12, 13, 7]


def test_predict_descends_rather_than_taking_the_nearest_leaf():
    nodes = {1: (4, np.array([0.0, 0.0]), 1.0), 2: (2, np.array([-1.0, 0.0]), 0.0), 3: (2, np.array([1.0, 0.0]), 1.0),
             6: (1, np.array([-0.5, 0.0]), 0.0), 7: (1, np.array([2.0, 0.0]), 0.0)}
    x = np.array([[-0.5, 0.0], [1.75, 0.0]], dtype=np.float32)
    lab, cost = bo.predict(x, nodes)
    # (-0.5, 0) sits on leaf 6's centre, but the root sends it to node 2 (0.25 < 2.25), a leaf
    assert list(lab) == [0, 2]
    np.testing.assert_allclose(cost, [0.25, 0.0625])
    nearest = np.argmin([((x[0] - nodes[i][1]) ** 2).sum() for i in bo.leaves(nodes)])
    assert nearest == 1


def test_cost_about_the_parent_centre_survives_an_offset():
    rng = np.random.default_rng(0)
    X = (1e3 + rng.normal(size=(200, 3))).astype(np.float32)
    n, c, cost = bo.summarize(X.astype(np.float64), np.full(3, 1e3))
    D = X.astype(np.float64) - X.astype(np.float64).mean(axis=0)
    assert n == 200
    np.testing.assert_allclose(cost, (D * D).sum(), rtol=1e-12)


@pytest.mark.parametrize("case", json.load(open(GOLDEN)), ids=lambda c: c["name"])
def test_known_answers(case):
    X = np.asarray(case["X"], dtype=np.float32)
    r = bo.fit(X, case["k"], case["max_iter"], case["min_divisible"], seed=11)
    nodes = r["nodes"]
    order = bo.dfs(nodes)
    assert order == case["node_index"]
    assert [nodes[i][0] for i in order] == case["sizes"]
    np.testing.assert_allclose([nodes[i][1] for i in order], case["centers"], atol=1e-12)
    np.testing.assert_allclose([nodes[i][2] for i in order], case["costs"], atol=1e-12)
    assert bo.training_cost(nodes) == pytest.approx(case["training_cost"], abs=1e-12)
    lab, _ = bo.predict(X, nodes)
    assert list(lab) == case["labels"]
    assert list(np.bincount(lab, minlength=len(r["leaves"]))) == case["cluster_sizes"]


def test_params_defaults_and_setters():
    est = BisectingKMeans()
    assert est.getK() == 4 and est.getMaxIter() == 20 and est.getMinDivisibleClusterSize() == 1.0
    assert est.getDistanceMeasure() == "euclidean" and est.getPredictionCol() == "prediction"
    assert est.getFeaturesCol() == "features"
    assert est.getSeed() == hash("BisectingKMeans") & 0x07FFFFFFF
    est = BisectingKMeans(k=5, maxIter=7, seed=3, minDivisibleClusterSize=0.25, featuresCol=["a", "b"])
    assert est.cuml_params["n_clusters"] == 5 and est.cuml_params["max_iter"] == 7
    assert est.cuml_params["random_state"] == 3 and est.cuml_params["min_divisible_cluster_size"] == 0.25
    assert est.getFeaturesCol() == ["a", "b"]
    est.setK(6).setMaxIter(3).setSeed(9).setMinDivisibleClusterSize(4.0).setDistanceMeasure("euclidean")
    assert (est.getK(), est.getMaxIter(), est.getSeed(), est.getMinDivisibleClusterSize()) == (6, 3, 9, 4.0)
    c = est.copy({est.k: 8})
    assert c.getK() == 8 and c.cuml_params["n_clusters"] == 8 and est.getK() == 6


@pytest.mark.parametrize("kw,msg", [({"k": 1}, "k given invalid"), ({"maxIter": 0}, "maxIter given invalid"),
                                    ({"minDivisibleClusterSize": 0.0}, "minDivisibleClusterSize given invalid"),
                                    ({"minDivisibleClusterSize": -2.0}, "minDivisibleClusterSize given invalid")])
def test_validation_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        BisectingKMeans(**kw)._validate_parameters()


def test_unsupported_params_raise():
    with pytest.raises(ValueError, match="weightCol"):
        BisectingKMeans(weightCol="w")
    with pytest.raises(ValueError, match="weightCol"):
        BisectingKMeans().setWeightCol("w")
    with pytest.raises(ValueError, match="cosine"):
        BisectingKMeans(distanceMeasure="cosine")
    with pytest.raises(ValueError, match="cosine"):
        BisectingKMeans().setDistanceMeasure("cosine")


def _model():
    return BisectingKMeansModel(node_index_=[1, 2, 3, 6, 7], node_centers_=[[0.0, 0.0], [-1.0, 0.0], [1.0, 0.0],
                                                                          [0.5, 0.0], [2.0, 0.0]],
                                node_sizes_=[6, 2, 4, 3, 1], node_costs_=[9.0, 0.5, 3.0, 1.0, 0.0],
                                cluster_sizes_=[2, 3, 1], training_cost_=1.5, num_iters=20, n_cols=2, dtype="float32")


def test_model_surface_and_persistence(tmp_path):
    m = _model()
    assert m.hasSummary and m.getK() == 3
    np.testing.assert_array_equal(np.stack(m.clusterCenters()), [[-1.0, 0.0], [0.5, 0.0], [2.0, 0.0]])
    s = m.summary
    assert (s.k, s.numIter, s.clusterSizes, s.trainingCost) == (3, 20, [2, 3, 1], 1.5)
    assert m._transform_outputs() == [("prediction", "int")]
    for f in (lambda: m.predict([0.0, 0.0]), m.cpu):
        with pytest.raises(NotImplementedError):
            f()
    m.setPredictionCol("leaf")
    m.write().overwrite().save(str(tmp_path / "model"))
    m2 = BisectingKMeansModel.load(str(tmp_path / "model"))
    assert m2.node_index_ == m.node_index_ and m2.node_centers_ == m.node_centers_
    assert m2.node_sizes_ == m.node_sizes_ and m2.node_costs_ == m.node_costs_
    assert m2.summary.clusterSizes == [2, 3, 1] and m2.summary.trainingCost == 1.5
    assert m2.getPredictionCol() == "leaf" and m2.getK() == 3
    est = BisectingKMeans(k=3, minDivisibleClusterSize=0.5)
    est.save(str(tmp_path / "est"))
    e2 = BisectingKMeans.load(str(tmp_path / "est"))
    assert e2.getK() == 3 and e2.getMinDivisibleClusterSize() == 0.5 and e2.cuml_params["n_clusters"] == 3
