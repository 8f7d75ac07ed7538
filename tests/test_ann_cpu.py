"""ApproximateNearestNeighbors on the CPU: params, defaults, copy, the unsupported calls, and the fp64 IVF oracle (its
training-subset rule, its fill rule, and nprobe = nlist equal to the exact k-NN oracle)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import ann_oracle as ao
import knn_oracle as ko
from spark_rapids_ml_b200.knn import ApproximateNearestNeighbors, NearestNeighbors

HERE = os.path.dirname(os.path.abspath(__file__))


def test_defaults_and_params():
    a = ApproximateNearestNeighbors()
    assert a.cuml_params == {"n_neighbors": 5, "verbose": False, "algorithm": "ivfflat", "metric": "euclidean",
                             "algo_params": None}
    assert (a.getK(), a.getAlgorithm(), a.getMetric(), a.getAlgoParams()) == (5, "ivfflat", "euclidean", None)
    a = ApproximateNearestNeighbors(k=3, algoParams={"nlist": 2, "nprobe": 1}, metric="sqeuclidean")
    assert a.cuml_params["n_neighbors"] == 3 and a.cuml_params["algo_params"] == {"nlist": 2, "nprobe": 1}
    a.setK(7).setAlgoParams({"n_lists": 4}).setMetric("l2")
    assert a.cuml_params["n_neighbors"] == 7 and a.getAlgoParams() == {"n_lists": 4} and a.getMetric() == "l2"
    b = a.copy()
    assert b.cuml_params == a.cuml_params and b.getK() == 7
    b.setK(9)
    assert a.getK() == 7


@pytest.mark.parametrize("algo", ["ivfpq", "cagra", "brute"])
def test_unsupported_algorithms(algo):
    with pytest.raises(ValueError):
        ApproximateNearestNeighbors(algorithm=algo)
    with pytest.raises(ValueError):
        ApproximateNearestNeighbors().setAlgorithm(algo)


@pytest.mark.parametrize("metric", ["inner_product", "cosine"])
def test_unsupported_metrics(metric):
    with pytest.raises(ValueError, match=metric):
        ApproximateNearestNeighbors(metric=metric)
    with pytest.raises(ValueError, match=metric):
        ApproximateNearestNeighbors().setMetric(metric)


def test_algo_params_keys():
    a = ApproximateNearestNeighbors(algoParams={"n_lists": 8, "n_probes": 2, "kmeans_n_iters": 3})
    assert a._validate_ann() == {"nlist": 8, "nprobe": 2, "kmeans_n_iters": 3, "kmeans_trainset_fraction": 0.5}
    with pytest.raises(ValueError, match="pq_dim"):
        ApproximateNearestNeighbors(algoParams={"pq_dim": 4})._validate_ann()


def test_no_persistence_and_message():
    with pytest.raises(NotImplementedError):
        ApproximateNearestNeighbors().write()
    with pytest.raises(NotImplementedError):
        ApproximateNearestNeighbors.load("x")
    from spark_rapids_ml_b200.knn import NearestNeighborsModel
    with pytest.raises(NotImplementedError, match="ApproximateNearestNeighbors"):
        NearestNeighborsModel.approxNearestNeighbors(None)
    assert NearestNeighbors().cuml_params["n_neighbors"] == 5


def test_train_mask():
    m = ao.train_mask(10, 0.5)
    assert m.tolist() == [False, True] * 5
    assert ao.train_mask(7, 1.0).all()
    assert ao.train_mask(1000, 0.3).sum() == 300


def _known_answers():
    out = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_ann_known_answers.py")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    with open(os.path.join(HERE, "golden", "ann_known_answers.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", ["docstring", "return_fewer_k"])
def test_known_answers(case):
    ka = _known_answers()[case]
    X = np.array([r[1] for r in ka["items"]], np.float32)
    Q = np.array([r[1] for r in ka["queries"]], np.float32)
    ids = np.array([r[0] for r in ka["items"]], np.int64)
    for C in ka["centers"]:   # every centre set the training run can reach gives the same answer
        D, I, _, _ = ao.ivf(X, Q, ka["k"], np.array(C, np.float32), ka["algoParams"]["nprobe"], ids)
        assert I.tolist() == ka["indices"]
        np.testing.assert_allclose(np.sqrt(D), ka["distances"], rtol=1e-6)
    if case == "docstring":   # the training subset of the docstring's six items
        assert ao.train_mask(6, 0.5).tolist() == [False, True, False, True, False, True]


def test_fewer_than_k_fill():
    X = np.array([[0, 0], [1, 0], [10, 0]], np.float32)
    Q = np.array([[0.1, 0], [10, 0], [np.nan, 0]], np.float32)
    C = np.array([[0, 0], [10, 0]], np.float32)
    D, I, _, _ = ao.ivf(X, Q, 3, C, 1)
    assert I[0].tolist() == [0, 1, 0] and np.isinf(D[0, 2])
    assert I[1].tolist() == [2, 2, 2] and np.isinf(D[1, 1:]).all()
    assert (I[2] == ao.INT64_MAX).all() and np.isinf(D[2]).all()


def test_all_lists_probed_is_exact():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(300, 5)).astype(np.float32)
    Q = rng.normal(size=(20, 5)).astype(np.float32)
    D, I, _, _ = ao.ivf(X, Q, 7, X[:6], 6)
    D0, I0 = ko.knn(X, Q, 7)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_allclose(D, D0)
