"""NearestNeighbors surface without a GPU: params and defaults, id columns, unsupported operations, the LocalDataFrame
operations kneighbors' plan uses, the fp64 oracle against scikit-learn, and the known-answer fixture."""
import json
import logging
import os
import subprocess
import sys

import numpy as np
import pytest

import knn_oracle as ko
from spark_rapids_ml_b200.knn import NearestNeighbors, NearestNeighborsModel
from spark_rapids_ml_b200.sparkshim.sql import LocalSession

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture
def spark():
    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "2"})


def test_params_and_defaults(spark):
    est = NearestNeighbors()
    assert est.getK() == 5 and est.cuml_params == {"n_neighbors": 5, "verbose": False, "batch_size": 2000000}
    assert est.getIdCol() is None
    est = NearestNeighbors(k=3, inputCol=["a", "b"], idCol="id", num_workers=1)
    assert est.getK() == 3 and est.cuml_params["n_neighbors"] == 3 and est.getInputCol() == ["a", "b"]
    assert est.getIdCol() == "id" and est.num_workers == 1
    est.setK(7).setInputCol("features")
    assert est.getK() == 7 and est.cuml_params["n_neighbors"] == 7 and est.getInputCol() in ("features", ["a", "b"])
    c = est.copy()
    assert c.getK() == 7 and c.cuml_params["n_neighbors"] == 7 and c.uid == est.uid


def test_float32_inputs_warning(caplog):
    with caplog.at_level(logging.WARNING):
        NearestNeighbors(float32_inputs=False)
    assert "does not support double precision" in caplog.text


@pytest.mark.parametrize("k", [0, -1])
def test_k_validation(spark, k):
    df = spark.createDataFrame([([1.0, 1.0],)], "features array<float>")
    with pytest.raises(ValueError):
        NearestNeighbors(k=k).setInputCol("features").fit(df)


def test_id_columns(spark):
    df = spark.createDataFrame([([1.0, 1.0], 5), ([2.0, 2.0], 6)], "features array<float>, unique_id long")
    with pytest.raises(ValueError, match="unique_id"):
        NearestNeighbors().setInputCol("features").fit(df)
    df = spark.createDataFrame([([float(i), 0.0],) for i in range(5)], "features array<float>", num_partitions=2)
    model = NearestNeighbors().setInputCol("features").fit(df)
    assert isinstance(model, NearestNeighborsModel)
    assert model._item_df_withid.columns == ["unique_id", "features"]
    ids = [r["unique_id"] for r in model._item_df_withid.collect()]
    assert ids == [0, 1, (1 << 33), (1 << 33) + 1, (1 << 33) + 2]
    df = spark.createDataFrame([(10, [1.0, 1.0])], "id int, features array<float>")
    m2 = NearestNeighbors().setInputCol("features").setIdCol("id").fit(df)
    assert m2._item_df_withid.columns == ["id", "features"]
    assert m2._processed_item_df.columns == ["id", "features", "cuml_label"]


def test_unsupported(spark, tmp_path):
    est = NearestNeighbors().setInputCol("features")
    for call in (lambda: est.save(str(tmp_path / "e")), est.write, NearestNeighbors.read,
                 lambda: NearestNeighbors.load(str(tmp_path / "e"))):
        with pytest.raises(NotImplementedError):
            call()
    df = spark.createDataFrame([([1.0, 1.0],)], "features array<float>")
    model = est.fit(df)
    for call in (lambda: model.save(str(tmp_path / "m")), model.write, NearestNeighborsModel.read,
                 lambda: NearestNeighborsModel.load(str(tmp_path / "m")), lambda: model.transform(df),
                 lambda: model.exactNearestNeighborsJoin(df), model.approxNearestNeighbors):
        with pytest.raises(NotImplementedError):
            call()


def test_local_frame_operations(spark):
    a = spark.createDataFrame([(1, [1.0]), (2, [2.0]), (3, [3.0])], "id long, f array<float>", num_partitions=2)
    b = spark.createDataFrame([(4, [4.0])], "key long, g array<float>")
    u = a.union(b)
    assert u.columns == ["id", "f"] and u.getNumPartitions() == 3
    assert [r["id"] for r in u.collect()] == [1, 2, 3, 4]
    with pytest.raises(ValueError):
        a.union(spark.createDataFrame([(4,)], "id long"))
    with pytest.raises(ValueError):
        a.union(spark.createDataFrame([(4, [4.0])], "id int, f array<float>"))
    c = a.with_constant_column("lab", 1)
    assert c.dtypes[-1] == ("lab", "int") and [r["lab"] for r in c.collect()] == [1, 1, 1]
    m = a.with_monotonically_increasing_id("mid")
    assert m.columns == ["mid", "id", "f"] and [r["mid"] for r in m.collect()] == [0, 1 << 33, (1 << 33) + 1]
    empty = spark.createDataFrame([], "features array<float>")
    assert empty.columns == ["features"] and empty.count() == 0


def test_oracle_matches_sklearn():
    neighbors = pytest.importorskip("sklearn.neighbors")
    rng = np.random.default_rng(0)
    for d in (2, 20):
        X = rng.normal(size=(500, d)).astype(np.float32)
        Q = rng.normal(size=(40, d)).astype(np.float32)
        D, I = ko.knn(X, Q, 7)
        sd, si = neighbors.NearestNeighbors(n_neighbors=7).fit(X.astype(np.float64)).kneighbors(Q.astype(np.float64))
        np.testing.assert_allclose(np.sqrt(D), sd, rtol=1e-10)
        np.testing.assert_array_equal(I, si)
        assert ko.compare(X, Q, 7, np.sqrt(D).astype(np.float32), I)["n_outside_margin"] == 0
        wrong = I.copy()
        wrong[:, [0, 6]] = wrong[:, [6, 0]]
        assert ko.compare(X, Q, 7, np.sqrt(D).astype(np.float32), wrong)["n_outside_margin"] == Q.shape[0]


def test_oracle_ties_to_lowest_row():
    X = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [1.0, 0.0]], np.float32)
    D, I = ko.knn(X, np.zeros((1, 2), np.float32), 4)
    assert I[0].tolist() == [0, 1, 2, 3] and D[0].tolist() == [1.0, 1.0, 1.0, 1.0]


def test_known_answers_fixture():
    out = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_knn_known_answers.py")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    with open(os.path.join(HERE, "golden", "knn_known_answers.json")) as f:
        ka = json.load(f)
    X = np.array([r[0] for r in ka["items"]], np.float32)
    Q = np.array([r[0] for r in ka["queries"]], np.float32)
    D, I = ko.knn(X, Q, ka["k"])
    assert I.tolist() == ka["indices"]
    np.testing.assert_allclose(np.sqrt(D), ka["distances"], rtol=1e-6)
