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


def _offset_data(n, nq, d, offset, seed=3):
    rng = np.random.default_rng(seed)
    return ((rng.normal(size=(n, d)) + offset).astype(np.float32),
            (rng.normal(size=(nq, d)) + offset).astype(np.float32))


def _answer(X, Q, ids):
    """(dist float32, ids) of the given rows per query, ordered as the device reports them."""
    e = ((Q.astype(np.float64)[:, None, :] - X.astype(np.float64)[ids]) ** 2).sum(-1)
    o = np.stack([np.lexsort((ids[i], e[i])) for i in range(e.shape[0])])
    return np.sqrt(np.take_along_axis(e, o, 1)).astype(np.float32), np.take_along_axis(ids, o, 1)


def _displaced(X, Q, k):
    """The oracle's answer with its third neighbour replaced by the (k + 3)-th nearest item."""
    _, I = ko.knn(X, Q, k + 3)
    wrong = I[:, :k].copy()
    wrong[:, 2] = I[:, k + 2]
    return _answer(X, Q, wrong)


def _old_rule_flags(X, Q, k, idx):
    """Queries the tolerance 1e-6 (||q||^2 + max ||x||^2) would flag, set and id clauses."""
    X64, Q64 = X.astype(np.float64), Q.astype(np.float64)
    D0, I0 = ko.knn(X, Q, k)
    t = 1e-6 * ((Q64 * Q64).sum(1) + (X64 * X64).sum(1).max())
    n = 0
    for i in range(Q.shape[0]):
        e = ((Q64[i] - X64[idx[i]]) ** 2).sum(1)
        eo = ((Q64[i] - X64[I0[i]]) ** 2).sum(1)
        n += bool(np.any(np.abs(np.sort(e) - D0[i]) > t[i]) or np.any(np.abs(e - eo) > t[i]))
    return n


def test_tau_is_translation_invariant():
    X, Q = _offset_data(2000, 64, 128, 0.0)
    X1, Q1 = (X + np.float32(1e3)), (Q + np.float32(1e3))
    np.testing.assert_allclose(ko.tau(X1, Q1), ko.tau(X, Q), rtol=1e-3)
    assert 4e-6 >= ko.TAU_C >= 1e-6
    for k in (8, 64):
        counts = []
        for A, B in ((X, Q), (X1, Q1)):
            D, I = ko.knn(A, B, k)
            right = ko.compare(A, B, k, np.sqrt(D).astype(np.float32), I)
            wrong = ko.compare(A, B, k, *_displaced(A, B, k))
            counts.append((right, {c: wrong[c] for c in ("n_outside_margin", "n_set", "n_dup", "n_order", "n_dist")}))
        assert counts[0] == counts[1]
        assert counts[0][0]["n_outside_margin"] == 0 and counts[0][1]["n_outside_margin"] == Q.shape[0]


def test_rule_is_not_vacuous_far_from_origin():
    # d = 128 at an offset of 1e3: the true squared distances of the nearest items are ~150-200 and about 1 apart, while
    # 1e-6 (||q||^2 + max ||x||^2) is ~260: that tolerance passes the wrong answer, the translation-invariant one flags it
    X, Q = _offset_data(2000, 64, 128, 1e3)
    dist, idx = _displaced(X, Q, 8)
    assert ko.compare(X, Q, 8, dist, idx)["n_outside_margin"] == Q.shape[0]
    assert _old_rule_flags(X, Q, 8, idx) == 0


def _screen_search(X, Q, k, shift):
    """The wgmma pass on the CPU: the k best by (emulated screen, row), reported by exact distance then row."""
    S = ko.screen_emulation(X, Q, shift)
    rows = np.arange(X.shape[0])
    sel = np.stack([np.lexsort((rows, S[i]))[:k] for i in range(Q.shape[0])])
    return _answer(X, Q, sel)


def test_screen_emulation_calibrates_the_rule():
    # unshifted, the fp32 screen loses neighbours at an offset of 100; screened in the frame of item row 0 it meets the
    # rule at every offset
    k = 8
    X, Q = _offset_data(2000, 64, 128, 100.0)
    assert ko.compare(X, Q, k, *_screen_search(X, Q, k, None))["n_outside_margin"] > 0
    for offset in (0.0, 100.0, 1e3):
        X, Q = _offset_data(2000, 64, 128, offset)
        bad = ko.compare(X, Q, k, *_screen_search(X, Q, k, X[0]))
        assert bad["n_outside_margin"] == 0, (offset, bad)


def test_screen_emulation_matches_fp64_on_small_integers():
    # integer data: every product and partial sum of the screen is exact, so it equals ||x - s||^2 - 2 (q - s).(x - s)
    rng = np.random.default_rng(1)
    X = rng.integers(-3, 4, size=(300, 64)).astype(np.float32) + np.float32(1024)
    Q = rng.integers(-3, 4, size=(20, 64)).astype(np.float32) + np.float32(1024)
    a, b = (Q - X[0]).astype(np.float64), (X - X[0]).astype(np.float64)
    np.testing.assert_array_equal(ko.screen_emulation(X, Q, X[0]), (b * b).sum(1)[None, :] - 2 * a @ b.T)


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
