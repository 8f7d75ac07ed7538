"""ALS without a GPU: Spark's param defaults and setters, the id, rating and param errors with their messages, the
start rule, the fp64 oracle against hand-derived known answers (tests/golden/make_als_known_answers.py), the oracle's
prediction and top-n rules, the persistence layout and a round trip, and the cold-start settings."""
import json
import os

import numpy as np
import pyarrow as pa
import pytest

import als_oracle as ao
from spark_rapids_ml_b200.recommendation import ALS, ALSModel, _id_values

HERE = os.path.dirname(os.path.abspath(__file__))


def test_defaults_and_setters():
    a = ALS()
    assert (a.getRank(), a.getMaxIter(), a.getRegParam(), a.getImplicitPrefs(), a.getAlpha()) == (10, 10, 0.1, False, 1.0)
    assert (a.getUserCol(), a.getItemCol(), a.getRatingCol(), a.getPredictionCol()) == ("user", "item", "rating",
                                                                                         "prediction")
    assert a.getColdStartStrategy() == "nan" and a.getNonnegative() is False
    assert (a.getNumUserBlocks(), a.getNumItemBlocks(), a.getCheckpointInterval(), a.getBlockSize()) == (10, 10, 10, 4096)
    assert a.getIntermediateStorageLevel() == a.getFinalStorageLevel() == "MEMORY_AND_DISK"
    assert a.getSeed() == ALS().getSeed() and 0 <= a.getSeed() < 2 ** 31
    a.setRank(64).setMaxIter(3).setRegParam(0.5).setImplicitPrefs(True).setAlpha(40.0).setUserCol("u").setItemCol("i")
    a.setRatingCol("").setColdStartStrategy("DROP").setSeed(7).setNumUserBlocks(4).setBlockSize(128)
    assert (a.getRank(), a.getMaxIter(), a.getRegParam(), a.getImplicitPrefs(), a.getAlpha()) == (64, 3, 0.5, True, 40.0)
    assert (a.getUserCol(), a.getItemCol(), a.getRatingCol(), a.getColdStartStrategy(), a.getSeed()) == ("u", "i", "",
                                                                                                        "drop", 7)
    assert ALS(rank=3, coldStartStrategy="drop").getRank() == 3


@pytest.mark.parametrize("kw,msg", [({"rank": 0}, "rank given invalid value"), ({"maxIter": -1}, "maxIter given"),
                                    ({"regParam": -0.1}, "regParam given"), ({"alpha": -1.0}, "alpha given"),
                                    ({"coldStartStrategy": "zero"}, "coldStartStrategy must be one of nan, drop")])
def test_param_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        ALS(**kw)


@pytest.mark.parametrize("vals,shown", [([1.0, 2.5], "2.5"), ([2.0 ** 31], "2147483648.0"), ([-(2.0 ** 31) - 1],
                                                                                           "-2147483649.0"),
                                        ([np.nan], "NaN")])
def test_id_errors_name_column_and_value(vals, shown):
    t = pa.table({"uid": pa.array(vals, type=pa.float64())})
    msg = (f"ALS only supports values in Integer range and without fractional part for column uid. Value {shown} was "
           "either out of Integer range or contained a fractional part that could not be converted.")
    with pytest.raises(ValueError) as e:
        _id_values(t, "uid")
    assert str(e.value) == msg
    assert ao.check_ids(vals, "uid") == msg


def test_id_rules_accept_int32_edges_and_reject_null_and_strings():
    t = pa.table({"a": pa.array([-(2 ** 31), 2 ** 31 - 1, 0], type=pa.int64()), "b": pa.array([1, None], type=pa.int32())
                  if False else pa.array([1, None, 2], type=pa.int32()), "c": pa.array(["x", "y", "z"])})
    np.testing.assert_array_equal(_id_values(t, "a"), [-(2 ** 31), 2 ** 31 - 1, 0])
    with pytest.raises(ValueError, match="Value null was"):
        _id_values(t, "b")
    with pytest.raises(TypeError, match="must be of type numeric"):
        _id_values(t, "c")


def test_start_rule():
    ids = np.array([-5, 0, 7, 2 ** 31 - 1])
    F = ao.start(ids, 10, 42)
    assert F.dtype == np.float32 and F.shape == (4, 10)
    np.testing.assert_allclose(np.linalg.norm(F.astype(np.float64), axis=1), 1.0, atol=1e-6)
    # keyed by the raw id, not its position, and by the seed
    np.testing.assert_array_equal(ao.start(ids[::-1], 10, 42), F[::-1])
    np.testing.assert_array_equal(ao.start(ids[:1], 10, 42)[0], F[0])
    assert not np.array_equal(ao.start(ids, 10, 43), F)
    # rank 1: the sign of one normal
    assert set(np.abs(ao.start(np.arange(50), 1, 0)).ravel().tolist()) == {1.0}
    # splitmix64 of 0 (the published first output of the generator seeded with 0)
    assert int(ao.splitmix64(np.uint64(0))) == 0xE220A8397B1DCDAF


def test_oracle_known_answers():
    with open(os.path.join(HERE, "golden", "als_known_answers.json")) as f:
        cases = json.load(f)
    for name, c in cases.items():
        m, k = c["m"], c["k"]
        u = np.repeat(np.arange(m), k).astype(np.float64)
        i = np.tile(np.arange(k), m).astype(np.float64)
        r = np.full(m * k, c["c"], dtype=np.float32)
        out = ao.fit(u, i, r, 1, c["iters"], c["reg"], c["implicit"], c["alpha"], init=np.ones((m, 1), np.float32))
        np.testing.assert_allclose(out["item_factors"], c["item"], rtol=2e-7, err_msg=name)
        np.testing.assert_allclose(out["user_factors"], c["user"], rtol=2e-7, err_msg=name)


def test_oracle_implicit_negative_ratings_and_duplicates():
    # a negative implicit rating adds confidence to A but nothing to b; a duplicate pair counts twice
    Y = np.array([[1.0, 0.0], [0.0, 2.0]], dtype=np.float32)
    x, _ = ao.half_step(np.array([0, 0, 0]), np.array([0, 1, 1]), np.array([2.0, -1.0, -1.0]), Y, 1, 0.1, True, 1.0)
    A = Y.T.astype(np.float64) @ Y + 2.0 * np.outer(Y[0], Y[0]) + 2 * 1.0 * np.outer(Y[1], Y[1]) + 0.1 * 1 * np.eye(2)
    b = 3.0 * Y[0]
    np.testing.assert_allclose(x[0], np.linalg.solve(A, b).astype(np.float32), rtol=1e-7)
    with pytest.raises(np.linalg.LinAlgError):   # regParam 0, one rating, rank 2: not positive definite
        ao.half_step(np.array([0]), np.array([0]), np.array([1.0]), Y, 1, 0.0)


def test_oracle_prediction_and_topn_rules():
    rng = np.random.default_rng(0)
    U = rng.normal(size=(4, 5)).astype(np.float32)
    T = np.concatenate([rng.normal(size=(6, 5)), rng.normal(size=(1, 5))]).astype(np.float32)
    T[6] = T[2]   # a tie: row 2 must come before row 6
    s = ao.predict(U[[0, 1]], T[[2, 3]])
    ref = np.float32(0)
    for j in range(5):
        ref = np.float32(ref + np.float32(U[0, j] * T[2, j]))
    assert s[0] == ref
    idx, sc = ao.recommend(U, T, 7)
    for q in range(4):
        assert list(idx[q]).index(2) < list(idx[q]).index(6)
        assert np.all(np.diff(sc[q].astype(np.float64)) <= 0)
    assert ao.recommend(U, T, 100)[0].shape == (4, 7)


def test_persistence_layout_and_round_trip(tmp_path):
    import pyarrow.parquet as pq

    m = ALSModel(2, np.array([3, 9], np.int32), np.arange(4, dtype=np.float32), np.array([-1], np.int32),
                 np.array([0.5, -0.5], np.float32))
    m.setUserCol("u").setColdStartStrategy("drop")
    p = str(tmp_path / "als")
    m.write().save(p)
    meta = json.loads(open(os.path.join(p, "metadata", "part-00000")).read())
    assert meta["rank"] == 2 and meta["paramMap"]["userCol"] == "u"
    t = pq.read_table(os.path.join(p, "userFactors"))
    assert t.schema.field("id").type == pa.int32() and t.schema.field("features").type == pa.list_(pa.float32())
    assert t.column("id").to_pylist() == [3, 9] and t.column("features").to_pylist() == [[0.0, 1.0], [2.0, 3.0]]
    assert pq.read_table(os.path.join(p, "itemFactors")).column("features").to_pylist() == [[0.5, -0.5]]
    with pytest.raises(IOError):
        m.write().save(p)
    m2 = ALSModel.load(p)
    assert m2.rank == 2 and m2.getUserCol() == "u" and m2.getColdStartStrategy() == "drop"
    np.testing.assert_array_equal(m2._uf, m._uf)
    np.testing.assert_array_equal(m2._iid_, m._iid_)
    assert m2.userFactors.toPandas()["id"].tolist() == [3, 9]


def test_cold_start_settings():
    m = ALSModel(1, np.array([1], np.int32), np.ones(1, np.float32), np.array([1], np.int32), np.ones(1, np.float32))
    assert m.getColdStartStrategy() == "nan"
    assert m.setColdStartStrategy("Drop").getColdStartStrategy() == "drop"
    with pytest.raises(ValueError, match="coldStartStrategy"):
        m.setColdStartStrategy("ignore")
