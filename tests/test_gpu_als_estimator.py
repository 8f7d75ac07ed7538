"""ALS / ALSModel end to end on a local frame over several partitions: fit, transform with both cold-start
strategies, the four recommend calls, save and load; RegressionEvaluator's RMSE of the transform equals the RMSE of
the oracle's fit from the same start within fp32 noise."""
import numpy as np
import pandas as pd
import pytest

import als_oracle as ao
from spark_rapids_ml_b200.recommendation import ALS, ALSModel

pytestmark = pytest.mark.gpu


@pytest.fixture()
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "700"})


def _data(seed, n=6000):
    rng = np.random.default_rng(seed)
    P, Q = rng.normal(size=(120, 3)), rng.normal(size=(90, 3))
    u, i = rng.integers(0, 120, n), rng.integers(0, 90, n)
    r = np.einsum("ij,ij->i", P[u], Q[i]) + 0.1 * rng.normal(size=n)
    return pd.DataFrame({"uid": (u * 10).astype(np.int64), "iid": i.astype(np.int32), "score": r})


def test_fit_transform_recommend_persist(session, tmp_path):
    from spark_rapids_ml_b200.evaluation import RegressionEvaluator

    pdf = _data(0)
    df = session.createDataFrame(pdf, num_partitions=3)
    als = ALS(rank=3, maxIter=8, regParam=0.02, userCol="uid", itemCol="iid", ratingCol="score", seed=5)
    model = als.fit(df)
    assert model.rank == 3
    uf = model.userFactors.toPandas()
    assert list(uf.columns) == ["id", "features"] and uf["id"].is_monotonic_increasing
    out = model.transform(df)
    rmse = RegressionEvaluator(metricName="rmse", labelCol="score", predictionCol="prediction").evaluate(out)
    ref = ao.fit(pdf["uid"].to_numpy(), pdf["iid"].to_numpy(), pdf["score"].to_numpy(np.float32), 3, 8, 0.02, seed=5)
    _, _, du, di = ao.index(pdf["uid"].to_numpy(), pdf["iid"].to_numpy())
    p_ref = ao.predict(ref["user_factors"][du], ref["item_factors"][di])
    rmse_ref = float(np.sqrt(np.mean((p_ref - pdf["score"].to_numpy(np.float32)) ** 2)))
    assert abs(rmse - rmse_ref) <= 1e-4 * max(1.0, rmse_ref) and rmse < 0.3, (rmse, rmse_ref)

    # cold start: an unknown user and an unknown item
    test = pd.DataFrame({"uid": np.array([0, 999999, 10], dtype=np.int64), "iid": np.array([1, 2, 777], np.int32),
                         "score": [1.0, 2.0, 3.0]})
    tdf = session.createDataFrame(test)
    p = model.transform(tdf).toPandas()["prediction"].to_numpy()
    assert np.isfinite(p[0]) and np.isnan(p[1:]).all()
    model.setColdStartStrategy("drop")
    assert model.transform(tdf).toPandas()["uid"].tolist() == [0]

    recs = model.recommendForAllUsers(5).toPandas()
    assert list(recs.columns) == ["uid", "recommendations"] and len(recs) == len(uf)
    S = ao.scores(model._uf, model._if)
    first = recs["recommendations"].iloc[0]
    assert [x["iid"] for x in first] == list(model._iid_[np.lexsort((np.arange(S.shape[1]), -S[0].astype(float)))[:5]])
    assert np.float32(first[0]["rating"]) == S[0].max()
    assert len(model.recommendForAllItems(4).toPandas()) == len(model._iid_)
    sub = model.recommendForUserSubset(session.createDataFrame(pd.DataFrame({"uid": [10, 20, 123456]})), 3).toPandas()
    assert sub["uid"].tolist() == [10, 20]
    assert model.recommendForItemSubset(session.createDataFrame(pd.DataFrame({"iid": [3]})), 2).toPandas()["iid"].tolist() == [3]

    model.write().overwrite().save(str(tmp_path / "als"))
    m2 = ALSModel.load(str(tmp_path / "als"))
    assert m2.rank == 3 and m2.getUserCol() == "uid" and m2.getColdStartStrategy() == "drop"
    np.testing.assert_array_equal(m2._uf, model._uf)
    np.testing.assert_array_equal(m2._if, model._if)
    m2.setColdStartStrategy("nan")
    np.testing.assert_array_equal(m2.transform(tdf).toPandas()["prediction"].to_numpy()[:1], p[:1])


def test_refusals(session):
    df = session.createDataFrame(_data(1, 300).rename(columns={"uid": "user", "iid": "item", "score": "rating"}))
    with pytest.raises(NotImplementedError, match="nonnegative"):
        ALS(nonnegative=True).fit(df)
    with pytest.raises(NotImplementedError):
        ALS().fitMultiple(df, [{}])
    bad = session.createDataFrame(pd.DataFrame({"user": [1.5, 2.0], "item": [1, 2], "rating": [1.0, 2.0]}))
    with pytest.raises(ValueError, match="for column user. Value 1.5 was either out of Integer range"):
        ALS(rank=2, maxIter=1).fit(bad)
