"""BisectingKMeans / BisectingKMeansModel end to end on local frames over several partitions: well-separated blobs
are recovered, computeCost on the training frame equals the training cost, the model round-trips through save and
load with the same transform, and ClusteringEvaluator scores the output."""
import numpy as np
import pytest

from spark_rapids_ml_b200.clustering import BisectingKMeans, BisectingKMeansModel

pytestmark = pytest.mark.gpu


@pytest.fixture()
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "500", "spark.rapids.ml.num_workers.local": "1"})


def test_fit_transform_cost_persistence_and_evaluator(session, tmp_path):
    rng = np.random.default_rng(0)
    # far apart: a bisecting split of the first level must not cut through a blob
    means = 5 * np.array([[0.0, 0.0, 0.0], [20.0, 0.0, 5.0], [0.0, 25.0, -10.0], [-15.0, -15.0, 10.0]])
    z = rng.integers(0, 4, size=4000)
    X = (means[z] + rng.normal(size=(4000, 3))).astype(np.float32)
    df = session.from_numpy(X, num_partitions=4)
    model = BisectingKMeans(k=4, seed=5).fit(df)
    assert model.hasSummary and model.summary.k == 4 and model.summary.numIter == 20
    centers = np.stack(model.clusterCenters())
    order = [int(np.argmin(np.linalg.norm(centers - m, axis=1))) for m in means]
    assert sorted(order) == [0, 1, 2, 3]
    np.testing.assert_allclose(centers[order], means, atol=0.2)
    pred = model.transform(df).toPandas()["prediction"].to_numpy()
    assert (np.asarray(order)[z] == pred).mean() > 0.99
    np.testing.assert_array_equal(np.bincount(pred, minlength=4), model.summary.clusterSizes)
    assert model.computeCost(df) == pytest.approx(model.summary.trainingCost, rel=1e-9)

    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    v = ClusteringEvaluator().evaluate(model.transform(df))
    assert 0.5 < v <= 1.0, v

    model.write().overwrite().save(str(tmp_path / "bkm"))
    m2 = BisectingKMeansModel.load(str(tmp_path / "bkm"))
    assert m2.node_index_ == model.node_index_ and m2.node_centers_ == model.node_centers_
    np.testing.assert_array_equal(m2.transform(df).toPandas()["prediction"].to_numpy(), pred)


def test_multi_column_features_and_fraction_min_size(session):
    import pandas as pd

    rng = np.random.default_rng(1)
    X = rng.normal(size=(1500, 3)).astype(np.float32)
    cols = ["a", "b", "c"]
    df1 = session.createDataFrame(pd.DataFrame(X, columns=cols), num_partitions=1)
    df3 = session.createDataFrame(pd.DataFrame(X, columns=cols), num_partitions=3)
    m1 = BisectingKMeans(k=5, seed=2, minDivisibleClusterSize=0.1, featuresCol=cols).fit(df1)
    m3 = BisectingKMeans(k=5, seed=2, minDivisibleClusterSize=0.1, featuresCol=cols).fit(df3)
    assert m1.node_index_ == m3.node_index_ and m1.node_centers_ == m3.node_centers_
    assert sum(m1.summary.clusterSizes) == 1500
    assert all(s >= 150 for i, s in zip(m1.node_index_, m1.node_sizes_) if 2 * i in m1.node_index_)
