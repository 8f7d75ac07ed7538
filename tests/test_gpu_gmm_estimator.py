"""GaussianMixture / GaussianMixtureModel end to end on local frames over several partitions: a well-separated mixture
is recovered, probabilities sum to 1, ClusteringEvaluator scores the output, the model round-trips through save and
load with the same transform, and scalar feature columns give the same fit however the frame is partitioned."""
import numpy as np
import pytest

import gmm_oracle as go
from spark_rapids_ml_b200.clustering import GaussianMixture, GaussianMixtureModel

pytestmark = pytest.mark.gpu


@pytest.fixture()
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "500", "spark.rapids.ml.num_workers.local": "1"})


def _data(n=4000, seed=0):
    rng = np.random.default_rng(seed)
    means = np.array([[0.0, 0.0, 0.0], [20.0, 0.0, 5.0], [0.0, 25.0, -10.0]])
    z = rng.integers(0, 3, size=n)
    A = np.stack([np.diag([1.0, 2.0, 0.5]), np.array([[1.0, 0.8, 0], [0, 1.0, 0], [0, 0, 0.3]]), np.eye(3) * 1.5])
    X = means[z] + np.einsum("nij,nj->ni", A[z], rng.normal(size=(n, 3)))
    return X.astype(np.float32), z, means


def test_fit_transform_recovers_mixture(session, tmp_path):
    X, z, means = _data()
    df = session.from_numpy(X, num_partitions=4)
    est = GaussianMixture(k=3, seed=5, maxIter=50, tol=1e-4, probabilityCol="prob")
    model = est.fit(df)
    assert model.hasSummary and model.summary.k == 3 and 1 <= model.summary.numIter <= 50
    order = [int(np.argmin(np.linalg.norm(np.asarray(model.means_) - m, axis=1))) for m in means]
    assert sorted(order) == [0, 1, 2]
    np.testing.assert_allclose(np.asarray(model.means_)[order], means, atol=0.3)
    np.testing.assert_allclose(np.asarray(model.weights)[order], np.bincount(z) / len(z), atol=0.02)
    assert sum(model.summary.clusterSizes) == len(X)
    g = model.gaussiansDF.toPandas()
    assert len(g) == 3 and len(g["mean"][0]) == 3
    out = model.transform(df)
    pdf = out.toPandas()
    prob = np.stack(pdf["prob"].to_numpy())
    np.testing.assert_allclose(prob.sum(axis=1), 1.0, atol=1e-12)
    pred = pdf["prediction"].to_numpy()
    assert (np.asarray(order)[z] == pred).mean() > 0.99
    np.testing.assert_array_equal(np.argmax(prob, axis=1), pred)
    np.testing.assert_array_equal(np.bincount(pred, minlength=3), model.summary.clusterSizes)
    # the oracle's E-step on the fitted model agrees
    r, _, _ = go.e_step(X, np.asarray(model.weights_), np.asarray(model.means_), np.asarray(model.covs_))
    np.testing.assert_allclose(prob, r, atol=2e-4)

    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator

    v = ClusteringEvaluator().evaluate(out)
    assert 0.5 < v <= 1.0, v

    model.write().overwrite().save(str(tmp_path / "gmm"))
    m2 = GaussianMixtureModel.load(str(tmp_path / "gmm"))
    assert m2.weights_ == model.weights_ and m2.covs_ == model.covs_
    p2 = m2.transform(df).toPandas()
    np.testing.assert_array_equal(np.stack(p2["prob"].to_numpy()), prob)
    np.testing.assert_array_equal(p2["prediction"].to_numpy(), pred)


def test_multi_column_features_and_partitions_of_one_rank(session):
    # one worker: the partitions are concatenated into the same device matrix, so the fits are bitwise equal (the
    # rank tests cover different splits across ranks)
    X, _, _ = _data(1500, seed=1)
    import pandas as pd

    cols = ["a", "b", "c"]
    df1 = session.createDataFrame(pd.DataFrame(X, columns=cols), num_partitions=1)
    df3 = session.createDataFrame(pd.DataFrame(X, columns=cols), num_partitions=3)
    m1 = GaussianMixture(k=3, seed=2, maxIter=5, tol=0.0, featuresCol=cols).fit(df1)
    m3 = GaussianMixture(k=3, seed=2, maxIter=5, tol=0.0, featuresCol=cols).fit(df3)
    assert m1.means_ == m3.means_ and m1.covs_ == m3.covs_ and m1.weights_ == m3.weights_
    assert m1.summary.numIter == m3.summary.numIter == 5
