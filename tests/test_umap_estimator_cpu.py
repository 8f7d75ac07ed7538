"""UMAP / UMAPModel's surface without a GPU: params, defaults, copy, Spark confs, float32_inputs, the host a/b fit, the
sample, persistence and the inputs it refuses (after the reference's test_params, test_umap_copy and
test_handle_param_spark_confs)."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest


def test_params_and_defaults():
    from spark_rapids_ml_b200.umap import UMAP

    est = UMAP()
    assert est.cuml_params["n_neighbors"] == 15 and est.cuml_params["n_components"] == 2
    assert est.cuml_params["init"] == "spectral" and est.cuml_params["a"] is None
    assert (est.getNNeighbors(), est.getNComponents(), est.getMetric(), est.getInit(), est.getMinDist(),
            est.getSpread(), est.getSetOpMixRatio(), est.getLocalConnectivity(), est.getRepulsionStrength(),
            est.getNegativeSampleRate(), est.getTransformQueueSize(), est.getBuildAlgo(), est.getSampleFraction(),
            est.getOutputCol()) == (15, 2, "euclidean", "spectral", 0.1, 1.0, 1.0, 1.0, 1.0, 5, 4.0, "auto", 1.0,
                                    "embedding")
    assert est.getNEpochs() is None and est.getRandomState() is None and est.getA() is None and est.getB() is None
    est = UMAP(n_neighbors=7, n_components=3, init="random", a=1.2, b=0.8, random_state=4, sample_fraction=0.5,
               featuresCol=["x", "y"], labelCol="lab", outputCol="e")
    assert est.cuml_params["n_neighbors"] == 7 and est.cuml_params["n_components"] == 3
    assert est.cuml_params["init"] == "random" and est.cuml_params["random_state"] == 4
    assert est.getFeaturesCol() == ["x", "y"] and est.getOrDefault("labelCol") == "lab" and est.getOutputCol() == "e"
    assert est.setNEpochs(30).getNEpochs() == 30 and est.cuml_params["n_epochs"] == 30
    assert est.setSampleFraction(0.25).getSampleFraction() == 0.25


def test_umap_copy():
    from spark_rapids_ml_b200.umap import UMAP

    est = UMAP(n_neighbors=10)
    c = est.copy({est.n_neighbors: 20, est.learning_rate: 0.5})
    assert c.getNNeighbors() == 20 and c.cuml_params["n_neighbors"] == 20 and c.cuml_params["learning_rate"] == 0.5
    assert est.getNNeighbors() == 10 and est.cuml_params["n_neighbors"] == 10


def test_handle_param_spark_confs_and_float32_inputs(caplog):
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession
    from spark_rapids_ml_b200.umap import UMAP

    sess = LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()
    sess.conf.set("spark.rapids.ml.num_workers", "3")
    sess.conf.set("spark.rapids.ml.verbose", "5")
    try:
        est = UMAP()
        assert est._input_kwargs["verbose"] == 5 and est._input_kwargs["num_workers"] == 3
        assert est.num_workers == 1   # the fit coalesces to one task whatever num_workers is
    finally:
        sess.conf.unset("spark.rapids.ml.num_workers")
        sess.conf.unset("spark.rapids.ml.verbose")
    est = UMAP(float32_inputs=False)
    assert est._float32_inputs is True


def test_find_ab_params_matches_curve_fit():
    opt = pytest.importorskip("scipy.optimize")
    from spark_rapids_ml_b200.umap import find_ab_params

    for spread, min_dist in ((1.0, 0.1), (2.0, 0.5), (1.0, 0.0)):
        a, b = find_ab_params(spread, min_dist)
        x = np.linspace(0, spread * 3, 300)
        y = np.where(x < min_dist, 1.0, np.exp(-(x - min_dist) / spread))
        (a2, b2), _ = opt.curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), x, y)
        assert abs(a - a2) < 1e-5 * max(1, a2) and abs(b - b2) < 1e-5, (spread, min_dist, a, a2, b, b2)
    a, b = find_ab_params(1.0, 0.1)
    assert abs(a - 1.577) < 1e-3 and abs(b - 0.895) < 1e-3


def test_bernoulli_sample():
    from spark_rapids_ml_b200.umap import bernoulli_sample

    assert np.array_equal(bernoulli_sample(10, 1.0, 3), np.arange(10))
    s = bernoulli_sample(10000, 0.3, 3)
    assert np.array_equal(s, np.nonzero(np.random.default_rng(3).random(10000) < 0.3)[0])
    assert 2800 < s.size < 3200


def test_persistence_round_trip_and_layout(tmp_path):
    pq = pytest.importorskip("pyarrow.parquet")
    from spark_rapids_ml_b200.umap import UMAPModel

    rng = np.random.default_rng(0)
    m = UMAPModel(embedding_=rng.random((6, 2)).astype(np.float32), raw_data_=rng.random((6, 3)).astype(np.float32),
                  n_cols=3, dtype="float32")
    m._set_params(n_neighbors=4, outputCol="emb")
    path = str(tmp_path / "m")
    m.write().save(path)
    assert os.path.isdir(os.path.join(path, "metadata"))
    for name in ("embedding_.parquet", "raw_data_.parquet", "metadata.json"):
        assert os.path.isfile(os.path.join(path, "data", name))
    t = pq.read_table(os.path.join(path, "data", "raw_data_.parquet"))
    assert t.column_names == ["row_id", "data"]
    assert json.load(open(os.path.join(path, "data", "metadata.json")))["n_cols"] == 3
    with pytest.raises(IOError):
        m.write().save(path)
    m.write().overwrite().save(path)
    r = UMAPModel.load(path)
    assert np.array_equal(r.embedding_, m.embedding_) and np.array_equal(r.raw_data_, m.raw_data_)
    assert r.uid == m.uid and r.getNNeighbors() == 4 and r.getOutputCol() == "emb"
    assert r.embedding == m.embedding and r.rawData == m.rawData


def test_unsupported_inputs_raise():
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession
    from spark_rapids_ml_b200.umap import UMAP

    sess = LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()
    df = sess.createDataFrame([([1.0, 2.0],), ([2.0, 3.0],)], ["features"])
    with pytest.raises(ValueError, match="metric"):
        UMAP(metric="cosine").setFeaturesCol("features").fit(df)
    with pytest.raises(ValueError, match="precomputed_knn"):
        UMAP(precomputed_knn=[[0.0]])
    with pytest.raises(ValueError, match="sparse"):
        UMAP(enable_sparse_data_optim=True)
    with pytest.raises(ValueError, match="sample_fraction"):
        UMAP(sample_fraction=0.0).setFeaturesCol("features").fit(df)
