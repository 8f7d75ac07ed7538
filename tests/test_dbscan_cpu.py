"""DBSCAN without a GPU: the fp64 oracle against scikit-learn, the wgmma screen's error bound against a NumPy restatement
of the screen on adversarial pairs, the reference's known answers, and the estimator surface (params, defaults, copy,
Spark confs, persistence)."""
import json
import os

import numpy as np
import pytest

import dbscan_oracle as do

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dbscan_known_answers.json")


def _blobs(n, d, k, seed, spread=4.0, std=1.0):
    rng = np.random.default_rng(seed)
    C = rng.uniform(-spread, spread, size=(k, d))
    return (C[rng.integers(0, k, size=n)] + std * rng.normal(size=(n, d))).astype(np.float32)


# ---- the oracle against scikit-learn ----
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("d, eps, ms", [(2, 0.6, 5), (8, 3.2, 6), (20, 5.0, 5)])
def test_oracle_matches_sklearn(metric, d, eps, ms):
    sk = pytest.importorskip("sklearn.cluster")
    X = _blobs(800, d, 5, seed=d)
    if metric == "cosine":
        X = X + 3.0
        eps = 0.02
    lab, core, n = do.dbscan(X, eps, ms, metric)
    ref = sk.DBSCAN(eps=eps, min_samples=ms, metric=metric, algorithm="brute").fit(X.astype(np.float64))
    rcore = np.zeros(len(X), dtype=bool)
    rcore[ref.core_sample_indices_] = True
    np.testing.assert_array_equal(core, rcore)
    np.testing.assert_array_equal(lab == -1, ref.labels_ == -1)
    assert n == len(set(ref.labels_[rcore]))
    # the same partition of the core rows
    pairs = {(a, b) for a, b in zip(lab[core], ref.labels_[core])}
    assert len(pairs) == n == len({a for a, _ in pairs}) == len({b for _, b in pairs})
    mapping = dict(pairs)
    # border rows: equal unless the row touches two clusters
    adj = do.adjacency_lists(X, eps, metric)
    for i in np.nonzero(~core & (lab >= 0))[0]:
        touched = {lab[j] for j in adj[i] if core[j]}
        if len(touched) == 1:
            assert mapping[lab[i]] == ref.labels_[i], i
    assert n >= 1


def test_numbering_is_by_lowest_core_row():
    X = np.array([[10.0, 0], [10.5, 0], [0.0, 0], [0.5, 0], [20.0, 0]], dtype=np.float32)
    lab, core, n = do.dbscan(X, 1.0, 2)
    assert lab.tolist() == [0, 0, 1, 1, -1] and n == 2


# ---- the screen's bound ----
def _adversarial_pairs(n_pairs, d, offset, seed, eps=0.75):
    """Pairs along feature 0 at eps, one ulp inside and one outside, other features equal within a pair."""
    rng = np.random.default_rng(seed)
    rows = []
    for p in range(n_pairs):
        a = (offset + rng.uniform(-1.0, 1.0, size=d)).astype(np.float32)
        b = a.copy()
        b[0] = np.float32(a[0] + np.float32(eps))
        b[0] = [b[0], np.nextafter(b[0], np.float32(-np.inf)), np.nextafter(b[0], np.float32(np.inf))][p % 3]
        c = (offset + rng.uniform(-1.0, 1.0, size=d)).astype(np.float32)   # an unrelated row
        rows += [a, b, c]
    return np.array(rows, dtype=np.float32)


@pytest.mark.parametrize("d", [4, 32, 128])
@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3])
def test_bound_is_never_exceeded(d, offset):
    X = _adversarial_pairs(200, d, offset, seed=d)
    n = len(X)
    rng = np.random.default_rng(1)
    i = np.concatenate([np.arange(0, n, 3), rng.integers(0, n, 3000)])
    j = np.concatenate([np.arange(1, n, 3), rng.integers(0, n, 3000)])
    D = np.array([do._pair_values(X[a:a + 1], X[b:b + 1], "euclidean")[0, 0] for a, b in zip(i, j)])
    E = 0.75 ** 2
    V = do.shifted(X)
    S = do.screen(V, i, j)
    B = do.bound(V, i, j, d, "euclidean", E)
    err = np.abs(S.astype(np.float64) - D)
    assert np.all(err <= B), float((err / B).max())
    # the kernel's decisions: outside the band the screen's side of E is the fp64 rule's side
    r = (S - np.float32(E)).astype(np.float32)
    inside, outside = r < -B, r > B
    assert np.all(D[inside] <= E) and np.all(D[outside] > E)
    assert (~inside & ~outside)[: n // 3].any()   # some pairs within one ulp of eps are left to the fp64 rule
    if offset == 1e3:
        Su = do.screen(X, i, j)   # the same screen without the shift
        assert np.any(np.abs(Su.astype(np.float64) - D) > B)


@pytest.mark.parametrize("d", [4, 32, 128])
def test_bound_cosine(d):
    rng = np.random.default_rng(d)
    X = (rng.normal(size=(600, d)) * rng.uniform(0.01, 100, size=(600, 1)) + 1.0).astype(np.float32)
    X[1::2] = (X[0::2] + 1e-3 * rng.normal(size=(300, d))).astype(np.float32)   # near-parallel pairs
    nrm = do.row_norms(X)
    i = np.concatenate([np.arange(0, 600, 2), rng.integers(0, 600, 3000)])
    j = np.concatenate([np.arange(1, 600, 2), rng.integers(0, 600, 3000)])
    D = np.array([2.0 * do._pair_values(X[a:a + 1], X[b:b + 1], "cosine", nrm[a:a + 1], nrm[b:b + 1])[0, 0]
                  for a, b in zip(i, j)])
    V = do.shifted(X, "cosine")
    S = do.screen(V, i, j)
    B = do.bound(V, i, j, d, "cosine", 2 * 0.01)
    assert np.all(np.abs(S.astype(np.float64) - D) <= B)


# ---- known answers ----
def test_known_answers_fixture():
    with open(GOLDEN) as f:
        cases = json.load(f)["cases"]
    assert [c["name"] for c in cases] == ["basic", "numeric_type_defaults"]
    for c in cases:
        lab, core, n = do.dbscan(np.array(c["X"], dtype=np.float32), c["eps"], c["min_samples"], c["metric"])
        assert lab.tolist() == c["labels"] and core.tolist() == c["core"] and n == c["n_clusters"]


# ---- estimator surface ----
def test_params_and_defaults():
    from spark_rapids_ml_b200.clustering import DBSCAN

    est = DBSCAN()
    assert est.cuml_params == {"eps": 0.5, "min_samples": 5, "metric": "euclidean", "algorithm": "brute",
                               "verbose": False, "max_mbytes_per_batch": None, "calc_core_sample_indices": False}
    assert (est.getEps(), est.getMinSamples(), est.getMetric(), est.getAlgorithm(), est.getMaxMbytesPerBatch()) == \
        (0.5, 5, "euclidean", "brute", None)
    assert est.getIdCol() == "unique_id" and est.getOrDefault("predictionCol") == "prediction"
    est = DBSCAN(eps=2.0, min_samples=3, metric="cosine", algorithm="rbc", max_mbytes_per_batch=64,
                 featuresCols=["a", "b"], idCol="id", verbose=True)
    assert est.cuml_params["eps"] == 2.0 and est.cuml_params["min_samples"] == 3
    assert est.cuml_params["metric"] == "cosine" and est.cuml_params["algorithm"] == "rbc"
    assert est.cuml_params["max_mbytes_per_batch"] == 64 and est.cuml_params["verbose"] is True
    assert est.getFeaturesCol() == ["a", "b"] and est.getIdCol() == "id"
    est.setEps(0.25).setMinSamples(7).setMetric("euclidean").setAlgorithm("brute").setMaxMbytesPerBatch(None)
    assert est.cuml_params["eps"] == 0.25 and est.cuml_params["min_samples"] == 7


def _frame(X, parts=1):
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({}).from_numpy(np.asarray(X, dtype=np.float32), num_partitions=parts)


def test_fit_is_lazy_and_copies_params():
    from spark_rapids_ml_b200.clustering import DBSCAN, DBSCANModel

    est = DBSCAN(eps=2.0, min_samples=2, metric="cosine")
    model = est.fit(_frame([[0.0, 1.0], [1.0, 1.0]]))
    assert isinstance(model, DBSCANModel) and model.n_cols == 0 and model.dtype == ""
    assert model.cuml_params == est.cuml_params and model.getOrDefault("eps") == 2.0


@pytest.mark.parametrize("metric, msg", [("precomputed", "precomputed"), ("manhattan", "not supported")])
def test_unsupported_metrics(metric, msg):
    from spark_rapids_ml_b200.clustering import DBSCAN

    with pytest.raises(ValueError, match=msg):
        DBSCAN(metric=metric).fit(_frame([[0.0, 1.0]]))


def test_dbscan_copy():
    from spark_rapids_ml_b200.clustering import DBSCAN

    est = DBSCAN(eps=1.0)
    c = est.copy({est.eps: 7.0, est.min_samples: 9})
    assert c.getEps() == 7.0 and c.cuml_params["eps"] == 7.0 and c.cuml_params["min_samples"] == 9
    assert est.getEps() == 1.0 and est.cuml_params["eps"] == 1.0


def test_handle_param_spark_confs():
    from spark_rapids_ml_b200.clustering import DBSCAN
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    sess = LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()
    sess.conf.set("spark.rapids.ml.num_workers", "3")
    sess.conf.set("spark.rapids.ml.verbose", "5")
    sess.conf.set("spark.rapids.ml.float32_inputs", "false")
    try:
        est = DBSCAN()
        assert est._input_kwargs["verbose"] == 5
        assert est._input_kwargs["float32_inputs"] is False
        assert est._input_kwargs["num_workers"] == 3
        assert DBSCAN(num_workers=2)._num_workers == 2
    finally:
        for k in ("num_workers", "verbose", "float32_inputs"):
            sess.conf.unset(f"spark.rapids.ml.{k}")


def test_persistence(tmp_path):
    from spark_rapids_ml_b200.clustering import DBSCAN, DBSCANModel

    est = DBSCAN(eps=2.0, min_samples=3, metric="cosine", algorithm="rbc", max_mbytes_per_batch=100)
    est.save(str(tmp_path / "est"))
    e2 = DBSCAN.load(str(tmp_path / "est"))
    assert e2.cuml_params == est.cuml_params and e2.getEps() == 2.0
    model = est.fit(_frame([[0.0, 1.0], [1.0, 1.0]]))
    model.write().overwrite().save(str(tmp_path / "model"))
    assert sorted(os.listdir(tmp_path / "model")) == ["data", "metadata"]
    m2 = DBSCANModel.load(str(tmp_path / "model"))
    assert m2.cuml_params == model.cuml_params and m2.n_cols == 0 and m2.dtype == ""
    assert m2.getOrDefault("min_samples") == 3
