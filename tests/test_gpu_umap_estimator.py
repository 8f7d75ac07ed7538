"""UMAP / UMAPModel end to end on the GPU: fit + transform on scikit-learn's bundled digits and iris, repeated with
noise as the reference's tests do, supervised and not, both inits; transform over several partitions; persistence."""
from __future__ import annotations

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _session():
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    return LocalSession.builder.getOrCreate() if hasattr(LocalSession, "builder") else LocalSession()


def _load(name, n_rows, seed=0):
    ds = pytest.importorskip("sklearn.datasets")
    X, y = (ds.load_digits if name == "digits" else ds.load_iris)(return_X_y=True)
    rng = np.random.default_rng(seed)
    reps = -(-n_rows // X.shape[0])
    X = np.concatenate([X] * reps)[:n_rows]
    y = np.concatenate([y] * reps)[:n_rows]
    X = X + rng.normal(scale=0.1 * X.std(), size=X.shape)   # as the reference's _load_dataset
    return X.astype(np.float32), y.astype(np.float64)


def _frame(X, y=None, parts=1):
    rows = [(list(map(float, x)),) + ((float(v),) if y is not None else ()) for x, v in
            zip(X, y if y is not None else [None] * len(X))]
    df = _session().createDataFrame(rows, ["features"] + (["label"] if y is not None else []))
    return df.repartition(parts) if parts > 1 else df


def _embedding(df, col="embedding"):
    return np.array([list(r[col]) for r in df.collect()], dtype=np.float32)


@pytest.mark.parametrize("name,n_rows", [("digits", 2000), ("iris", 500)])
@pytest.mark.parametrize("init", ["random", "spectral"])
@pytest.mark.parametrize("supervised", [False, True])
def test_fit_transform_trustworthiness(name, n_rows, init, supervised):
    man = pytest.importorskip("sklearn.manifold")
    from spark_rapids_ml_b200.umap import UMAP

    X, y = _load(name, n_rows)
    df = _frame(X, y if supervised else None)
    est = UMAP(n_neighbors=15, init=init, random_state=42).setFeaturesCol("features")
    if supervised:
        est = est.setLabelCol("label")
    model = est.fit(df)
    assert np.asarray(model.embedding).shape == (n_rows, 2)
    emb = _embedding(model.transform(df))
    assert np.isfinite(emb).all()
    t = man.trustworthiness(X, emb, n_neighbors=10)
    # a random 2-d layout of these sets scores about 0.5; umap-learn reaches about 0.98 on digits and 0.99 on iris
    assert t >= 0.9, (name, init, supervised, t)


def test_transform_partitions_equal_one_partition_and_persistence(tmp_path):
    from spark_rapids_ml_b200.umap import UMAP, UMAPModel

    X, _ = _load("digits", 1000)
    model = UMAP(n_neighbors=10, n_epochs=60, init="random", random_state=3).setFeaturesCol("features").fit(_frame(X))
    Q, _ = _load("digits", 700, seed=1)
    whole = _embedding(model.transform(_frame(Q)))
    split = _embedding(model.transform(_frame(Q, parts=3)))
    # rows are independent: the partitioning changes nothing, bit for bit (after restoring row order)
    order = lambda E: E[np.lexsort(E.T)]   # noqa: E731
    assert np.array_equal(order(whole), order(split))
    model.write().save(str(tmp_path / "m"))
    again = _embedding(UMAPModel.load(str(tmp_path / "m")).transform(_frame(Q)))
    assert np.array_equal(whole, again)
    # the fit is deterministic and records its seed
    model2 = UMAP(n_neighbors=10, n_epochs=60, init="random", random_state=3).setFeaturesCol("features").fit(_frame(X))
    assert np.array_equal(np.asarray(model.embedding), np.asarray(model2.embedding))
    m3 = UMAP(n_neighbors=10, n_epochs=5, init="random").setFeaturesCol("features").fit(_frame(X[:200]))
    assert isinstance(m3.cuml_params["random_state"], int)


def test_n_neighbors_above_rows_is_clamped(caplog):
    from spark_rapids_ml_b200.umap import UMAP

    X, _ = _load("iris", 20)
    model = UMAP(n_neighbors=50, n_epochs=10, init="random", random_state=0).setFeaturesCol("features").fit(_frame(X))
    assert np.asarray(model.embedding).shape == (20, 2)
