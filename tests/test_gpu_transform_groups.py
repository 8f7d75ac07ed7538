"""transform() on the GPU does not depend on how the rows are split: for every model with a grouped device transform, the
same rows as one partition and as three partitions (one empty, one led by a zero-row batch), in groups of a few hundred
rows, give the same columns, Arrow types and values, bit for bit.  Every one of these transforms computes each row on its
own, so the group boundaries cannot change a value."""
import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
pytest.importorskip("torch")

N, D = 3000, 12


def _data():
    rng = np.random.default_rng(5)
    X = rng.normal(size=(N, D)).astype(np.float32)
    y = ((X[:, 0] + X[:, 1] > 0).astype(int) + (X[:, 2] > 1.0)).astype(np.float32)   # three classes
    return X, y


def _fit_frame(X, y):
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    return LocalSession().createDataFrame([(X[i].tolist(), float(y[i])) for i in range(len(y))],
                                          "features array<float>, label float")


def _frame(parts):
    """A local frame with one partition per entry of `parts`, each a list of row blocks (one batch per block)."""
    from spark_rapids_ml_b200.sparkshim.sql import LocalDataFrame, LocalSession

    schema = pa.schema([pa.field("features", pa.list_(pa.float32()))])
    batches = [[pa.RecordBatch.from_arrays([pa.array(list(blk), type=schema[0].type)], schema=schema) for blk in p]
               for p in parts]
    return LocalDataFrame(LocalSession(), batches, schema)


_PRED = [("rawPrediction", pa.list_(pa.float64())), ("probability", pa.list_(pa.float64())),
         ("prediction", pa.float64())]


def _model(name, X, y):
    """A fitted model and the (name, Arrow type) of each column its transform() appends."""
    from spark_rapids_ml_b200.classification import LogisticRegression, RandomForestClassifier
    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.feature import PCA
    from spark_rapids_ml_b200.regression import LinearRegression, RandomForestRegressor
    from spark_rapids_ml_b200.umap import UMAP

    df = _fit_frame(X, y)
    if name == "kmeans":
        return KMeans(k=5, maxIter=10, seed=1, num_workers=1).fit(df), [("prediction", pa.int32())]
    if name == "pca":
        return PCA(k=3, inputCol="features", outputCol="pca", num_workers=1).fit(df), [("pca", pa.list_(pa.float32()))]
    if name == "linreg":
        return LinearRegression(regParam=0.01, num_workers=1).fit(df), [("prediction", pa.float64())]
    if name == "logreg":
        return LogisticRegression(regParam=0.01, num_workers=1).fit(df), _PRED
    if name == "rf_classifier":
        return RandomForestClassifier(numTrees=6, maxDepth=5, seed=2, num_workers=1).fit(df), _PRED
    if name == "rf_regressor":
        return (RandomForestRegressor(numTrees=6, maxDepth=5, seed=2, num_workers=1).fit(df),
                [("prediction", pa.float64())])
    assert name == "umap"
    model = UMAP(n_neighbors=10, n_epochs=60, init="random", random_state=3).setFeaturesCol("features")
    return model.fit(_fit_frame(X[:1000], y[:1000])), [("embedding", pa.list_(pa.float32()))]


@pytest.mark.parametrize("name", ["kmeans", "pca", "linreg", "logreg", "rf_classifier", "rf_regressor", "umap"])
def test_split_rows_transform_like_one_partition(name, monkeypatch):
    from spark_rapids_ml_b200 import core

    X, y = _data()
    model, cols = _model(name, X, y)
    monkeypatch.setattr(core, "TRANSFORM_GROUP_ROWS", 700)   # several device passes per partition
    blocks = lambda A, n: [A[i:i + n] for i in range(0, len(A), n)]   # noqa: E731
    whole = model.transform(_frame([blocks(X, 500)]))
    split = model.transform(_frame([blocks(X[:1100], 300), [], [X[:0]] + blocks(X[1100:], 450)]))
    for out in (whole, split):
        assert [(f.name, f.type) for f in out.schema][1:] == cols
        assert out.count() == N
    t1, t2 = whole._table(), split._table()
    for c, _ in cols:
        assert t1.column(c).to_pylist() == t2.column(c).to_pylist(), c
