"""The grouped transform path of core.py without a GPU: the device row appender and the library context are replaced by
host stand-ins whose predict calls compute in NumPy, so what is under test is the grouping of frames into device passes,
the split of each pass's outputs back into one result per frame, zero-row frames and partitions, and the Arrow column
each output becomes."""
import numpy as np
import pyarrow as pa
import pytest
import torch

from spark_rapids_ml_b200 import core
from spark_rapids_ml_b200.sparkshim.sql import LocalDataFrame, LocalSession

D = 3


class HostAppender:
    def __init__(self, ctx, d, first_capacity=0):
        self.d, self.rows_ = d, []

    def append_values(self, values, offsets, n_b):
        lo = int(offsets[0]) if offsets is not None else 0
        self.rows_.append(np.asarray(values[lo:lo + n_b * self.d], dtype=np.float32).reshape(n_b, self.d))

    def append_columns(self, cols):
        self.rows_.append(np.stack(cols, 1).astype(np.float32))

    def finish(self):
        return torch.from_numpy(np.concatenate(self.rows_))


class HostContext:
    """The library context's predict calls, in NumPy with each row on its own (no BLAS), so that the grouping cannot
    change a value; `passes` records the rows of each device pass."""
    device = torch.device("cpu")

    def __init__(self):
        self.passes = []

    def kmeans_assign(self, X, C):
        self.passes.append(int(X.shape[0]))
        d2 = ((X.numpy()[:, None, :] - C.numpy()[None]) ** 2).sum(-1)
        return torch.from_numpy(d2.argmin(1).astype(np.int32)), None

    def pca_transform(self, X, C):
        self.passes.append(int(X.shape[0]))
        return torch.from_numpy((X.numpy()[:, None, :] * C.numpy()[None]).sum(-1))

    def linreg_predict(self, X, w, b):
        self.passes.append(int(X.shape[0]))
        return torch.from_numpy(b + (X.numpy().astype(np.float64) * w.numpy()).sum(1))

    def logreg_predict(self, X, W, b, cls):
        self.passes.append(int(X.shape[0]))
        m = (X.numpy().astype(np.float64)[:, None, :] * W[None]).sum(-1) + b
        raw = np.c_[-m, m] if W.shape[0] == 1 else m
        prob = np.exp(raw) / np.exp(raw).sum(1, keepdims=True)
        return torch.from_numpy(raw), torch.from_numpy(prob), torch.from_numpy(cls[raw.argmax(1)])


@pytest.fixture
def ctx(monkeypatch):
    c = HostContext()
    monkeypatch.setattr(core, "DeviceRowAppender", HostAppender)
    monkeypatch.setattr(core, "_transform_context", lambda gpu: c)
    monkeypatch.setattr(core._CumlCommon, "_set_gpu_device", staticmethod(lambda *a, **k: 0))
    return c


def _models():
    from spark_rapids_ml_b200.classification import LogisticRegressionModel
    from spark_rapids_ml_b200.clustering import KMeansModel
    from spark_rapids_ml_b200.feature import PCAModel
    from spark_rapids_ml_b200.regression import LinearRegressionModel

    pca = PCAModel(mean_=[0.0] * D, components_=[[1.0, 0.5, 0.0], [0.0, -1.0, 2.0]], explained_variance_ratio_=[0.6, 0.4],
                   singular_values_=[2.0, 1.0], n_cols=D, dtype="float32").setInputCol("features").setOutputCol("pca")
    return {
        "kmeans": (KMeansModel(cluster_centers_=[[0.0, 0.0, 0.0], [5.0, 5.0, 5.0], [-5.0, 0.0, 5.0]], n_cols=D,
                               dtype="float32"), [("prediction", pa.int32())]),
        "pca": (pca, [("pca", pa.list_(pa.float32()))]),
        "linreg": (LinearRegressionModel(coef_=[1.0, -2.0, 0.5], intercept_=0.25, n_cols=D, dtype="float32"),
                   [("prediction", pa.float64())]),
        "logreg": (LogisticRegressionModel(coef_=[[1.0, -1.0, 0.5], [0.0, 2.0, -1.0], [-1.0, 0.0, 0.0]],
                                           intercept_=[0.1, 0.0, -0.1], classes_=[0.0, 1.0, 2.0], n_cols=D,
                                           dtype="float32", num_iters=1),
                   [("rawPrediction", pa.list_(pa.float64())), ("probability", pa.list_(pa.float64())),
                    ("prediction", pa.float64())]),
    }


def _rows(n, seed=0):
    return np.random.default_rng(seed).normal(scale=4.0, size=(n, D)).astype(np.float32)


def _frame(parts):
    """A local frame with one partition per entry of `parts`, each a list of row blocks (one batch per block)."""
    schema = pa.schema([pa.field("features", pa.list_(pa.float32()))])
    batches = [[pa.RecordBatch.from_arrays([pa.array([list(map(float, r)) for r in blk], type=schema[0].type)],
                                           schema=schema) for blk in p] for p in parts]
    return LocalDataFrame(LocalSession(), batches, schema)


@pytest.mark.parametrize("name", ["kmeans", "pca", "linreg", "logreg"])
def test_partitions_and_zero_row_frames_give_the_rows_of_one_pass(ctx, monkeypatch, name):
    """The same rows as one partition of one batch and as three partitions (one empty, one led by a zero-row batch) in
    groups of at most 7 rows: the same column names, Arrow types and values, and one device pass per group."""
    model, cols = _models()[name]
    X = _rows(30)
    whole = model.transform(_frame([[X]]))
    assert ctx.passes == [30]
    del ctx.passes[:]
    monkeypatch.setattr(core, "TRANSFORM_GROUP_ROWS", 7)
    split = model.transform(_frame([[X[:4], X[4:9], X[9:9], X[9:12]], [], [X[12:12], X[12:20], X[20:30]]]))
    assert ctx.passes == [9, 3, 8, 10]
    for out in (whole, split):
        assert [(f.name, f.type) for f in out.schema][1:] == cols
        assert out.count() == 30
    t1, t2 = whole._table(), split._table()
    for c, _ in cols:
        assert t1.column(c).to_pylist() == t2.column(c).to_pylist(), c
    # zero-row batches keep their place: one (empty) array per batch
    assert [[b.num_rows for b in p] for p in split._parts] == [[4, 5, 0, 3], [], [0, 8, 10]]


@pytest.mark.parametrize("name", ["kmeans", "pca", "linreg", "logreg"])
def test_a_group_without_rows_makes_no_device_pass(ctx, name):
    model, cols = _models()[name]
    X0 = _rows(0)
    out = model.transform(_frame([[X0, X0], [], [X0]]))
    assert ctx.passes == []
    assert [(f.name, f.type) for f in out.schema][1:] == cols
    assert [[b.num_rows for b in p] for p in out._parts] == [[0, 0], [], [0]]


def test_grouped_function_splits_each_output_per_frame(ctx):
    """The grouped function itself: one predict call per group, each output cut back into the frames' rows, and
    zero-length outputs of each type's dtype for a group of zero-row frames (what a pandas_udf turns into a Series)."""
    seen = []

    def predict(m, X):
        seen.append(int(X.shape[0]))
        x = X.numpy()
        return (torch.from_numpy(x[:, 0].astype(np.int32)), torch.from_numpy(x.astype(np.float64)),
                torch.from_numpy(x[:, :2].copy()), torch.from_numpy(x.sum(1, dtype=np.float64)))

    types = ["int", "array<double>", "array<float>", "double"]
    transform = core._GroupedTransform(predict, D, 4 * D, types)
    model = core._DeviceModel(0)
    frames = [_rows(n, seed=n) for n in (3, 0, 5)]
    got = transform(model, frames)
    assert seen == [8] and len(got) == 3
    for f, res in zip(frames, got):
        assert [r.shape for r in res] == [(len(f),), (len(f), D), (len(f), 2), (len(f),)]
        np.testing.assert_array_equal(res[1], f.astype(np.float64))
    empty = transform(model, [frames[1], frames[1]])
    assert seen == [8] and len(empty) == 2
    for res in empty:
        assert [(r.shape, r.dtype) for r in res] == [((0,), np.int32), ((0, 0), np.float64), ((0, 0), np.float32),
                                                     ((0,), np.float64)]
        arrs = [core._transform_result_array(r, t) for r, t in zip(res, types)]
        assert [a.type for a in arrs] == [pa.int32(), pa.list_(pa.float64()), pa.list_(pa.float32()), pa.float64()]
        assert all(len(a) == 0 for a in arrs)


def test_device_model_holds_its_arrays_until_closed(ctx):
    m = core._DeviceModel(0, C=np.ones((2, D), np.float32), w=np.arange(D, dtype=np.float64))
    assert m.ctx is ctx
    assert m.arrays["C"].dtype == torch.float32 and m.arrays["w"].dtype == torch.float64
    m.close()
    assert m.arrays == {}


def test_appended_column_must_have_one_array_per_batch():
    df = _frame([[_rows(2), _rows(3)], [_rows(4)]])
    arrs = [[pa.array(np.zeros(2)), pa.array(np.zeros(3))], [pa.array(np.zeros(4))]]
    assert df.with_appended_column("x", arrs).count() == 9
    with pytest.raises(ValueError, match="partition 0 has 2 batches but 1 arrays"):
        df.with_appended_column("x", [arrs[0][:1], arrs[1]])
    with pytest.raises(ValueError, match="partition 1 has 1 batches but 0 arrays"):
        df.with_appended_column("x", [arrs[0], []])
    with pytest.raises(ValueError, match="1 partitions of arrays for a frame of 2 partitions"):
        df.with_appended_column("x", arrs[:1])
