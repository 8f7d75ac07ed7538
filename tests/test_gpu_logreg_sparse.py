"""Sparse logistic regression on the device: b2k_logreg_eval_csr against the fp64 SciPy oracle and against the dense
pass, bitwise reproducibility (several grid limits, several row chunks with a ragged last one), C-ABI fits, and the
estimator's CSR fit, fitMultiple, transform and errors."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import logreg_oracle as lo
import logreg_sparse_oracle as so

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    with _native.Context(0) as c:
        yield c


def _edge_csr(n, d, seed, per_row=6):
    """Random rows plus the edges: empty rows, a fully dense row among short ones, stored zeros, empty columns (the
    last ones) and column 0 present in every row, so that its run crosses many CSC pieces."""
    X = so.random_csr(n, d, min(per_row, d), seed).tolil()
    X[:, 0] = np.random.default_rng(seed).normal(size=(n, 1)).astype(np.float32)
    X[3, :] = 0.0
    X[7, :] = 0.0
    X[11, :] = np.linspace(-1, 1, d, dtype=np.float32)
    if d > 4:
        X[:, d - 2:] = 0.0
    X = sp.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    X.data[X.indptr[12]] = 0.0   # a stored zero
    X[7, 0] = 0.0   # row 7: empty again (column 0 was set)
    X.eliminate_zeros()
    X.data[X.indptr[12]] = 0.0
    return sp.csr_matrix(X)


def _ingest(ctx, X, dense_rows=()):
    import pandas as pd

    from spark_rapids_ml_b200.utils import DeviceCsrAppender

    app = DeviceCsrAppender(ctx, X.shape[1], first_rows=16, first_nnz=64)   # small: exercises growth
    arr = so.vector_array(X, dense_rows)
    for s in range(0, len(arr), 700):   # several batches
        app.append_column(pd.Series(pd.arrays.ArrowExtensionArray(arr.slice(s, 700))))
    return app.finish()


def _model(d, kp, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(kp, d)) / np.sqrt(min(d, 64)), rng.normal(size=kp)


def _check(got, X, yi, W, b, scale=1.0):
    loss, gW, gb, _ = got
    rl, rW, rb = so.loss_grad(X, yi, W, b)
    bd = so.eval_bound(X, W, b)
    assert abs(loss - rl) <= scale * bd["loss"], (loss, rl, bd["loss"])
    assert np.all(np.abs(gW - rW) <= scale * bd["dW"]), np.max(np.abs(gW - rW) - scale * bd["dW"])
    assert np.all(np.abs(gb - rb) <= scale * bd["db"])


def _labels(n, kp, seed):
    K = max(kp, 2)
    yi = np.random.default_rng(seed).integers(0, K, size=n)
    yi[:K] = np.arange(K)
    return yi, np.arange(K, dtype=np.float64)


@pytest.mark.parametrize("kp", [1, 2, 10, 40])
@pytest.mark.parametrize("d", [1, 3, 1024, 1025, 1 << 18])
def test_eval_matches_oracle(ctx, d, kp):
    import torch

    n = 2000
    X = _edge_csr(n, d, seed=d + kp)
    yi, classes = _labels(n, kp, seed=kp)
    W, b = _model(d, kp, seed=d)
    Xd = _ingest(ctx, X, dense_rows=[20, 21])
    y = torch.as_tensor(yi.astype(np.float32), device="cuda")
    got = ctx.logreg_eval_csr(Xd, d, y, classes if kp > 1 else classes[:2], W, b)
    assert got[3] == n
    _check(got, X, yi if kp > 1 else yi.clip(0, 1), W, b)


@pytest.mark.parametrize("d,kp", [(3, 1), (1024, 1), (40, 10), (1024, 2)])
def test_eval_matches_dense_pass(ctx, d, kp):
    import torch

    n = 3000
    X = _edge_csr(n, d, seed=5)
    yi, classes = _labels(n, kp, seed=6)
    W, b = _model(d, kp, seed=7)
    y = torch.as_tensor(yi.astype(np.float32), device="cuda")
    cls = classes if kp > 1 else classes[:2]
    got = ctx.logreg_eval_csr(_ingest(ctx, X), d, y, cls, W, b)
    dense = ctx.logreg_eval(torch.as_tensor(X.toarray(), device="cuda"), y, cls, W, b)
    _check(dense, X, yi if kp > 1 else yi.clip(0, 1), W, b)
    bd = so.eval_bound(X, W, b)
    assert abs(got[0] - dense[0]) <= 2 * bd["loss"]
    assert np.all(np.abs(got[1] - dense[1]) <= 2 * bd["dW"])
    assert np.all(np.abs(got[2] - dense[2]) <= 2 * bd["db"])


def _bits(r):
    return (np.float64(r[0]).tobytes(), r[1].tobytes(), r[2].tobytes())


@pytest.mark.parametrize("grid_limit", [1, 3, 7, 0])
def test_eval_bitwise_reproducible(ctx, grid_limit):
    import torch

    n, d, kp = 50000, 5000, 3
    X = so.random_csr(n, d, 20, seed=8, zipf=1.3)
    yi, classes = _labels(n, kp, seed=9)
    W, b = _model(d, kp, seed=10)
    Xd = _ingest(ctx, X)
    y = torch.as_tensor(yi.astype(np.float32), device="cuda")
    ctx.set_option("grid_limit", grid_limit)
    try:
        a = ctx.logreg_eval_csr(Xd, d, y, classes, W, b)
        c = ctx.logreg_eval_csr(Xd, d, y, classes, W, b)
    finally:
        ctx.set_option("grid_limit", 0)
    assert _bits(a) == _bits(c)
    _check(a, X, yi, W, b)


def test_eval_over_row_chunks_with_a_ragged_last_one(ctx):
    import torch

    kp, d = 1024, 8
    n = 2 * so.chunk_rows(kp) + 777   # two full row chunks and a ragged third
    X = so.random_csr(n, d, 3, seed=11)
    yi, classes = _labels(n, kp, seed=12)
    W, b = _model(d, kp, seed=13)
    Xd = _ingest(ctx, X)
    y = torch.as_tensor(yi.astype(np.float32), device="cuda")
    a = ctx.logreg_eval_csr(Xd, d, y, classes, W, b)
    assert _bits(a) == _bits(ctx.logreg_eval_csr(Xd, d, y, classes, W, b))
    _check(a, X, yi, W, b)


SETTING = {"reg": 0.01, "l1_ratio": 0.0, "tol": 1e-12, "max_iter": 1000, "fit_intercept": True,
           "standardization": True, "family": "auto"}


@pytest.mark.parametrize("K,setting", [(2, {}), (3, {"l1_ratio": 0.5}), (2, {"standardization": False,
                                                                              "fit_intercept": False})])
def test_cabi_fit_optimal_and_equal_to_dense_fit(ctx, K, setting):
    import torch

    n, d = 4000, 60
    X = so.random_csr(n, d, 8, seed=14, zipf=1.5)
    rng = np.random.default_rng(15)
    Wt = rng.normal(size=(K, d))
    y = (np.asarray(X @ Wt.T) + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    s = dict(SETTING, **setting)
    yd = torch.as_tensor(y, device="cuda")
    classes, counts, _ = ctx.logreg_labels(yd)
    coef, icpt, _ = ctx.logreg_fit_csr(_ingest(ctx, X), d, yd, classes, counts, [s])[0]
    dcoef, dicpt, _ = ctx.logreg_fit(torch.as_tensor(X.toarray(), device="cuda"), yd, classes, counts, [s])[0]
    prob = lo.Problem(X.toarray(), y, reg=s["reg"], l1_ratio=s["l1_ratio"], fit_intercept=s["fit_intercept"],
                      standardization=s["standardization"])
    np.testing.assert_allclose(so.sigma(X), prob.sig, rtol=1e-10, atol=1e-14)
    theta = np.concatenate([(coef * prob.sig).ravel(), icpt if s["fit_intercept"] else np.zeros(0)])
    assert prob.residual(theta) <= 1e-7
    np.testing.assert_allclose(coef, dcoef, atol=1e-6)
    np.testing.assert_allclose(icpt, dicpt, atol=1e-6)


def _errors(ctx, X, d, y, classes, W=None, b=None):
    from spark_rapids_ml_b200 import _native

    with pytest.raises(_native.B2KError) as e:
        ctx.logreg_eval_csr(X, d, y, classes, np.zeros((1, d)) if W is None else W, np.zeros(1) if b is None else b)
    return e.value


def test_cabi_validation_and_caps(ctx):
    import torch

    from spark_rapids_ml_b200 import _native

    y = torch.zeros(2, dtype=torch.float32, device="cuda")
    y[1] = 1.0
    cls = np.array([0.0, 1.0])

    def csr(indptr, indices, values):
        return (torch.tensor(indptr, dtype=torch.int64, device="cuda"),
                torch.tensor(indices, dtype=torch.int32, device="cuda"),
                torch.tensor(values, dtype=torch.float32, device="cuda"))

    e = _errors(ctx, csr([0, 1, 2], [0, 4], [1.0, 2.0]), 4, y, cls)
    assert e.code == 1 and "out of bounds for vectors of size 4" in str(e)
    e = _errors(ctx, csr([0, 2, 2], [2, 1], [1.0, 2.0]), 4, y, cls)
    assert "strictly increasing" in str(e)
    e = _errors(ctx, csr([0, 1, 2], [1, 1], [np.nan, 2.0]), 4, y, cls)
    assert "NaN or an infinity" in str(e)
    ok = csr([0, 1, 2], [0, 1], [1.0, 2.0])
    big = (1 << 25)   # kp (d + 1) = 2^25 + 1: one past the cap
    with pytest.raises(_native.B2KError) as e:
        ctx.logreg_eval_csr(ok, big, y, cls, np.zeros((1, big)), np.zeros(1))
    assert e.value.code == 4 and "kp (d + 1) <= 33554432" in str(e.value)
    L = _native.load_library()
    for d, msg in [(1 << 31, "d < 2^31")]:   # d = 2^31: one past the cap (no W of that width is formed)
        loss = __import__("ctypes").c_double(0.0)
        rc = L.b2k_logreg_eval_csr(ctx._h, *[a.data_ptr() for a in ok], 2, 2, d, y.data_ptr(), cls.ctypes.data, 2, 1,
                                   np.zeros(1).ctypes.data, np.zeros(1).ctypes.data, __import__("ctypes").byref(loss),
                                   np.zeros(1).ctypes.data, None, ctx._stream())
        assert rc == 4 and msg in L.b2k_last_error(ctx._h).decode()


def _fit_data(n, d, K, seed):
    X = so.random_csr(n, d, 10, seed, zipf=1.4)
    rng = np.random.default_rng(seed)
    W = rng.normal(size=(K, d))
    y = (np.asarray(X @ W.T) + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    return X, y


def _dense_df(X, y, parts=1):
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    return LocalSession().from_numpy(X.toarray(), extra={"label": y}, num_partitions=parts)


def test_estimator_sparse_fit_transform_fit_multiple():
    from spark_rapids_ml_b200.classification import LogisticRegression

    X, y = _fit_data(3000, 300, 3, seed=16)
    sdf = so.vector_frame(X, y, parts=1, dense_rows=[5], max_records=512)
    ddf = _dense_df(X, y)
    lr = LogisticRegression(regParam=0.01, tol=1e-10, num_workers=1)
    ms, md = lr.fit(sdf), lr.fit(ddf)
    np.testing.assert_allclose(ms.coefficientMatrix, md.coefficientMatrix, atol=1e-6)
    np.testing.assert_allclose(ms.intercept_, md.intercept_, atol=1e-6)
    # the transform of a sparse frame (by either model) equals the dense transform within the evaluation bound
    ts = ms.transform(sdf).collect()
    td = ms.transform(ddf).collect()
    xs = md.transform(sdf).collect()
    xd = md.transform(ddf).collect()
    # two fp64 margins of one row in different orders: each within (d + 4) u |w||x| + 16 u of the exact one
    u = 2.0 ** -53
    A = np.asarray(abs(X) @ np.abs(np.asarray(ms.coef_)).T) + np.abs(ms.intercept_)
    tol = 4 * ((X.shape[1] + 4) * u * A.max() + 16 * u)
    for (a, b_), (c, e) in zip(zip(ts, td), zip(xs, xd)):
        for p, q in ((a, b_), (c, e)):
            np.testing.assert_allclose(p["rawPrediction"], q["rawPrediction"], atol=tol, rtol=0)
            np.testing.assert_allclose(p["probability"], q["probability"], atol=tol, rtol=0)
    for p, q in ((ts, td), (xs, xd)):
        assert np.mean([a["prediction"] == b_["prediction"] for a, b_ in zip(p, q)]) > 0.999
    maps = [{lr.regParam: r} for r in (0.0, 0.05)]
    got = dict(lr.fitMultiple(sdf, maps))
    for i, pm in enumerate(maps):
        one = lr.copy(pm).fit(sdf)
        assert got[i].coef_ == one.coef_ and got[i].intercept_ == one.intercept_
    off = LogisticRegression(regParam=0.01, tol=1e-10, num_workers=1, enable_sparse_data_optim=False).fit(sdf)
    assert off.coef_ == md.coef_ and off.intercept_ == md.intercept_


def test_estimator_known_answers_as_sparse_vectors():
    from spark_rapids_ml_b200.classification import LogisticRegression

    for c in json.load(open(os.path.join(ROOT, "tests", "golden", "logreg_known_answers.json")))["cases"]:
        if "data" in c:
            z = np.load(os.path.join(ROOT, "tests", "golden", c["data"]))
            X, y = z["X"], z["y"]
        else:
            X, y = np.array(c["X"], dtype=np.float32), np.array(c["y"], dtype=np.float32)
        Xs = sp.csr_matrix(X)
        if Xs.indptr[1] == 0 or Xs.nnz == 0:
            continue
        m = LogisticRegression(regParam=c["regParam"], elasticNetParam=c["elasticNetParam"],
                               fitIntercept=c["fitIntercept"], standardization=c["standardization"],
                               family=c["family"], num_workers=1).fit(so.vector_frame(Xs, y))
        np.testing.assert_allclose(np.asarray(m.coefficientMatrix), c["coefficientMatrix"], atol=1e-4)
        np.testing.assert_allclose(np.asarray(m.intercept_), c["interceptVector"], atol=1e-4)


def test_estimator_errors():
    import pyarrow as pa

    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.sparkshim.evaluation import MulticlassClassificationEvaluator
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    def frame(rows, y):
        t = pa.Table.from_arrays([pa.array(rows, type=so.VECTOR_TYPE), pa.array(np.asarray(y, np.float32))],
                                 names=["features", "label"])
        return LocalSession().createDataFrame(t)

    lr = LogisticRegression(num_workers=1)
    sv = lambda size, idx, val: {"type": 0, "size": size, "indices": idx, "values": val}   # noqa: E731
    cases = [([sv(4, [0], [1.0]), sv(5, [1], [1.0])], "has size 5, expected 4"),
             ([sv(4, [0], [1.0]), sv(4, [4], [1.0])], "out of bounds for vectors of size 4"),
             ([sv(4, [0], [1.0]), sv(4, [2, 1], [1.0, 2.0])], "strictly increasing"),
             ([sv(4, [0], [1.0]), sv(4, [1], [float("inf")])], "NaN or an infinity"),
             ([sv(4, [0], [1.0]), {"type": 1, "size": None, "indices": None, "values": [1.0, 2.0]}], "expected 4")]
    for rows, msg in cases:
        with pytest.raises(Exception, match=msg):
            lr.fit(frame(rows, [0.0, 1.0]))
    cap = 1 << 25   # binomial: kp (d + 1) = 2^25 + 1
    with pytest.raises(Exception, match="kp \\(d \\+ 1\\) <= 33554432"):
        lr.fit(frame([sv(cap, [0], [1.0]), sv(cap, [cap - 1], [2.0])], [0.0, 1.0]))
    X, y = _fit_data(200, 20, 2, seed=17)
    model = lr.fit(so.vector_frame(X, y))
    with pytest.raises(NotImplementedError, match="sparse input"):
        model._transformEvaluate(so.vector_frame(X, y), MulticlassClassificationEvaluator())


@pytest.mark.parametrize("name", ["binomial_fi1", "binomial_fi0", "multinomial_fi1", "multinomial_fi0"])
def test_estimator_reference_sparse_compat_datasets(name):
    """The reference's test_compat_sparse_binomial / _multinomial rows (a dense row among sparse ones in the binomial
    set), fitted as vector struct frames through the CSR path, against the fp64 oracle's answers
    (tests/golden/make_logreg_sparse_compat.py); the multinomial set also densified (enable_sparse_data_optim=False)."""
    import pyarrow as pa

    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    c = {c["name"]: c for c in json.load(open(os.path.join(ROOT, "tests", "golden", "logreg_sparse_compat.json")))
         ["cases"]}[name]
    t = pa.Table.from_arrays([pa.array(c["rows"], type=so.VECTOR_TYPE), pa.array(np.asarray(c["y"], np.float32))],
                             names=["features", "label"])
    df = LocalSession().createDataFrame(t)
    opts = [None, False] if name.startswith("multinomial") else [None]
    for opt in opts:
        lr = LogisticRegression(regParam=c["regParam"], fitIntercept=c["fitIntercept"],
                                standardization=c["standardization"], tol=1e-12, maxIter=1000, num_workers=1,
                                enable_sparse_data_optim=opt)
        assert lr._pre_process_data(df)[3] == ("csr" if opt is None else "float")
        m = lr.fit(df)
        np.testing.assert_allclose(np.asarray(m.coefficientMatrix), c["coefficientMatrix"], atol=1e-5)
        np.testing.assert_allclose(np.asarray(m.intercept_), c["interceptVector"], atol=1e-5)
