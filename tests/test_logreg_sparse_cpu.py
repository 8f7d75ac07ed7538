"""Sparse logistic regression without a GPU: which path a vector struct column takes (enable_sparse_data_optim None,
False, True), the struct column handling (densify, widths, nulls), other estimators' refusal of struct columns, and the
sparse fp64 oracle against the dense one (and the host optimiser on it)."""
import numpy as np
import pyarrow as pa
import pytest
import scipy.sparse as sp

import logreg_oracle as lo
import logreg_sparse_oracle as so


def _data(n=60, d=7, seed=0):
    X = so.random_csr(n, d, 3, seed)
    X[5, :] = 0.0
    X.eliminate_zeros()
    X[6] = sp.csr_matrix(np.arange(1, d + 1, dtype=np.float32))   # a full row
    X = sp.csr_matrix(X)
    X.data[0] = 0.0   # a stored zero stays an entry
    y = (np.random.default_rng(seed).random(n) < 0.5).astype(np.float32)
    return X, y


def _fit_frame(lr, df):
    """What the fit scaffold sees: the pre-processed frame and its feature type."""
    out, multi, dim, ftype = lr._pre_process_data(df)
    return out, dim, ftype


def test_path_rule_for_none_false_true():
    from spark_rapids_ml_b200.classification import LogisticRegression

    X, y = _data()
    sparse_first = so.vector_frame(X, y)
    dense_first = so.vector_frame(X, y, dense_rows=[0])
    _, dim, ftype = _fit_frame(LogisticRegression(), sparse_first)
    assert (dim, ftype) == (7, "csr")
    _, dim, ftype = _fit_frame(LogisticRegression(), dense_first)
    assert (dim, ftype) == (7, "float")
    out, dim, ftype = _fit_frame(LogisticRegression(enable_sparse_data_optim=False), sparse_first)
    assert (dim, ftype) == (7, "float")
    got = np.array([r for b in out._parts[0] for r in b.column(0).to_pylist()], dtype=np.float32)
    np.testing.assert_array_equal(got, X.toarray())
    with pytest.raises(ValueError, match="leave it at None"):
        LogisticRegression(enable_sparse_data_optim=True)


def test_densify_mixed_rows_and_stored_zeros():
    from spark_rapids_ml_b200.utils import densify_vector_column

    X, _ = _data()
    arr = so.vector_array(X, dense_rows=[1, 2, 9])
    got = np.array(densify_vector_column(arr.slice(1, 40), 7).to_pylist(), dtype=np.float32)
    np.testing.assert_array_equal(got, X.toarray()[1:41])


def test_struct_column_buffers_zero_copy_and_widths():
    import pandas as pd

    from spark_rapids_ml_b200.utils import arrow_vector_column_buffers, densify_vector_column, is_vector_struct

    X, _ = _data()
    arr = so.vector_array(X, dense_rows=[3]).slice(2, 10)
    assert is_vector_struct(arr.type) and not is_vector_struct(pa.list_(pa.float32()))
    t, size, io, iv, vo, vv = arrow_vector_column_buffers(pd.Series(pd.arrays.ArrowExtensionArray(arr)))
    assert t.tolist() == [0] + [1] + [0] * 8 and size[1] == 0 and (size[[0, 2]] == 7).all()
    lens = np.diff(vo)
    assert lens[1] == 7 and list(lens[2:]) == [X.indptr[i + 1] - X.indptr[i] for i in range(4, 12)]
    # the child buffers are the whole Arrow buffers, located by the offsets
    assert vv[vo[0]:vo[-1]].size == lens.sum()
    bad = pa.array([{"type": 0, "size": 5, "indices": [0], "values": [1.0]}], type=so.VECTOR_TYPE)
    with pytest.raises(ValueError, match="different sizes"):
        densify_vector_column(bad, 7)
    with pytest.raises(ValueError, match="null feature rows"):
        arrow_vector_column_buffers(pd.Series(pd.arrays.ArrowExtensionArray(pa.array([None], type=so.VECTOR_TYPE))))


def test_other_estimators_still_refuse_struct_columns():
    from spark_rapids_ml_b200.classification import RandomForestClassifier
    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.regression import LinearRegression

    X, y = _data()
    df = so.vector_frame(X, y)
    for est in (KMeans(k=2), LinearRegression(), RandomForestClassifier()):
        with pytest.raises(ValueError, match="VectorUDT columns need pyspark"):
            est._pre_process_data(df)


def test_cross_validator_refuses_sparse_input_before_any_fit():
    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder
    from spark_rapids_ml_b200.sparkshim.evaluation import MulticlassClassificationEvaluator

    X, y = _data()
    lr = LogisticRegression()
    cv = CrossValidator(estimator=lr, estimatorParamMaps=ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.1]).build(),
                        evaluator=MulticlassClassificationEvaluator(), numFolds=2)
    with pytest.raises(NotImplementedError, match="sparse input"):
        cv.fit(so.vector_frame(X, y))


@pytest.mark.parametrize("kp", [1, 3])
def test_sparse_oracle_equals_dense_oracle(kp):
    X, y = _data(80, 9, seed=3)
    rng = np.random.default_rng(kp)
    yi = rng.integers(0, max(kp, 2), size=80)
    yi[0] = -1
    W, b = rng.normal(size=(kp, 9)), rng.normal(size=kp)
    Xd = X.toarray().astype(np.float64)
    l1, g1, h1 = so.loss_grad(X, yi, W, b)
    l2, g2, h2 = lo.loss_grad(Xd, yi, W, b)
    assert abs(l1 - l2) <= 1e-14 * max(1.0, abs(l2))
    np.testing.assert_allclose(g1, g2, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(h1, h2, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(so.sigma(X), lo.sigma(Xd), rtol=1e-12, atol=1e-15)
    bs, bd = so.eval_bound(X, W, b), lo.eval_bound(Xd, W, b)
    assert np.isclose(bs["loss"], bd["loss"], rtol=1e-12)
    np.testing.assert_allclose(bs["dW"], bd["dW"], rtol=1e-12)
    np.testing.assert_allclose(bs["db"], bd["db"], rtol=1e-12)


def test_host_optimiser_on_the_sparse_oracle():
    from spark_rapids_ml_b200 import _native

    X, y = _data(200, 6, seed=4)
    prob = lo.Problem(X.toarray(), y, reg=0.01)
    inv = prob.inv

    def fun(theta):
        V, b = prob.split(theta)
        loss, gW, gb = so.loss_grad(X, prob.yi, V * inv, b)
        return loss + 0.5 * prob.l2 * float((prob.pen * V * V).sum()), np.concatenate([(gW * inv + prob.l2 * prob.pen
                                                                                         * V).ravel(), gb])

    theta, iters, _, _ = _native.logreg_minimize(fun, prob.start(), max_iter=1000, tol=1e-12)
    assert prob.residual(theta) <= 1e-8
