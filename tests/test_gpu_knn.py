"""Exact k-NN on the GPU: b2k_knn_search against the fp64 oracle under the parity rule (tests/knn_oracle.py), both search
paths, splits, determinism, errors, and NearestNeighbors.kneighbors on the reference's known answers."""
import json
import os

import numpy as np
import pytest

import knn_oracle as ko

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200 import _native  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "knn_known_answers.json")


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


def _search(ctx, X, Q, k, path=0, ids=None, grid=0):
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid)
    try:
        dist, idx = ctx.knn_search(torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda(), k,
                                   None if ids is None else torch.from_numpy(ids).cuda())
        return dist.cpu().numpy(), idx.cpu().numpy(), ctx.stats()["last_path"]
    finally:
        ctx.set_option("kernel_path", 0)
        ctx.set_option("grid_limit", 0)


def _data(n, nq, d, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) + offset).astype(np.float32)
    Q = (rng.normal(size=(nq, d)) + offset).astype(np.float32)
    return X, Q


@pytest.mark.parametrize("d", [2, 20, 64, 128])
@pytest.mark.parametrize("k", [1, 5, 32, 64, 65])
def test_search_matches_oracle(ctx, d, k):
    X, Q = _data(3001, 299, d, seed=d * 100 + k)
    dist, idx, path = _search(ctx, X, Q, k)
    assert path == (2 if d % 4 == 0 and k <= 64 else 1)
    bad = ko.compare(X, Q, k, dist, idx)
    assert bad["n_outside_margin"] == 0, bad


@pytest.mark.parametrize("d", [20, 128])
def test_paths_agree_and_report(ctx, d):
    X, Q = _data(2000, 333, d, seed=5)
    dw, iw, pw = _search(ctx, X, Q, 16, path=2)
    dg, ig, pg = _search(ctx, X, Q, 16, path=1)
    assert (pw, pg) == (2, 1)
    for dist, idx in ((dw, iw), (dg, ig)):
        assert ko.compare(X, Q, 16, dist, idx)["n_outside_margin"] == 0
    assert np.mean(iw == ig) > 0.99   # both exact up to near-ties


def test_few_queries_split_index(ctx):
    # 5 queries: one query tile, so the index is split over many units (S > 1); S = 1 with one CTA
    X, Q = _data(20011, 5, 128, seed=1)
    d_many, i_many, _ = _search(ctx, X, Q, 10)
    d_one, i_one, _ = _search(ctx, X, Q, 10, grid=1)
    assert ko.compare(X, Q, 10, d_many, i_many)["n_outside_margin"] == 0
    np.testing.assert_array_equal(i_many, i_one)
    np.testing.assert_array_equal(d_many, d_one)


@pytest.mark.parametrize("path", [1, 2])
def test_duplicates_and_exact_hits(ctx, path):
    X, _ = _data(1000, 1, 64, seed=2)
    X = np.concatenate([X, X[:300], X[:300]])   # every one of the first 300 items three times
    Q = X[[0, 5, 299, 700, 999]].copy()
    dist, idx, _ = _search(ctx, X, Q, 3, path=path)
    assert np.all(dist[:, 0] == 0.0)
    for i, r in enumerate([0, 5, 299]):
        assert idx[i].tolist() == [r, r + 1000, r + 1300] and np.all(dist[i] == 0.0)
    assert idx[3, 0] == 700 and idx[4, 0] == 999
    assert ko.compare(X, Q, 3, dist, idx)["n_outside_margin"] == 0


@pytest.mark.parametrize("path", [1, 2])
def test_offset_data(ctx, path):
    # ||q||^2 + ||x||^2 - 2 q.x cancels badly at a 1e3 offset; the reported distance is the exact fp32 sum
    X, Q = _data(4000, 200, 128, seed=3, offset=1e3)
    Q[:10] = X[:10]
    dist, idx, _ = _search(ctx, X, Q, 8, path=path)
    assert np.all(dist[:10, 0] == 0.0)
    assert ko.compare(X, Q, 8, dist, idx)["n_outside_margin"] == 0


def test_ids_and_determinism(ctx):
    X, Q = _data(5000, 700, 128, seed=4)
    ids = np.arange(5000, dtype=np.int64) * 7 + 1000
    d1, i1, _ = _search(ctx, X, Q, 64, ids=ids)
    d2, i2, _ = _search(ctx, X, Q, 64, ids=ids)
    np.testing.assert_array_equal(d1, d2)
    np.testing.assert_array_equal(i1, i2)
    assert ko.compare(X, Q, 64, d1, i1, ids)["n_outside_margin"] == 0


def test_errors(ctx):
    X, Q = _data(10, 3, 8, seed=0)
    for k in (0, 11):
        with pytest.raises(_native.B2KError):
            _search(ctx, X, Q, k)
    with pytest.raises(_native.B2KError):
        _search(ctx, X[:, :6].copy(), Q[:, :6].copy(), 5, path=2)   # d % 4 != 0: no wgmma path
    with pytest.raises(_native.B2KError):
        _search(ctx, np.zeros((2000, 4), np.float32), Q[:, :4].copy(), 1025)
    d, i, _ = _search(ctx, X, Q[:0].copy(), 5)
    assert d.shape == (0, 5) and i.shape == (0, 5)


# ---- estimator surface on the reference's known answers ----
def _known():
    with open(GOLDEN) as f:
        return json.load(f)


def _session():
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "2"})


@pytest.mark.parametrize("layout", ["array", "scalar"])
@pytest.mark.parametrize("with_id", [False, True])
def test_kneighbors_known_answers(layout, with_id):
    from spark_rapids_ml_b200.knn import NearestNeighbors

    ka = _known()
    spark = _session()
    items = [r[0] for r in ka["items"]]
    queries = [r[0] for r in ka["queries"]]
    if layout == "array":
        rows_i = [(101 + i, x, m) for i, (x, m) in enumerate(ka["items"])]
        rows_q = [(201 + i, x, m) for i, (x, m) in enumerate(ka["queries"])]
        schema = "id long, features array<float>, metadata string"
    else:
        rows_i = [(101 + i, x[0], x[1], m) for i, (x, m) in enumerate(ka["items"])]
        rows_q = [(201 + i, x[0], x[1], m) for i, (x, m) in enumerate(ka["queries"])]
        schema = "id long, f1 float, f2 float, metadata string"
    if not with_id:
        rows_i = [r[1:] for r in rows_i]
        rows_q = [r[1:] for r in rows_q]
        schema = schema.split(", ", 1)[1]
    item_df = spark.createDataFrame(rows_i, schema)
    query_df = spark.createDataFrame(rows_q, schema)
    est = NearestNeighbors(num_workers=1).setInputCol("features" if layout == "array" else ["f1", "f2"])
    if with_id:
        est = est.setIdCol("id")
    est = est.setK(ka["k"])
    model = est.fit(item_df)
    _, _, empty = model.kneighbors(spark.createDataFrame([], schema))
    assert empty.count() == 0
    item_withid, query_withid, knn_df = model.kneighbors(query_df)
    idc = "id" if with_id else "unique_id"
    item_ids = [r[idc] for r in item_withid.collect()]
    query_ids = [r[idc] for r in query_withid.collect()]
    rows = knn_df.collect()
    assert [r[f"query_{idc}"] for r in rows] == sorted(query_ids)
    by_q = {r[f"query_{idc}"]: r for r in rows}
    for qi, qid in enumerate(query_ids):
        r = by_q[qid]
        assert list(r["indices"]) == [item_ids[j] for j in ka["indices"][qi]]
        np.testing.assert_allclose(r["distances"], ka["distances"][qi], rtol=1e-6)
    assert len(items) == 8 and len(queries) == 5


def test_kneighbors_two_workers_match_one():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from spark_rapids_ml_b200.knn import NearestNeighbors

    spark = _session()
    X, Q = _data(3000, 257, 32, seed=9)
    item_df = spark.from_numpy(X, num_partitions=2, extra={"id": np.arange(3000, dtype=np.int64)})
    query_df = spark.from_numpy(Q, num_partitions=2, extra={"id": np.arange(257, dtype=np.int64) + 10 ** 6})
    out = []
    for w in (1, 2):
        model = NearestNeighbors(num_workers=w, k=7).setInputCol("features").setIdCol("id").fit(item_df)
        rows = model.kneighbors(query_df)[2].collect()
        out.append(([list(r["indices"]) for r in rows], [list(r["distances"]) for r in rows]))
    assert out[0] == out[1]
