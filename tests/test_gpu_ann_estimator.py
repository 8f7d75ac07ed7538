"""ApproximateNearestNeighbors end to end on local frames, against the fp64 IVF oracle with the trained centres found
again by a direct search on the same items."""
import json
import os

import numpy as np
import pytest

import ann_oracle as ao

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200.knn import ApproximateNearestNeighbors  # noqa: E402
from spark_rapids_ml_b200.sparkshim import LocalSession  # noqa: E402


def _frames(session, X, Q, cols=False):
    if cols:
        names = [f"c{j}" for j in range(X.shape[1])]
        items = session.createDataFrame([(i, *map(float, r)) for i, r in enumerate(X)], ["id"] + names)
        queries = session.createDataFrame([(100 + i, *map(float, r)) for i, r in enumerate(Q)], ["id"] + names)
        return items, queries, names
    items = session.createDataFrame([(i, r.tolist()) for i, r in enumerate(X)], "id int, features array<float>")
    queries = session.createDataFrame([(100 + i, r.tolist()) for i, r in enumerate(Q)], "id int, features array<float>")
    return items, queries, "features"


def _golden(case):
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ann_known_answers.json")) as f:
        return json.load(f)[case]


@pytest.mark.parametrize("case", ["docstring", "return_fewer_k"])
def test_known_answers(case):
    # the reference's docstring example and test_return_fewer_k (tests/golden/make_ann_known_answers.py)
    ka = _golden(case)
    session = LocalSession()
    items = session.createDataFrame([(i, v) for i, v in ka["items"]], "id int, features array<float>")
    queries = session.createDataFrame([(i, v) for i, v in ka["queries"]], "id int, features array<float>")
    knn = ApproximateNearestNeighbors(k=ka["k"], algoParams=ka["algoParams"]).setInputCol("features").setIdCol("id")
    _, _, knn_df = knn.fit(items).kneighbors(queries)
    rows = sorted(knn_df.collect(), key=lambda r: r["query_id"])
    assert [list(r["indices"]) for r in rows] == ka["indices"]
    np.testing.assert_allclose([list(r["distances"]) for r in rows], ka["distances"], rtol=1e-6)


@pytest.mark.parametrize("with_id", [False, True])
def test_example_one_list_probed_twice(with_id):
    # the reference's test_example: ivfflat with nlist 1, nprobe 2 (clamped to 1) is the exact search
    ka = _golden("docstring")
    session = LocalSession()
    items = session.createDataFrame([(i, v) for i, v in ka["items"]], "id int, features array<float>")
    queries = session.createDataFrame([(i, v) for i, v in ka["queries"]], "id int, features array<float>")
    params = {"nlist": 1, "nprobe": 2}
    knn = ApproximateNearestNeighbors(algorithm="ivfflat", algoParams=params, k=2).setInputCol("features")
    if with_id:
        knn = knn.setIdCol("id")
    model = knn.fit(items)
    for obj in (knn, model):
        assert obj.cuml_params["algorithm"] == "ivfflat" and obj.cuml_params["algo_params"] == params
    _, _, knn_df = model.kneighbors(queries)
    qname = "query_id" if with_id else "query_unique_id"
    rows = sorted(knn_df.collect(), key=lambda r: r[qname])
    ids = [[0, 1], [5, 4]]
    if not with_id:   # unique ids of the items in frame order
        item_ids = [r["unique_id"] for r in model._item_df_withid.collect()]
        ids = [[item_ids[i] for i in row] for row in ids]
    assert [list(r["indices"]) for r in rows] == ids
    np.testing.assert_allclose([list(r["distances"]) for r in rows], [[0, 1.4142134], [0, 14.142137]], rtol=1e-6)


@pytest.mark.parametrize("cols,metric,with_id", [(False, "euclidean", True), (True, "sqeuclidean", True),
                                                 (False, "l2", False)])
def test_against_oracle(cols, metric, with_id):
    session = LocalSession()
    rng = np.random.default_rng(1)
    X = rng.normal(size=(800, 8)).astype(np.float32)
    Q = rng.normal(size=(50, 8)).astype(np.float32)
    items, queries, col = _frames(session, X, Q, cols)
    knn = ApproximateNearestNeighbors(k=4, metric=metric, algoParams={"nlist": 8, "nprobe": 3}).setInputCol(col)
    if with_id:
        knn = knn.setIdCol("id")
    _, qdf, knn_df = knn.fit(items).kneighbors(queries)
    qname = "query_id" if with_id else "query_unique_id"
    rows = sorted(knn_df.collect(), key=lambda r: r[qname])
    idx = np.array([list(r["indices"]) for r in rows])
    dist = np.array([list(r["distances"]) for r in rows])
    from spark_rapids_ml_b200 import _native
    with _native.Context(0) as ctx:
        _, _, C, lists, probes = ctx.ivf_search(torch.from_numpy(X).cuda(), torch.from_numpy(Q).cuda(), 4, 8, 3,
                                                return_lists=True)
    assert ao.check_lists(X, C.cpu().numpy(), lists.cpu().numpy()) == 0
    bad = ao.check_result(X, Q, 4, lists.cpu().numpy(), probes.cpu().numpy(), dist, idx,
                          squared=metric == "sqeuclidean")
    assert bad == {"n_outside_margin": 0, "n_fill": 0}
