"""Argument checks of the binding, without a GPU: every Context method that hands the library a tensor must reject a
tensor on another device, of another dtype, of another shape or width, or that is not contiguous, naming the argument,
before anything reaches the library.  The library trusts the addresses it receives, so a tensor that slipped through
would be read or written out of bounds on the device.

The Context here has no library context: its device is the CPU, a recorder stands in for _invoke (the one place that
enters a CUDA device), and a recording fake stands in for the library's direct calls."""
import inspect
import re

import numpy as np
import pytest
import torch

from spark_rapids_ml_b200 import _native

N, D = 6, 4


def f32(*s):
    return torch.rand(*s, dtype=torch.float32)


def f64(*s):
    return torch.rand(*s, dtype=torch.float64)


def i32(*s):
    return torch.zeros(*s, dtype=torch.int32)


def i64(*s):
    return torch.zeros(*s, dtype=torch.int64)


def u8(*s):
    return torch.zeros(*s, dtype=torch.uint8)


def labels01(n=N):
    return (torch.arange(n) % 2).to(torch.float32)


def csr(n=4, nnz=6):
    return {"indptr": torch.tensor([0, 2, 3, 5, 6][: n + 1], dtype=torch.int64), "indices": i32(nnz),
            "values": f32(nnz)}


FOREST = {"tree_offsets": [0, 1], "feature": [-1], "threshold": [0.0], "children": [[-1, -1]], "value": [[0.5, 0.5]]}
MODEL = {"kind": "logistic", "W": np.zeros((1, D)), "b": np.zeros(1), "class_values": [0.0, 1.0]}
SETTING = {"reg": 0.0, "l1_ratio": 0.0, "tol": 1e-6, "max_iter": 10, "fit_intercept": True, "standardization": True,
           "family": "auto"}
UMAP = _native.umap_params(n_neighbors=2, n_components=2)
LAYERS = [D, 3, 2]
P = 3 * (D + 1) + 2 * 4


def _vector_batch():
    """The Arrow child buffers of one dense Spark vector row of width D."""
    return (np.ones(1, np.int8), np.zeros(1, np.int32), np.zeros(2, np.int32), np.zeros(0, np.int32),
            np.array([0, D], np.int32), np.ones(D))


# method -> (entry point, valid tensors, the call, wrong shapes, arguments the method converts itself).  A converted
# argument is copied to the device with the dtype the library wants, so only its shape can be wrong.
CASES = {
    "ingest_rows": ("b2k_ingest_append", {"dst": f32(8, D)},
                    lambda c, a: c.ingest_rows(a["dst"], 0, np.zeros(2 * D, np.float32), D),
                    {"dst": f32(8, D - 1)}, ()),
    "ingest_pinned_tensor": ("b2k_ingest_append", {"dst": f32(8, D), "src": f32(2, D)},
                             lambda c, a: c.ingest_pinned_tensor(a["dst"], 0, a["src"]),
                             {"dst": f32(8, D + 1), "src": f32(2 * D)}, ()),
    "ingest_columns": ("b2k_ingest_append", {"dst": f32(8, D)},
                       lambda c, a: c.ingest_columns(a["dst"], 0, [np.zeros(2, np.float32)] * D),
                       {"dst": f32(8, D + 1)}, ()),
    "ingest_csr": ("b2k_ingest_csr_append", csr(),
                   lambda c, a: c.ingest_csr(a["indptr"], a["indices"], a["values"], D, 0, 0, *_vector_batch()),
                   {"indptr": i64(5, 1), "indices": i32(6, 1), "values": f32(7)}, ()),
    "kmeans_fit": ("b2k_kmeans_fit", {"X": f32(N, D), "init": f32(2, D)},
                   lambda c, a: c.kmeans_fit(a["X"], 2, init=a["init"]),
                   {"X": f32(N * D), "init": f32(2, D + 1)}, ("init",)),
    "kmeans_lloyd": ("b2k_kmeans_lloyd", {"X": f32(N, D), "centers": f32(2, D)},
                     lambda c, a: c.kmeans_lloyd(a["X"], a["centers"], 5, 0.0),
                     {"X": f32(N, D, 1), "centers": f32(2, D + 1)}, ()),
    "kmeans_assign": ("b2k_kmeans_assign", {"X": f32(N, D), "centers": f32(2, D)},
                      lambda c, a: c.kmeans_assign(a["X"], a["centers"], want_mindist=True),
                      {"X": f32(N * D), "centers": f32(2, D + 1)}, ("centers",)),
    "pca_fit": ("b2k_pca_fit", {"X": f32(N, D)}, lambda c, a: c.pca_fit(a["X"], 2), {"X": f32(N * D)}, ()),
    "pca_transform": ("b2k_pca_transform", {"X": f32(N, D), "components": f32(2, D)},
                      lambda c, a: c.pca_transform(a["X"], a["components"]),
                      {"X": f32(N * D), "components": f32(2, D - 1)}, ("components",)),
    "knn_search": ("b2k_knn_search", {"items": f32(N, D), "queries": f32(3, D), "item_ids": i64(N)},
                   lambda c, a: c.knn_search(a["items"], a["queries"], 2, a["item_ids"]),
                   {"items": f32(N * D), "queries": f32(3, D + 1), "item_ids": i64(N + 1)}, ()),
    "ivf_search": ("b2k_ivf_search",
                   {"items": f32(N, D), "queries": f32(3, D), "item_ids": i64(N), "centers": f32(2, D)},
                   lambda c, a: c.ivf_search(a["items"], a["queries"], 2, 2, 1, a["item_ids"], a["centers"],
                                             return_lists=True),
                   {"items": f32(N * D), "queries": f32(3, D + 1), "item_ids": i64(N + 1), "centers": f32(3, D)}, ()),
    "linreg_moments": ("b2k_linreg_moments", {"X": f32(N, D), "y": f32(N)},
                       lambda c, a: c.linreg_moments(a["X"], a["y"]), {"X": f32(N * D), "y": f32(N + 1)}, ()),
    "linreg_predict": ("b2k_linreg_predict", {"X": f32(N, D), "coef": f64(D)},
                       lambda c, a: c.linreg_predict(a["X"], a["coef"], 0.5), {"X": f32(N * D), "coef": f64(D + 1)},
                       ("coef",)),
    "gmm_fit": ("b2k_gmm_fit", {"X": f32(N, D)}, lambda c, a: c.gmm_fit(a["X"], 2), {"X": f32(N * D)}, ()),
    "gmm_predict": ("b2k_gmm_predict", {"X": f32(N, D)},
                    lambda c, a: c.gmm_predict(a["X"], np.ones(2) / 2, np.zeros((2, D)), np.stack([np.eye(D)] * 2)),
                    {"X": f32(N * D)}, ()),
    "bkm_fit": ("b2k_bkm_fit", {"X": f32(N, D)}, lambda c, a: c.bkm_fit(a["X"], 2), {"X": f32(N * D)}, ()),
    "bkm_predict": ("b2k_bkm_predict", {"X": f32(N, D)},
                    lambda c, a: c.bkm_predict(a["X"], [1, 2, 3], np.zeros((3, D)), with_cost=True),
                    {"X": f32(N * D)}, ()),
    "mlp_eval": ("b2k_mlp_eval", {"X": f32(N, D), "y": labels01()},
                 lambda c, a: c.mlp_eval(a["X"], a["y"], LAYERS, np.zeros(P)), {"X": f32(N * D), "y": f32(N, 1)}, ()),
    "mlp_fit": ("b2k_mlp_fit", {"X": f32(N, D), "y": labels01()}, lambda c, a: c.mlp_fit(a["X"], a["y"], LAYERS),
                {"X": f32(N * D), "y": f32(N + 1)}, ()),
    "mlp_predict": ("b2k_mlp_predict", {"X": f32(N, D)}, lambda c, a: c.mlp_predict(a["X"], LAYERS, np.zeros(P)),
                    {"X": f32(N * D)}, ()),
    "als_fit": ("b2k_als_fit", {"users": f64(N), "items": f64(N), "ratings": f32(N)},
                lambda c, a: c.als_fit(a["users"], a["items"], a["ratings"], rank=2),
                {"users": f64(N, 1), "items": f64(N + 1), "ratings": f32(N - 1)}, ()),
    "als_predict": ("b2k_als_predict",
                    {"users": f64(3), "items": f64(3), "user_ids": i32(4), "user_factors": f32(4, 2),
                     "item_ids": i32(5), "item_factors": f32(5, 2)},
                    lambda c, a: c.als_predict(a["users"], a["items"], a["user_ids"], a["user_factors"],
                                               a["item_ids"], a["item_factors"]),
                    {"users": f64(3, 1), "items": f64(4), "user_ids": i32(4, 1), "user_factors": f32(3, 2),
                     "item_ids": i32(5, 1), "item_factors": f32(5, 3)}, ()),
    "als_recommend": ("b2k_als_recommend", {"Q": f32(3, 2), "T": f32(5, 2)},
                      lambda c, a: c.als_recommend(a["Q"], a["T"], 2), {"Q": f32(6), "T": f32(5, 3)}, ()),
    "logreg_labels": ("b2k_logreg_labels", {"y": labels01()}, lambda c, a: c.logreg_labels(a["y"]), {"y": f32(N, 1)},
                      ()),
    "logreg_eval": ("b2k_logreg_eval", {"X": f32(N, D), "y": labels01()},
                    lambda c, a: c.logreg_eval(a["X"], a["y"], [0.0, 1.0], np.zeros((1, D)), np.zeros(1)),
                    {"X": f32(N * D), "y": f32(N + 1)}, ()),
    "logreg_fit": ("b2k_logreg_fit", {"X": f32(N, D), "y": labels01()},
                   lambda c, a: c.logreg_fit(a["X"], a["y"], np.array([0.0, 1.0]), np.array([3, 3]), [SETTING]),
                   {"X": f32(N * D), "y": f32(N - 1)}, ()),
    "logreg_predict": ("b2k_logreg_predict", {"X": f32(N, D)},
                       lambda c, a: c.logreg_predict(a["X"], np.zeros((1, D)), np.zeros(1), [0.0, 1.0]),
                       {"X": f32(N * D)}, ()),
    "logreg_eval_csr": ("b2k_logreg_eval_csr", dict(csr(), y=labels01(4)),
                        lambda c, a: c.logreg_eval_csr((a["indptr"], a["indices"], a["values"]), D, a["y"],
                                                       [0.0, 1.0], np.zeros((1, D)), np.zeros(1)),
                        {"indptr": i64(5, 1), "indices": i32(6, 1), "values": f32(5), "y": f32(5)}, ()),
    "logreg_fit_csr": ("b2k_logreg_fit_csr", dict(csr(), y=labels01(4)),
                       lambda c, a: c.logreg_fit_csr((a["indptr"], a["indices"], a["values"]), D, a["y"],
                                                     np.array([0.0, 1.0]), np.array([2, 2]), [SETTING]),
                       {"indptr": i64(5, 1), "indices": i32(6, 1), "values": f32(7), "y": f32(3)}, ()),
    "logreg_predict_csr": ("b2k_logreg_predict_csr", csr(),
                           lambda c, a: c.logreg_predict_csr((a["indptr"], a["indices"], a["values"]), D,
                                                             np.zeros((1, D)), np.zeros(1), [0.0, 1.0]),
                           {"indptr": i64(5, 1), "indices": i32(6, 1), "values": f32(7)}, ()),
    "dbscan_fit": ("b2k_dbscan_fit", {"X": f32(N, D)}, lambda c, a: c.dbscan_fit(a["X"], 0.5, 2), {"X": f32(N * D)},
                   ()),
    "silhouette": ("b2k_silhouette", {"X": f32(N, D), "cluster_ids": i64(N)},
                   lambda c, a: c.silhouette(a["X"], a["cluster_ids"]), {"X": f32(N * D), "cluster_ids": i64(N + 1)},
                   ()),
    "silhouette_multi": ("b2k_silhouette_multi", {"X": f32(N, D), "ids_list[0]": i64(N)},
                         lambda c, a: c.silhouette_multi(a["X"], [a["ids_list[0]"]]),
                         {"X": f32(N * D), "ids_list[0]": i64(N, 1)}, ()),
    "rf_fit": ("b2k_rf_fit", {"X": f32(N, D), "y": labels01()}, lambda c, a: c.rf_fit(a["X"], a["y"]),
               {"X": f32(N * D), "y": f32(N + 1)}, ()),
    "rf_predict": ("b2k_rf_predict", {"X": f32(N, D)}, lambda c, a: c.rf_predict(a["X"], FOREST, True),
                   {"X": f32(N * D)}, ()),
    "eval_linear": ("b2k_eval_linear", {"X": f32(N, D), "y": labels01()},
                    lambda c, a: c.eval_linear(a["X"], a["y"], [MODEL]), {"X": f32(N * D), "y": f32(N + 1)}, ()),
    "eval_forest": ("b2k_eval_forest", {"X": f32(N, D), "y": labels01()},
                    lambda c, a: c.eval_forest(a["X"], a["y"], [FOREST], True), {"X": f32(N * D), "y": f32(N + 1)},
                    ()),
    "binary_scores_linear": ("b2k_eval_linear_scores",
                             {"X": f32(N, D), "y": labels01(), "scores": f64(2, N + 2), "pos": u8(N + 2)},
                             lambda c, a: c.binary_scores_linear(a["X"], a["y"], [MODEL, MODEL], a["scores"], a["pos"],
                                                                 2),
                             {"X": f32(N * D), "y": f32(N + 1), "scores": f64(3, N + 2), "pos": u8(N + 1)}, ()),
    "binary_scores_forest": ("b2k_eval_forest_scores",
                             {"X": f32(N, D), "y": labels01(), "scores": f64(2, N), "pos": u8(N)},
                             lambda c, a: c.binary_scores_forest(a["X"], a["y"], [FOREST, FOREST], a["scores"],
                                                                 a["pos"]),
                             {"X": f32(N * D), "y": f32(N + 1), "scores": f64(3, N), "pos": u8(N + 1)}, ()),
    "eval_binary": ("b2k_eval_binary", {"scores": f64(2, N), "pos": u8(N)},
                    lambda c, a: c.eval_binary(a["scores"], a["pos"], 10, "areaUnderROC"),
                    {"scores": f64(2 * N), "pos": u8(N + 1)}, ()),
    "umap_fit": ("b2k_umap_fit", {"X": f32(N, D), "labels": i32(N)},
                 lambda c, a: c.umap_fit(a["X"], UMAP, labels=a["labels"]), {"X": f32(N * D), "labels": i32(N + 1)},
                 ()),
    "umap_transform": ("b2k_umap_transform", {"X_train": f32(N, D), "embedding": f32(N, 2), "Q": f32(3, D)},
                       lambda c, a: c.umap_transform(a["X_train"], a["embedding"], a["Q"], UMAP),
                       {"X_train": f32(N * D), "embedding": f32(N, 3), "Q": f32(3, D + 1)}, ()),
}

_OTHER_DTYPE = {torch.float32: torch.float64, torch.float64: torch.float32, torch.int32: torch.int64,
                torch.int64: torch.int32, torch.uint8: torch.int32}


def _faults(x):
    """Tensors like x (at least 2 wide in every dimension) that are each wrong in one way."""
    strided = torch.empty(tuple(reversed(x.shape)), dtype=x.dtype).t() if x.dim() == 2 else \
        torch.empty(2 * x.shape[0], dtype=x.dtype)[::2]
    assert not strided.is_contiguous() and strided.shape == x.shape
    return {"device": torch.empty(x.shape, dtype=x.dtype, device="meta"), "dtype": x.to(_OTHER_DTYPE[x.dtype]),
            "contiguous": strided}


class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, fn, *args, after=()):
        self.calls.append(fn)
        return 0


class _FakeLib:
    """The library's direct (stream-less) calls: each is recorded and succeeds with its outputs left zero."""

    def __init__(self, calls):
        self._calls = calls

    def __getattr__(self, name):
        def call(*args):
            self._calls.append(name)
            return 0
        return call


class _Stream:
    def synchronize(self):
        pass


@pytest.fixture
def ctx(monkeypatch):
    c = _native.Context.__new__(_native.Context)
    c._torch = torch
    c.device = torch.device("cpu")
    c.device_index = 0
    c._h = None
    c._invoke = _Recorder()
    c.direct = []
    c._L = _FakeLib(c.direct)
    # a method that keeps a temporary alive synchronises the device's stream after its call
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
    return c


def _fault_cases():
    for method, (_, tensors, _, shapes, converted) in CASES.items():
        for name, x in tensors.items():
            if name not in converted:
                for fault in _faults(x):
                    yield method, name, fault
            if name in shapes:
                yield method, name, "shape"


def test_the_table_covers_every_method_that_reaches_the_library():
    reach = re.compile(r"self\._(call|invoke|logreg_eval|logreg_fit)\(")
    methods = {name for name, fn in vars(_native.Context).items()
               if not name.startswith("_") and callable(fn) and reach.search(inspect.getsource(fn))}
    assert methods == set(CASES)
    for method, (_, tensors, _, shapes, _) in CASES.items():
        assert set(shapes) <= set(tensors), method


@pytest.mark.parametrize("method", sorted(CASES))
def test_valid_call_reaches_the_library_once(ctx, method):
    entry, tensors, call, _, _ = CASES[method]
    call(ctx, dict(tensors))
    assert ctx._invoke.calls == [entry]


@pytest.mark.parametrize("method,name,fault", list(_fault_cases()))
def test_bad_tensor_is_rejected_before_the_library(ctx, method, name, fault):
    _, tensors, call, shapes, _ = CASES[method]
    args = dict(tensors)
    args[name] = shapes[name] if fault == "shape" else _faults(tensors[name])[fault]
    with pytest.raises(ValueError, match=rf"^{re.escape(name)}(?!\w)"):
        call(ctx, args)
    assert ctx._invoke.calls == [] and ctx.direct == []


@pytest.mark.parametrize("offsets", [[], [-D, 0], [-1, D - 1], [D, 3 * D], [0, D, 2 * D, 3 * D]])
def test_ingest_rows_keeps_offsets_within_values(ctx, offsets):
    """The library reads values[offsets[0]:offsets[-1]] and checks only that each row is d wide: offsets that start
    before the buffer or end past it would make it read host memory outside the buffer."""
    values = np.zeros(2 * D, np.float32)
    with pytest.raises(ValueError, match="^offsets"):
        ctx.ingest_rows(f32(8, D), 0, values, D, offsets=np.array(offsets, np.int32))
    assert ctx._invoke.calls == []
    ctx.ingest_rows(f32(8, D), 0, values, D, offsets=np.array([D, 2 * D], np.int32))   # a sliced list: one row
    assert ctx._invoke.calls == ["b2k_ingest_append"]


def test_comm_init_checks_the_unique_id_length(ctx):
    with pytest.raises(ValueError, match="^uid"):
        ctx.comm_init(2, 0, b"x" * (_native.UNIQUE_ID_BYTES - 1))
    assert ctx.direct == []
