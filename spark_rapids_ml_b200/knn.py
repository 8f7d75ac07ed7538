"""NearestNeighbors / NearestNeighborsModel — the reference's exact k-NN surface (python/src/spark_rapids_ml/knn.py:76-804),
with cuML NearestNeighborsMG replaced by b2k_knn_search (hand-written sm_90a CUDA behind include/b2kmeans.h).

  NearestNeighborsClass (k -> n_neighbors, defaults)                  knn.py:76-86
  _NearestNeighborsCumlParams (k, idCol, inputCol(s), _ensureIdCol)   knn.py:89-200
  NearestNeighbors (lazy fit, no persistence)                         knn.py:203-408
  NearestNeighborsModel.kneighbors and its fit function               knn.py:511-804

Semantics: Euclidean distance on float32 rows; per query the k items with the smallest distance, ascending, ties to the
lower global row (rank-major ingest order); the distance reported is sqrt of the exact fp32 sum (q_f - x_f)^2 in feature
order, so a query equal to an item reports 0.0.  Indices are the item ids of idCol; without idCol a `unique_id` column of
monotonically increasing ids is added (an existing `unique_id` column is then an error).

Differences that are deliberate: the fit function splits the device matrix into items and queries by the label slot and
maps rows to ids on the device, where the reference all-gathers every item id as JSON through the barrier context
(knn.py:723-796).  exactNearestNeighborsJoin, approximate search and kneighbors on a pyspark DataFrame raise
NotImplementedError.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import pyarrow as pa

from .core import FitInputType, _CumlCaller, _CumlEstimator, _CumlModel, alias, param_alias
from .params import HasIDCol, HasInputCol, HasInputCols, HasLabelCol, P, _CumlClass, _CumlParams
from .sparkshim import HAVE_PYSPARK, LocalDataFrame, Param, TypeConverters, keyword_only
from .utils import get_logger

_NO_PERSIST = "does not support saving/loading, just re-create the estimator."


class NearestNeighborsClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {"k": "n_neighbors"}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_neighbors": 5, "verbose": False, "batch_size": 2000000}


class _NearestNeighborsCumlParams(_CumlParams, HasInputCol, HasLabelCol, HasInputCols, HasIDCol):
    """Shared Spark Params of NearestNeighbors and NearestNeighborsModel (reference: knn.py:89-200)."""

    k = Param("parent", "k", "The number nearest neighbors to retrieve. Must be >= 1.", TypeConverters.toInt)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(idCol=None, k=5)

    def setK(self: P, value: int) -> P:
        return self._set_params(k=value)

    def getK(self) -> int:
        return self.getOrDefault("k")

    def setIdCol(self: P, value: str) -> P:
        return self._set_params(idCol=value)

    def _getIdColOrDefault(self) -> str:
        res = self.getIdCol()
        return alias.row_number if res is None else res

    def setInputCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(inputCol=value)
        else:
            self._set_params(inputCols=value)
        return self

    def setInputCols(self: P, value: List[str]) -> P:
        return self._set_params(inputCols=value)

    def getInputCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.inputCols):
            return self.getOrDefault(self.inputCols)
        if self.isDefined(self.inputCol):
            return self.getOrDefault(self.inputCol)
        raise RuntimeError("inputCol is not set")

    def _ensureIdCol(self, df: LocalDataFrame) -> LocalDataFrame:
        """The frame with its id column: idCol when set and present; else a monotonically increasing `unique_id`
        (reference knn.py:170-200, including its error on a pre-existing `unique_id` when idCol is unset)."""
        id_col_name = self.getIdCol()
        if id_col_name is None and alias.row_number in df.columns:
            raise ValueError(f"Trying to create an id column with default name {alias.row_number}. "
                             "But a column with the same name already exists.")
        if id_col_name is not None and id_col_name in df.columns:
            return df
        get_logger(self.__class__).info(f"idCol not set or absent: adding an id column named {alias.row_number}.")
        return df.with_monotonically_increasing_id(alias.row_number)

    def _validate_k(self) -> int:
        k = self.cuml_params.get("n_neighbors")
        if isinstance(k, bool) or not isinstance(k, int) or k < 1:
            raise ValueError(f"k given invalid value {k} (must be >= 1)")
        return k


def _no_pyspark(dataset: Any) -> None:
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError("kneighbors on a pyspark DataFrame is not supported yet; use a local frame")


class NearestNeighbors(NearestNeighborsClass, _CumlEstimator, _NearestNeighborsCumlParams):
    """Exact k nearest neighbours on H100 (reference: knn.py:203-408).  fit() is lazy: the model keeps the item frame
    with its ids; kneighbors() runs one barrier task per GPU.  Parameters: k (default 5), inputCol (str for an array
    column, list of str for scalar columns), idCol, num_workers, verbose.  batch_size is accepted and unused.

    >>> from spark_rapids_ml_b200.knn import NearestNeighbors
    >>> items = session.createDataFrame([(0, [1.0, 1.0]), (1, [2.0, 2.0]), (2, [3.0, 3.0])], "id int, features array<float>")
    >>> queries = session.createDataFrame([(3, [1.0, 1.0]), (4, [3.0, 3.0])], "id int, features array<float>")
    >>> model = NearestNeighbors(k=2).setInputCol("features").setIdCol("id").fit(items)
    >>> model.kneighbors(queries)[2].collect()   # query_id 3: indices [0, 1], distances [0.0, 1.4142135]
    """

    @keyword_only
    def __init__(self, *, k: Optional[int] = None, inputCol: Optional[Union[str, List[str]]] = None,
                 idCol: Optional[str] = None, num_workers: Optional[int] = None, verbose: Union[int, bool] = False,
                 **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        if not self._input_kwargs.get("float32_inputs", True):
            get_logger(self.__class__).warning("This estimator does not support double precision inputs. Setting "
                                               "float32_inputs to False will be ignored.")
            self._input_kwargs.pop("float32_inputs")
        for name in ("k", "inputCol", "idCol", "num_workers"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        self._set_params(**self._input_kwargs)
        self._label_isdata = 0
        self._label_isquery = 1
        self._set_params(labelCol=alias.label)

    def _fit(self, item_df: LocalDataFrame) -> "NearestNeighborsModel":
        _no_pyspark(item_df)
        self._validate_k()
        item_df_withid = self._ensureIdCol(item_df)
        processed = item_df_withid.with_constant_column(alias.label, self._label_isdata)
        model = NearestNeighborsModel(item_df_withid, processed, self._label_isdata, self._label_isquery)
        model._num_workers = self._num_workers
        model._float32_inputs = self._float32_inputs
        self._copyValues(model)
        self._copy_cuml_params(model)
        return model

    def _out_schema(self) -> Any:   # fit is lazy: no barrier task runs here
        return None

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None) -> Any:
        return None

    def _create_pyspark_model(self, result: Any) -> Any:
        raise NotImplementedError("NearestNeighbors.fit builds its model directly")

    def write(self) -> Any:
        raise NotImplementedError(f"NearestNeighbors {_NO_PERSIST}")

    @classmethod
    def read(cls) -> Any:
        raise NotImplementedError(f"NearestNeighbors {_NO_PERSIST}")

    def save(self, path: str, overwrite: bool = False) -> None:
        raise NotImplementedError(f"NearestNeighbors {_NO_PERSIST}")

    @classmethod
    def load(cls, path: str) -> Any:
        raise NotImplementedError(f"NearestNeighbors {_NO_PERSIST}")


class NearestNeighborsModel(_CumlCaller, _CumlModel, NearestNeighborsClass, _NearestNeighborsCumlParams):
    """reference: knn.py:511-804."""

    def __init__(self, item_df_withid: LocalDataFrame, processed_item_df: LocalDataFrame, label_isdata: int,
                 label_isquery: int) -> None:
        super().__init__()
        self._item_df_withid = item_df_withid
        self._processed_item_df = processed_item_df
        self._label_isdata = label_isdata
        self._label_isquery = label_isquery

    def _out_schema(self, input_schema: Any = None) -> Any:
        return None

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None) -> Any:
        raise NotImplementedError("NearestNeighborsModel does not provide a transform function. Use 'kneighbors'.")

    def _transform(self, dataset: Any) -> Any:
        raise NotImplementedError("NearestNeighborsModel does not provide a transform function. Use 'kneighbors'.")

    def exactNearestNeighborsJoin(self, query_df: Any, distCol: str = "distCol") -> Any:
        raise NotImplementedError("exactNearestNeighborsJoin needs DataFrame joins, which the local frame lacks")

    def approxNearestNeighbors(self, *args: Any, **kwargs: Any) -> Any:
        raise NotImplementedError("approxNearestNeighbors is not provided: use ApproximateNearestNeighbors")

    def write(self) -> Any:
        raise NotImplementedError(f"NearestNeighborsModel {_NO_PERSIST}")

    @classmethod
    def read(cls) -> Any:
        raise NotImplementedError(f"NearestNeighborsModel {_NO_PERSIST}")

    def save(self, path: str, overwrite: bool = False) -> None:
        raise NotImplementedError(f"NearestNeighborsModel {_NO_PERSIST}")

    @classmethod
    def load(cls, path: str) -> Any:
        raise NotImplementedError(f"NearestNeighborsModel {_NO_PERSIST}")

    def _pre_process_data(self, dataset: LocalDataFrame) -> Tuple[LocalDataFrame, Optional[List[str]], int, str]:
        """The feature columns as for every estimator, plus the label and the id (as alias.row_number) per row
        (reference knn.py:540-572)."""
        df, multi_col_names, dimension, ftype = super()._pre_process_data(dataset)
        id_col = self._getIdColOrDefault()
        for src, dst in ((alias.label, alias.label), (id_col, alias.row_number)):
            df = df.with_appended_column(dst, [[b.column(src).cast(pa.int64()) for b in p] for p in dataset._parts])
        return df, multi_col_names, dimension, ftype

    def kneighbors(self, query_df: LocalDataFrame, sort_knn_df_by_query_id: bool = True
                   ) -> Tuple[LocalDataFrame, LocalDataFrame, LocalDataFrame]:
        """(item_df_withid, query_df_withid, knn_df): knn_df has one row per query with columns query_<id>, indices
        (array<long> of item ids) and distances (array<float>, ascending)."""
        _no_pyspark(query_df)
        k = self._validate_k()
        id_col = self._getIdColOrDefault()
        query_df_withid = self._ensureIdCol(query_df)
        qname = f"query_{id_col}"
        if query_df_withid.count() == 0:
            schema = pa.schema([(qname, pa.int64()), ("indices", pa.list_(pa.int64())),
                                ("distances", pa.list_(pa.float32()))])
            return self._item_df_withid, query_df_withid, LocalDataFrame(query_df.sparkSession, [[]], schema)
        processed_query = query_df_withid.with_constant_column(alias.label, self._label_isquery)
        input_col, input_cols = self._get_input_columns()
        cols = [id_col, alias.label] + ([input_col] if input_col is not None else list(input_cols))
        union_df = self._processed_item_df.select(cols).union(processed_query.select(cols)).repartition(self.num_workers)
        res = self._call_cuml_fit_func(union_df, partially_collect=False)
        table = res._table()
        if table.num_rows and sort_knn_df_by_query_id:
            table = table.sort_by(qname)
        return self._item_df_withid, query_df_withid, res._derive([table.to_batches()], table.schema)

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        self._validate_k()

    def _search(self, ctx: Any, items: Any, queries: Any, ids: Any, params: Dict[str, Any]) -> Tuple[Any, Any]:
        return ctx.knn_search(items, queries, int(params["n_neighbors"]), ids)

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        label_isdata, label_isquery = self._label_isdata, self._label_isquery
        qname = f"query_{self._getIdColOrDefault()}"
        search = self._search

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for NearestNeighborsMG(handle).kneighbors(...) and the row -> id mapping (knn.py:662-804)
            import torch

            ctx = params[param_alias.handle]
            X, label, row_number = dfs[0]
            is_item = label == label_isdata
            is_query = label == label_isquery
            sel = lambda m: torch.from_numpy(np.nonzero(m)[0]).to(X.device)   # noqa: E731
            items = X.index_select(0, sel(is_item)).contiguous()
            queries = X.index_select(0, sel(is_query)).contiguous()
            ids = torch.from_numpy(np.ascontiguousarray(row_number[is_item])).to(X.device)
            dist, idx = search(ctx, items, queries, ids, params[param_alias.cuml_init])
            return {qname: row_number[is_query], "indices": list(idx.cpu().numpy()),
                    "distances": list(dist.cpu().numpy())}

        return _cuml_fit


# ---- approximate search: IVF-Flat (reference knn.py:838-1723) ----
_IVF_KEYS = {"nlist": "nlist", "n_lists": "nlist", "nprobe": "nprobe", "n_probes": "nprobe",
             "kmeans_n_iters": "kmeans_n_iters", "kmeans_trainset_fraction": "kmeans_trainset_fraction"}
_IVF_DEFAULTS = {"nlist": 1024, "nprobe": 20, "kmeans_n_iters": 20, "kmeans_trainset_fraction": 0.5}


def _check_algorithm(value: Optional[str]) -> None:
    if value in ("ivfpq", "cagra"):
        raise ValueError(f"algorithm '{value}' is not supported yet; use 'ivfflat'")
    if value != "ivfflat":
        raise ValueError(f"algorithm must be 'ivfflat' (got {value!r})")


def _ivf_params(algo_params: Optional[Dict[str, Any]]) -> Dict[str, Any]:
    """algoParams with the reference's aliases resolved (nlist / n_lists, nprobe / n_probes) and defaults filled in."""
    out = dict(_IVF_DEFAULTS)
    for key, v in (algo_params or {}).items():
        if key not in _IVF_KEYS:
            raise ValueError(f"algoParams key '{key}' is not supported by ivfflat (supported: {sorted(_IVF_KEYS)})")
        out[_IVF_KEYS[key]] = v
    return out


def _check_metric(value: str) -> None:
    if value not in ("euclidean", "l2", "sqeuclidean"):
        raise ValueError(f"metric '{value}' is not supported by ivfflat (supported: euclidean, l2, sqeuclidean)")


def _to_dict(v: Any) -> Any:
    return v if v is None or isinstance(v, dict) else dict(v)


class ApproximateNearestNeighborsClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {"k": "n_neighbors", "algorithm": "algorithm", "metric": "metric", "algoParams": "algo_params"}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_neighbors": 5, "verbose": False, "algorithm": "ivfflat", "metric": "euclidean", "algo_params": None}


class _ApproximateNearestNeighborsParams(_NearestNeighborsCumlParams):
    """reference: knn.py:861-935."""

    algorithm = Param("parent", "algorithm", "The algorithm to use for approximate nearest neighbors search.",
                      TypeConverters.toString)
    algoParams = Param("parent", "algoParams", "The parameters to use to set up a neighbor algorithm.", _to_dict)
    metric = Param("parent", "metric", "The distance metric to use.", TypeConverters.toString)

    def _set_ann_defaults(self) -> None:   # the estimator and the model run NearestNeighbors(Model).__init__
        self._setDefault(algorithm="ivfflat", algoParams=None, metric="euclidean")

    def setAlgorithm(self: P, value: str) -> P:
        _check_algorithm(value)
        return self._set_params(algorithm=value)

    def getAlgorithm(self) -> str:
        return self.getOrDefault("algorithm")

    def setAlgoParams(self: P, value: Dict[str, Any]) -> P:
        return self._set_params(algoParams=value)

    def getAlgoParams(self) -> Dict[str, Any]:
        return self.getOrDefault("algoParams")

    def setMetric(self: P, value: str) -> P:
        _check_metric(value)
        return self._set_params(metric=value)

    def getMetric(self) -> str:
        return self.getOrDefault("metric")

    def _validate_ann(self) -> Dict[str, Any]:
        _check_algorithm(self.cuml_params.get("algorithm"))
        _check_metric(self.cuml_params.get("metric"))
        return _ivf_params(self.cuml_params.get("algo_params"))


class ApproximateNearestNeighbors(ApproximateNearestNeighborsClass, _ApproximateNearestNeighborsParams,
                                  NearestNeighbors):
    """Approximate k nearest neighbours, IVF-Flat, on H100 (reference: knn.py:938-1217).  fit() is lazy, as for
    NearestNeighbors; kneighbors() builds one index over all items (one coarse quantizer trained on a subset of every
    GPU's items, see include/b2kmeans.h b2k_ivf_search) and probes the nprobe nearest lists of each query.  The
    reference builds one index per partition instead, so its results depend on the partitioning; these do not.

    algoParams: nlist / n_lists (default 1024), nprobe / n_probes (default 20, clamped to nlist), kmeans_n_iters
    (default 20), kmeans_trainset_fraction (default 0.5).  metric: euclidean, l2 or sqeuclidean.  Queries that find
    fewer than k items report +inf past the found ones, with the first id (or 2^63 - 1 when nothing was found).

    >>> items = session.createDataFrame([(i, [float(i), float(i)]) for i in range(6)], "id int, features array<float>")
    >>> knn = ApproximateNearestNeighbors(k=2).setInputCol("features").setIdCol("id")
    >>> model = knn.setAlgoParams({"nlist": 2, "nprobe": 1}).fit(items)
    """

    @keyword_only
    def __init__(self, *, k: Optional[int] = None, algorithm: str = "ivfflat",
                 metric: str = "euclidean", algoParams: Optional[Dict[str, Any]] = None,
                 inputCol: Optional[Union[str, List[str]]] = None, idCol: Optional[str] = None,
                 num_workers: Optional[int] = None, verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        _check_algorithm(algorithm)
        _check_metric(metric)
        kw = dict(self._input_kwargs)
        NearestNeighbors.__init__.__wrapped__(self, **{key: v for key, v in kw.items()
                                                      if key not in ("algorithm", "metric", "algoParams")})
        self._set_ann_defaults()
        for key in ("algorithm", "metric", "algoParams"):
            if key in kw:
                self._set_params(**{key: kw[key]})

    def _fit(self, item_df: LocalDataFrame) -> "ApproximateNearestNeighborsModel":
        _no_pyspark(item_df)
        self._validate_k()
        item_df_withid = self._ensureIdCol(item_df)
        processed = item_df_withid.with_constant_column(alias.label, self._label_isdata)
        model = ApproximateNearestNeighborsModel(item_df_withid, processed, self._label_isdata, self._label_isquery)
        model._num_workers = self._num_workers
        model._float32_inputs = self._float32_inputs
        self._copyValues(model)
        self._copy_cuml_params(model)
        return model

    def write(self) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighbors {_NO_PERSIST}")

    @classmethod
    def read(cls) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighbors {_NO_PERSIST}")

    def save(self, path: str, overwrite: bool = False) -> None:
        raise NotImplementedError(f"ApproximateNearestNeighbors {_NO_PERSIST}")

    @classmethod
    def load(cls, path: str) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighbors {_NO_PERSIST}")


class ApproximateNearestNeighborsModel(ApproximateNearestNeighborsClass, _ApproximateNearestNeighborsParams,
                                       NearestNeighborsModel):
    """reference: knn.py:1219-1723.  kneighbors shares NearestNeighborsModel's barrier task over the union frame; only
    the search it runs differs."""

    def __init__(self, item_df_withid: LocalDataFrame, processed_item_df: LocalDataFrame, label_isdata: int,
                 label_isquery: int) -> None:
        NearestNeighborsModel.__init__(self, item_df_withid, processed_item_df, label_isdata, label_isquery)
        self._set_ann_defaults()

    def exactNearestNeighborsJoin(self, query_df: Any, distCol: str = "distCol") -> Any:
        raise NotImplementedError("ApproximateNearestNeighborsModel has no exactNearestNeighborsJoin")

    def approxSimilarityJoin(self, query_df: Any, distCol: str = "distCol") -> Any:
        raise NotImplementedError("approxSimilarityJoin needs DataFrame joins, which the local frame lacks")

    def write(self) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighborsModel {_NO_PERSIST}")

    @classmethod
    def read(cls) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighborsModel {_NO_PERSIST}")

    def save(self, path: str, overwrite: bool = False) -> None:
        raise NotImplementedError(f"ApproximateNearestNeighborsModel {_NO_PERSIST}")

    @classmethod
    def load(cls, path: str) -> Any:
        raise NotImplementedError(f"ApproximateNearestNeighborsModel {_NO_PERSIST}")

    def kneighbors(self, query_df: LocalDataFrame, sort_knn_df_by_query_id: bool = True
                   ) -> Tuple[LocalDataFrame, LocalDataFrame, LocalDataFrame]:
        self._validate_ann()
        return super().kneighbors(query_df, sort_knn_df_by_query_id)

    def _search(self, ctx: Any, items: Any, queries: Any, ids: Any, params: Dict[str, Any]) -> Tuple[Any, Any]:
        ivf = _ivf_params(params["algo_params"])
        dist, idx, _ = ctx.ivf_search(items, queries, int(params["n_neighbors"]), int(ivf["nlist"]),
                                      int(ivf["nprobe"]), ids, n_iters=int(ivf["kmeans_n_iters"]),
                                      train_fraction=float(ivf["kmeans_trainset_fraction"]), metric=params["metric"])
        return dist, idx
