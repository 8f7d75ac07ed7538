"""Driver- and executor-side fit/transform scaffolding for the KMeans path.

Mirrors the reference's contract (python/src/spark_rapids_ml/core.py):
  * _CumlCaller._pre_process_data      core.py:463-562   select/cast feature columns, infer dimension
  * _CumlCaller._call_cuml_fit_func    core.py:742-1013  repartition(num_workers), build the pickled
                                                         `_train_udf`, run it as ONE BARRIER TASK PER GPU
                                                         through mapInPandas
  * _train_udf                         core.py:845-1003  BarrierTaskContext, GPU select, ingest, CumlContext
                                                         (NCCL uid over allGather), call
                                                         cuml_fit_func(inputs, params), barrier, partition 0
                                                         yields the model rows
  * _CumlEstimator._fit_internal       core.py:1230-1281 collect rows, merge chunks, build the model
  * _CumlModel(WithColumns)._transform core.py:1797-1941 per-batch predict appended as predictionCol
  * persistence                        core.py:268-355   metadata JSON + model-attribute JSON under path/data

What is re-designed (GPU-first): the executor never stacks Python objects or concatenates on the host —
each Arrow batch goes host -> pinned -> HBM once through b2k_ingest_append into a device-resident matrix
(utils.DeviceRowAppender), and `inputs` handed to the fit function are device tensors.  The internal hook keeps
the reference's signature: cuml_fit_func(inputs: List[Tuple[X, None, None]], params: Dict) -> Dict[str, list].
"""
from __future__ import annotations

import json
import os
import threading
import uuid
from abc import abstractmethod
from collections import namedtuple
from typing import Any, Callable, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple, Union

import numpy as np
import pandas as pd
import pyarrow as pa

from .params import _CumlParams
from .sparkshim import (HAVE_PYSPARK, BarrierTaskContext, EstimatorBase, LocalDataFrame, ModelBase, Params, Row,
                        get_session)
from .utils import DeviceCsrAppender, DeviceRowAppender, arrow_list_column_buffers, get_logger

# same tags as the reference (core.py:128-175) so the worker-side column contract is recognisable
Alias = namedtuple("Alias", ("featureVectorType", "featureVectorSize", "featureVectorIndices", "data", "label",
                             "row_number"))
col_name_unique_tag = "c3BhcmstcmFwaWRzLW1sCg=="
alias = Alias(f"vector_type_{col_name_unique_tag}", f"vector_size_{col_name_unique_tag}",
              f"vector_indices_{col_name_unique_tag}", f"cuml_values_{col_name_unique_tag}", "cuml_label",
              "unique_id")
Pred = namedtuple("Pred", ("prediction", "probability", "model_index", "raw_prediction"))
pred = Pred("prediction", "probability", "model_index", "raw_prediction")
ParamAlias = namedtuple("ParamAlias", ("cuml_init", "handle", "num_cols", "part_sizes", "loop",
                                       "fit_multiple_params", "mem_config"))
param_alias = ParamAlias("cuml_init", "handle", "num_cols", "part_sizes", "loop", "fit_multiple_params",
                         "mem_config")

FitInputType = List[Tuple[Any, Optional[Any], Optional[Any]]]
_CumlFitFunc = Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]


class _CumlCommon:
    """reference: core.py:359-432."""

    @staticmethod
    def _get_gpu_device(context: Any, is_local: bool, is_transform: bool = False) -> int:
        import torch

        if is_local:
            # local mode: partitionId doubles as the GPU id (core.py:377-384); transform wraps around
            n = max(1, torch.cuda.device_count())
            pid = context.partitionId() if context is not None else 0
            return pid % n if is_transform else pid
        from .utils import _get_gpu_id

        return _get_gpu_id(context)

    @staticmethod
    def _set_gpu_device(context: Any, is_local: bool, is_transform: bool = False) -> int:
        import torch

        gpu_id = _CumlCommon._get_gpu_device(context, is_local, is_transform)
        torch.cuda.set_device(gpu_id)
        return gpu_id


def _feature_columns(arrays: Sequence[Any]) -> List[np.ndarray]:
    """Scalar feature columns as the library ingests them.  Columns that share one of its source dtypes go over as
    they are, and the device converts them to float32.  Any other set (mixed dtypes, unsigned, boolean) is converted
    on the host column by column: each column's astype(float32) rounds every value once from that column's own type,
    exactly as the device would, so the matrix equals ingesting each column alone.  A common type first would not:
    int64 -> float64 -> float32 rounds twice, and int64 -> int8 or float64 -> int64 truncates."""
    from ._native import _DTYPE_CODES

    cols = [np.ascontiguousarray(a) for a in arrays]
    dt = cols[0].dtype
    if dt in _DTYPE_CODES and all(c.dtype == dt for c in cols):
        return cols
    with np.errstate(over="ignore"):   # beyond float32's range is +-inf, as on the device
        return [np.ascontiguousarray(c, dtype=np.float32) for c in cols]


def _features_from_pdf(pdf: pd.DataFrame, multi_col_names: Optional[List[str]], appender: DeviceRowAppender,
                       logger: Any) -> int:
    """One Arrow batch -> rows of the device matrix.  Fast path: the Arrow child buffer, zero-copy.
    Compat path (classic Spark conversion: object column of ndarrays): host stacking, as core.py:916 does."""
    n_b = int(pdf.shape[0])
    if n_b == 0:
        return 0
    if multi_col_names:
        appender.append_columns(_feature_columns([pdf[c].to_numpy() for c in multi_col_names]))
        return n_b
    col = pdf[alias.data]
    bufs = arrow_list_column_buffers(col, appender.d)
    if bufs is not None:
        vals, offsets, n_rows = bufs
        appender.append_values(vals, offsets, n_rows)
    else:
        stacked = np.array(list(col), order="C")  # reference idiom (core.py:916): slow, kept for compatibility
        if stacked.ndim != 2:
            raise ValueError("feature rows have different lengths")
        if stacked.shape[1] != appender.d:
            raise ValueError(f"feature rows are {stacked.shape[1]} wide, expected {appender.d}")
        if stacked.dtype not in (np.float32, np.float64):
            stacked = stacked.astype(np.float32)
        appender.append_values(np.ascontiguousarray(stacked).reshape(-1), None, n_b)
    return n_b


def _append_transform_features(app: DeviceRowAppender, df: Union[pd.DataFrame, np.ndarray], n_cols: int) -> None:
    """One transform input batch -> rows of the device matrix: the Arrow child buffer of the feature column (zero-copy),
    an object column of ndarrays (stacked on the host), scalar feature columns, or a plain array."""
    n_b = len(df)
    if isinstance(df, pd.DataFrame) and alias.data in df.columns:
        col = df[alias.data]
        bufs = arrow_list_column_buffers(col, n_cols)
        if bufs is not None:
            app.append_values(bufs[0], bufs[1], bufs[2])
        else:
            stacked = np.ascontiguousarray(np.array(list(col), order="C"), dtype=np.float32)
            if stacked.ndim != 2 or stacked.shape[1] != n_cols:
                raise ValueError(f"feature rows do not match the model's {n_cols} columns")
            app.append_values(stacked.reshape(-1), None, n_b)
    elif isinstance(df, pd.DataFrame):
        if len(df.columns) != n_cols:
            raise ValueError(f"{len(df.columns)} feature columns do not match the model's {n_cols}")
        app.append_columns(_feature_columns([df[c].to_numpy() for c in df.columns]))
    else:
        arr = np.ascontiguousarray(df, dtype=np.float32)
        if arr.ndim != 2 or arr.shape[1] != n_cols:
            raise ValueError(f"feature rows do not match the model's {n_cols} columns")
        app.append_values(arr.reshape(-1), None, n_b)


_TRANSFORM_CONTEXTS: Dict[int, Any] = {}
_TRANSFORM_CONTEXTS_LOCK = __import__("threading").Lock()


def _transform_context(gpu: int) -> Any:
    """One library context per (process, GPU) for transform tasks: a Spark Python worker is reused across tasks, and a
    context's set-up (stream, pinned staging buffers, scratch, copy threads) costs more than labelling a small
    partition.  Released at interpreter exit."""
    from . import _native

    with _TRANSFORM_CONTEXTS_LOCK:
        ctx = _TRANSFORM_CONTEXTS.get(gpu)
        if ctx is None:
            ctx = _native.Context(gpu)
            _TRANSFORM_CONTEXTS[gpu] = ctx
            if len(_TRANSFORM_CONTEXTS) == 1:
                import atexit

                atexit.register(_close_transform_contexts)
        return ctx


def _close_transform_contexts() -> None:
    with _TRANSFORM_CONTEXTS_LOCK:
        for ctx in _TRANSFORM_CONTEXTS.values():
            try:
                ctx.close()
            except Exception:
                pass
        _TRANSFORM_CONTEXTS.clear()


class _DeviceModel:
    """A model placed on one GPU for transform and evaluation: the process's context for that GPU and the model's
    arrays, uploaded once with their NumPy dtype."""

    def __init__(self, gpu: int, **arrays: np.ndarray) -> None:
        import torch

        self.ctx = _transform_context(gpu)
        self.arrays = {k: torch.from_numpy(np.ascontiguousarray(a)).to(self.ctx.device) for k, a in arrays.items()}

    def close(self) -> None:   # the context (pinned staging, scratch, copy threads) stays with the process
        self.arrays = {}


_ARROW_SCALARS = {"int": pa.int32(), "float": pa.float32(), "double": pa.float64()}


def _out_dtype(out_type: str) -> Any:
    """The NumPy dtype of an output type's values: "int" / "double", or the element of "array<float>" / "array<double>"."""
    return _ARROW_SCALARS[out_type[len("array<"):-1] if out_type.startswith("array<") else out_type].to_pandas_dtype()


def _transform_result_array(res: np.ndarray, out_type: str) -> pa.Array:
    """One output of one frame as the Arrow array of its type: one value per row ("int", "double") or, from a 2-D
    array, one fixed-width vector per row ("array<float>", "array<double>")."""
    if out_type.startswith("array<"):
        elem = _ARROW_SCALARS[out_type[len("array<"):-1]]
        vals = np.ascontiguousarray(res, dtype=elem.to_pandas_dtype()).reshape(-1)
        offsets = np.arange(len(res) + 1, dtype=np.int32) * np.int32(res.shape[1])
        return pa.ListArray.from_arrays(pa.array(offsets), pa.array(vals, type=elem))
    return pa.array(np.asarray(res, dtype=_out_dtype(out_type)), type=_ARROW_SCALARS[out_type])


def _ingest(ctx: Any, frames: Iterable[Any], n_cols: int, rows: int) -> Any:
    """Every non-empty frame, in order, as the rows of one device matrix (`rows` in all)."""
    app = DeviceRowAppender(ctx, n_cols, first_capacity=max(1, rows))
    for f in frames:
        if len(f):
            _append_transform_features(app, f, n_cols)
    return app.finish()


def _ingest_csr(ctx: Any, frames: Iterable[Any], n_cols: int) -> Any:
    """Every non-empty frame's vector struct column, in order, as the rows of one device CSR."""
    app = DeviceCsrAppender(ctx, n_cols)
    for f in frames:
        if len(f):
            app.append_column(f[alias.data])
    return app.finish()


def _vector_bytes(frame: Any) -> int:
    """The device bytes of a frame's vector struct column as CSR entries: 12 per stored value."""
    from .utils import _arrow_array

    arr = _arrow_array(frame[alias.data])
    offs = arr.flatten()[3].offsets
    return 12 * (int(offs[-1].as_py()) - int(offs[0].as_py())) if len(arr) else 0


class _GroupedTransform:
    """A model's transform function: a group of frames in one device pass.  Every non-empty frame is ingested into one
    device matrix, `predict(device_model, X)` returns one CUDA tensor per output type (the first dimension is the row),
    each output is read back once, and each frame gets its rows of every output, in order.  A group without rows makes
    no device call: its frames get zero-length outputs of each type's dtype.  `row_bytes`, the device bytes per row,
    bounds a group's size (TRANSFORM_GROUP_BYTES)."""

    def __init__(self, predict: Callable[[Any, Any], Sequence[Any]], n_cols: int, row_bytes: int,
                 out_types: Sequence[str], sparse: bool = False) -> None:
        self.predict = predict
        self.n_cols = n_cols
        self.row_bytes = row_bytes
        self.out_types = list(out_types)
        # sparse: the frames' features are a vector struct column, ingested as one device CSR (indptr, indices,
        # values); `row_bytes` then counts the bytes per row of the outputs and groups are also capped by the entries'
        # bytes (12 per stored entry)
        self.sparse = sparse

    def __call__(self, model: Any, frames: List[Any]) -> List[Tuple[np.ndarray, ...]]:
        sizes = [len(f) for f in frames]
        total = sum(sizes)
        if total == 0:
            return [tuple(np.zeros((0, 0) if t.startswith("array<") else 0, _out_dtype(t)) for t in self.out_types)
                    for _ in frames]
        X = _ingest_csr(model.ctx, frames, self.n_cols) if self.sparse else _ingest(model.ctx, frames, self.n_cols, total)
        host = [t.cpu().numpy() for t in self.predict(model, X)]
        ends = np.cumsum(sizes)
        return [tuple(h[e - n:e] for h in host) for n, e in zip(sizes, ends)]


def _select_features(batches: Iterable[pa.RecordBatch], input_col: Optional[str],
                     input_cols: Optional[List[str]]) -> Iterator[pa.RecordBatch]:
    """The feature columns of each batch, a single one renamed to alias.data at the Arrow level (zero-copy)."""
    for b in batches:
        yield b.select(list(input_cols)) if input_cols else b.select([input_col]).rename_columns([alias.data])



class _CumlCaller(_CumlParams, _CumlCommon):
    """reference: core.py:435-1019."""

    def __init__(self) -> None:
        super().__init__()
        self._initialize_cuml_params()

    # -- hooks a concrete estimator provides --
    @abstractmethod
    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None) -> _CumlFitFunc:
        raise NotImplementedError

    @abstractmethod
    def _out_schema(self) -> Any:
        raise NotImplementedError

    def _require_nccl_ucx(self) -> Tuple[bool, bool]:
        return (True, False)  # collectives only (core.py:564-571)

    def _fit_array_order(self) -> str:
        return "C"

    def _fit_label_col(self) -> Optional[str]:
        """The label column of a supervised estimator: the pre-processed frame carries it as alias.label, and the fit
        function receives it in slot 2 as a float32 device vector.  None: slot 2 is whatever alias.label the frame
        carries (kneighbors' item / query tags), as int64 host values."""
        return None

    def _validate_parameters(self) -> None:
        """reference round-trips the params through the JVM estimator (core.py:579-602); without a JVM the
        same constraints are checked here."""
        cp = self.cuml_params
        if "n_clusters" in cp and not (isinstance(cp["n_clusters"], int) and cp["n_clusters"] > 1):
            raise ValueError(f"k given invalid value {cp['n_clusters']} (must be > 1)")
        if "max_iter" in cp and cp["max_iter"] < 0:
            raise ValueError(f"maxIter given invalid value {cp['max_iter']}")
        if "tol" in cp and cp["tol"] < 0:
            raise ValueError(f"tol given invalid value {cp['tol']}")

    def _pre_process_data(self, dataset: LocalDataFrame) -> Tuple[LocalDataFrame, Optional[List[str]], int, str]:
        """-> (selected/cast dataframe, multi_col_names, dimension, feature dtype).  The frame holds the features of
        _pre_process_features and, when _fit_label_col() names one, the label cast to float32 as alias.label."""
        label = self._fit_label_col()
        if label is not None and label not in dataset.columns:
            raise ValueError(f"label column '{label}' not found in {dataset.columns}")
        df, multi_col_names, dimension, ftype = self._pre_process_features(dataset)
        if label is not None:
            df = df.with_appended_column(alias.label,
                                         [[b.column(label).cast(pa.float32()) for b in p] for p in dataset._parts])
        return df, multi_col_names, dimension, ftype

    def _pre_process_features(self, dataset: LocalDataFrame) -> Tuple[LocalDataFrame, Optional[List[str]], int, str]:
        """The feature columns selected and cast -> (dataframe, multi_col_names, dimension, feature dtype)."""
        input_col, input_cols = self._get_input_columns()
        types = dict(dataset.dtypes)
        if input_col is not None:
            if input_col not in types:
                raise ValueError(f"features column '{input_col}' not found in {dataset.columns}")
            t = types[input_col]
            if not t.startswith("array<"):
                raise ValueError(f"column '{input_col}' has type {t}; expected array<float|double> "
                                 "(VectorUDT columns need pyspark)")
            df = dataset.select(input_col).withColumnRenamed(input_col, alias.data)
            inner = t[len("array<"):-1]
            if inner == "double" and self._float32_inputs:
                df = df.cast_column(alias.data, pa.list_(pa.float32()))   # core.py:489-495
                inner = "float"
            elif inner not in ("float", "double"):
                df = df.cast_column(alias.data, pa.list_(pa.float32() if self._float32_inputs else pa.float64()))
                inner = "float" if self._float32_inputs else "double"
            first = df.first()
            if first is None:
                raise RuntimeError("A python worker received no data.  Please increase amount of data or use fewer workers.")
            dimension = len(first[alias.data])
            return df, None, dimension, inner
        assert input_cols is not None
        for c in input_cols:
            if c not in types:
                raise ValueError(f"features column '{c}' not found in {dataset.columns}")
        df = dataset.select(*input_cols)
        for c in input_cols:  # core.py:543-557 casts every scalar column
            want = pa.float32() if (self._float32_inputs or types[c] not in ("double",)) else pa.float64()
            if types[c] == "double" and not self._float32_inputs:
                want = pa.float64()
            df = df.cast_column(c, want)
        return df, list(input_cols), len(input_cols), "float"

    def _call_cuml_fit_func(self, dataset: Any, partially_collect: bool = True,
                            paramMaps: Optional[Sequence[Dict[Any, Any]]] = None) -> Any:
        """Local frames: one barrier task per partition through the shim.  pyspark DataFrames (pyspark importable):
        the reference's plan — mapInPandas(_train_udf).rdd.barrier().mapPartitions — through spark_binding; returns
        the collected model rows in that case."""
        self._validate_parameters()
        cls = self.__class__
        spark_df = False
        if HAVE_PYSPARK:
            from . import spark_binding

            spark_df = spark_binding.is_spark_dataframe(dataset)
        num_workers = self.num_workers
        if spark_df:
            df, multi_col_names, dimension, ftype = spark_binding.pre_process_data(self, dataset, alias.data)
            is_local = spark_binding.is_local(dataset)
        else:
            df, multi_col_names, dimension, ftype = self._pre_process_data(dataset)
            if df.getNumPartitions() != num_workers:
                df = df.repartition(num_workers)   # core.py:771-772
            is_local = True   # the local frame runs on this host: partition id doubles as the GPU id (core.py:377-384)
        # "csr": the features are Spark vectors kept sparse; the fit function gets the device CSR triple in slot 0
        csr = ftype == "csr"
        params: Dict[str, Any] = {param_alias.cuml_init: dict(self.cuml_params), param_alias.fit_multiple_params: None}
        extra_cols = [c for c in (alias.label, alias.row_number) if c in df.columns]
        float_label = self._fit_label_col() is not None
        cuml_fit_func = self._get_cuml_fit_func(dataset, None)
        (enable_nccl, require_ucx) = self._require_nccl_ucx()
        cuml_verbose = self.cuml_params.get("verbose", False)

        def _train_udf(pdf_iter: Iterator[pd.DataFrame]) -> Iterator[pd.DataFrame]:
            from spark_rapids_ml_b200 import _native
            from spark_rapids_ml_b200.common.cuml_context import CumlContext
            from spark_rapids_ml_b200.sparkshim import BarrierTaskContext as _BTC

            logger = get_logger(cls)
            if spark_df:
                from spark_rapids_ml_b200 import spark_binding as _sb

                context = _sb.current_barrier_context()
            else:
                context = _BTC.get()
            partition_id = context.partitionId()
            gpu_id = _CumlCommon._set_gpu_device(context, is_local)
            logger.info("Loading data into device memory (b2k_ingest_append)")
            with CumlContext(partition_id, num_workers, context, enable_nccl, require_ucx, device=gpu_id) as cc:
                appender = DeviceCsrAppender(cc.handle, dimension) if csr else DeviceRowAppender(cc.handle, dimension)
                sizes: List[int] = []
                # label / row-number columns the pre-processed frame carries (kneighbors): host arrays, per batch
                extra: Dict[str, List[np.ndarray]] = {c: [] for c in extra_cols}
                for pdf in pdf_iter:
                    sizes.append(appender.append_column(pdf[alias.data]) if csr else
                                 _features_from_pdf(pdf, multi_col_names, appender, logger))
                    for c in extra_cols:
                        if float_label and c == alias.label:
                            extra[c].append(np.asarray(pdf[c].to_numpy(), dtype=np.float32))
                        else:
                            extra[c].append(np.asarray(pdf[c].to_numpy(), dtype=np.int64))
                if len(sizes) == 0 or all(sz == 0 for sz in sizes):
                    raise RuntimeError(
                        "A python worker received no data.  Please increase amount of data or use fewer workers.")
                X = appender.finish()
                slots = [np.concatenate(extra[c]) if c in extra else None for c in (alias.label, alias.row_number)]
                if float_label:
                    import torch

                    slots[0] = torch.from_numpy(slots[0]).to(cc.handle.device)
                inputs: FitInputType = [(X, slots[0], slots[1])]
                params[param_alias.handle] = cc.handle
                params[param_alias.part_sizes] = sizes
                params[param_alias.num_cols] = dimension
                params[param_alias.loop] = cc._loop
                params[param_alias.mem_config] = {"cuda_managed_mem_enabled": False, "cuda_system_mem_enabled": False,
                                                  "cuda_system_mem_headroom": None}
                logger.info("Invoking fit")
                import signal

                if hasattr(signal, "SIGHUP"):
                    try:
                        signal.signal(signal.SIGHUP, signal.SIG_DFL)  # core.py:975-981
                    except ValueError:
                        pass  # not the main thread (in-process single-partition run)
                result = cuml_fit_func(inputs, params)
                logger.info("Fit complete")
            if partially_collect:
                if enable_nccl:
                    context.barrier()
                if context.partitionId() == 0:
                    yield pd.DataFrame(data=result)
            else:
                yield pd.DataFrame(data=result)

        if spark_df:
            return spark_binding.run_barrier_fit(df, _train_udf, self._out_schema(), num_workers)
        return df.mapInPandas(_train_udf, schema=self._out_schema(), barrier=True)


class _CumlEstimator(EstimatorBase, _CumlCaller):
    """reference: core.py:1067-1311."""

    def __init__(self) -> None:
        super().__init__()
        self.logger = get_logger(self.__class__)

    @abstractmethod
    def _create_pyspark_model(self, result: Row) -> "_CumlModel":
        raise NotImplementedError

    def _merge_model_chunks(self, rows: List[Row], paramMaps: Optional[Sequence[Dict[Any, Any]]] = None) -> List[Row]:
        return rows

    def _handle_param_spark_confs(self) -> None:
        """Constructor arguments the user did NOT pass may be given session-wide through Spark confs — the only way to set
        them under Spark Connect (reference core.py:1124-1170): spark.rapids.ml.verbose (bool or 0..6),
        spark.rapids.ml.float32_inputs (bool), spark.rapids.ml.num_workers (int > 0).  Values land in _input_kwargs
        before _set_params reads them; an explicit argument always wins."""
        conf = _active_session_conf()
        if conf is None:
            return
        kw = self._input_kwargs
        for name, key, parse, expects in _CONF_PARAMS:
            raw = conf.get(key, None)
            if kw.get(name) is not None or raw is None:   # an explicit argument always wins
                continue
            try:
                kw[name] = parse(str(raw).strip().lower())
            except Exception:
                raise ValueError(f"Invalid value for {key} which should be {expects}: {raw}") from None

    def _fit_internal(self, dataset: LocalDataFrame, paramMaps: Optional[Sequence[Dict[Any, Any]]]) -> List["_CumlModel"]:
        self.logger.info(f"Training spark-rapids-ml (b200) with {self.num_workers} worker(s) ...")
        try:
            res = self._call_cuml_fit_func(dataset=dataset, partially_collect=True, paramMaps=paramMaps)
            rows = res if isinstance(res, list) else res.collect()   # the pyspark branch returns the collected rows
        except Exception as e:
            # Spark refuses a barrier stage on some RDD chains (e.g. after coalesce): retry once on a repartitioned
            # dataset, as the reference does (core.py:1245-1257)
            if "BarrierJobUnsupportedRDDChainException" not in str(e):
                raise
            self.logger.warning("Barrier rdd error encountered with input dataset. Retrying with repartitioning.")
            res = self._call_cuml_fit_func(dataset=dataset.repartition(self.num_workers), partially_collect=True,
                                           paramMaps=paramMaps)
            rows = res if isinstance(res, list) else res.collect()
        self.logger.info("Finished training")
        rows = self._merge_model_chunks(rows, paramMaps)
        models: List["_CumlModel"] = []
        for index in range(1 if paramMaps is None else len(paramMaps)):
            model = self._create_pyspark_model(rows[index])
            model._num_workers = self._num_workers
            model._float32_inputs = self._float32_inputs
            self._copyValues(model, paramMaps[index] if paramMaps is not None else None)
            self._copy_cuml_params(model)
            models.append(model)
        return models

    if not HAVE_PYSPARK:   # pyspark.ml.Estimator.fit(dataset, params) -> self._fit(dataset) provides this otherwise
        def fit(self, dataset: LocalDataFrame, params: Optional[Dict[Any, Any]] = None) -> "_CumlModel":
            est = self.copy(params) if params else self
            return est._fit(dataset)

        def fitMultiple(self, dataset: LocalDataFrame, paramMaps: Sequence[Dict[Any, Any]]) -> Iterator[Tuple[int, "_CumlModel"]]:
            """pyspark.ml.Estimator.fitMultiple: (index, model) per param map, one fit each (reference
            core.py:1172-1228); _TunedEstimator replaces it for the estimators CrossValidator tunes."""
            for index, pm in enumerate(paramMaps):
                yield index, self.copy(pm)._fit(dataset)

    def _fit(self, dataset: LocalDataFrame) -> "_CumlModel":
        if self._use_cpu_fallback():
            # reference: core.py:1283-1295 falls back to pyspark.ml on CPU; this build has NO CPU path.
            raise ValueError("a Spark Param without GPU support is set and spark_rapids_ml_b200 has no CPU fallback")
        return self._fit_internal(dataset, None)[0]

    # -- persistence (core.py:268-307): Spark's DefaultParamsWriter layout (path/metadata/part-00000 JSON) --
    def save(self, path: str, overwrite: bool = False) -> None:
        """pyspark.ml.util.MLWritable.save: a shortcut of write().save(path) — an existing path is an error unless
        write().overwrite() (or overwrite=True here) is used."""
        w = self.write()
        (w.overwrite() if overwrite else w).save(path)

    def write(self) -> Any:
        if _spark_context_active():   # real pyspark with a live SparkContext: MLWriter + DefaultParamsWriter
            from . import spark_binding

            return spark_binding.make_writer(self, None)
        return _Writer(self, None)

    @classmethod
    def read(cls) -> Any:
        if _spark_context_active():
            from . import spark_binding

            return spark_binding.make_reader(cls, False)
        return _Reader(cls, False)

    @classmethod
    def load(cls, path: str) -> "_CumlEstimator":
        return cls.read().load(path)


class _ModelIterator:
    """(index, model) pairs in map order; safe to share between the threads of pyspark's tuning loops."""

    def __init__(self, models: List[Any]) -> None:
        self._it = iter(enumerate(models))
        self._lock = threading.Lock()

    def __iter__(self) -> "_ModelIterator":
        return self

    def __next__(self) -> Tuple[int, Any]:
        with self._lock:
            return next(self._it)


class _TunedEstimator(_CumlEstimator):
    """An estimator whose fitMultiple fits a grid of param maps from one ingest when every map changes only
    `_single_pass_params`.  The fit function then runs once per task over `_fit_grid`, one `_settings()` per map,
    and returns one model row per map in map order."""

    _single_pass_params: frozenset = frozenset()
    _fit_grid: Optional[List[Dict[str, Any]]] = None

    @abstractmethod
    def _settings(self) -> Dict[str, Any]:
        """What the fit function needs of one map, read from a copy of the estimator that carries the map."""
        raise NotImplementedError

    @classmethod
    def _shares_ingest(cls, paramMaps: Sequence[Dict[Any, Any]]) -> bool:
        """Whether fitMultiple fits these maps from one ingest: there are maps and each changes only
        `_single_pass_params`."""
        return bool(paramMaps) and all(p.name in cls._single_pass_params for pm in paramMaps for p in pm)

    def fitMultiple(self, dataset: Any, paramMaps: Sequence[Dict[Any, Any]]) -> Iterator[Tuple[int, Any]]:
        """(index, model) per param map, in map order; each model equals self.copy(map).fit(dataset), its cuml params
        included.  When the maps share one ingest (_shares_ingest) a single fit serves them all; otherwise each map is
        one fit."""
        maps = list(paramMaps)
        if not self._shares_ingest(maps):
            return _ModelIterator([self.copy(pm)._fit(dataset) for pm in maps])
        copies = [self.copy(pm) for pm in maps]
        for c in copies:
            c._validate_parameters()
        est = self.copy()
        est._fit_grid = [c._settings() for c in copies]
        if est._use_cpu_fallback():
            raise ValueError("a Spark Param without GPU support is set and spark_rapids_ml_b200 has no CPU fallback")
        models = est._fit_internal(dataset, maps)
        for m, c in zip(models, copies):
            c._copy_cuml_params(m)
        return _ModelIterator(models)


TRANSFORM_GROUP_ROWS = 1 << 20    # rows per device pass of transform and evaluation ...
TRANSFORM_GROUP_BYTES = 2 << 30   # ... and the cap on the device bytes they take (`row_bytes` per row)


def _row_groups(items: Iterable[Any], row_bytes: int,
                extra_bytes: Optional[Callable[[Any], int]] = None) -> Iterator[List[Any]]:
    """Consecutive frames or batches, in order, in groups that end once they reach TRANSFORM_GROUP_ROWS rows or
    TRANSFORM_GROUP_BYTES at `row_bytes` per row (plus `extra_bytes(item)` per item when given); the last group may be
    smaller."""
    limit = max(1, min(TRANSFORM_GROUP_ROWS, TRANSFORM_GROUP_BYTES // max(1, row_bytes)))
    group: List[Any] = []
    rows = nbytes = 0
    for it in items:
        group.append(it)
        rows += len(it)
        if extra_bytes is not None:
            nbytes += len(it) * row_bytes + extra_bytes(it)
        if rows >= limit or nbytes >= TRANSFORM_GROUP_BYTES:
            yield group
            group, rows, nbytes = [], 0, 0
    if group:
        yield group


def _iter_transform(transform: Callable, model: Any, frames: Iterable[Any]) -> Iterator[Any]:
    """One result per input frame, in order: `transform` (a model's grouped transform function) takes each group of
    consecutive frames in one device pass."""
    extra = _vector_bytes if getattr(transform, "sparse", False) else None
    for group in _row_groups(frames, transform.row_bytes, extra):
        yield from transform(model, group)


def _supports_transform_evaluate(classification: bool, evaluator: Any) -> bool:
    """Whether the single-pass evaluation serves (estimator kind, evaluator): a classifier with a
    MulticlassClassificationEvaluator and a metric of metrics.MULTICLASS_METRICS or a BinaryClassificationEvaluator
    and a metric of metrics.BINARY_METRICS, or a regressor with a RegressionEvaluator."""
    from . import metrics

    name = type(evaluator).__name__
    try:
        metric = evaluator.getMetricName()
    except Exception:
        return False
    if classification:
        return ((name == "MulticlassClassificationEvaluator" and metric in metrics.MULTICLASS_METRICS) or
                (name == "BinaryClassificationEvaluator" and metric in metrics.BINARY_METRICS))
    return name == "RegressionEvaluator" and metric in metrics.REGRESSION_METRICS


def _eval_metric_info(evaluator: Any) -> Dict[str, Any]:
    """What the device pass and the metric need from an evaluator (pyspark's or the local one)."""
    if evaluator.isSet("weightCol") and evaluator.getOrDefault("weightCol"):
        raise NotImplementedError("weightCol is not supported by the single-pass evaluation")
    info = {"metric": evaluator.getMetricName(), "labelCol": evaluator.getLabelCol(), "binary": False}
    if type(evaluator).__name__ == "MulticlassClassificationEvaluator":
        info.update(classification=True, eps=float(evaluator.getEps()), metricLabel=float(evaluator.getMetricLabel()),
                    beta=float(evaluator.getBeta()))
    elif type(evaluator).__name__ == "BinaryClassificationEvaluator":
        num_bins = int(evaluator.getNumBins())
        if num_bins < 0:
            raise ValueError(f"numBins must be >= 0, got {num_bins}")
        info.update(classification=True, binary=True, eps=0.0, numBins=num_bins,
                    rawPredictionCol=evaluator.getRawPredictionCol())
    else:
        info.update(classification=False, eps=0.0, throughOrigin=bool(evaluator.getThroughOrigin()))
    return info


def _transform_evaluate_internal(model: Any, dataset: Any, evaluator: Any) -> List[float]:
    """One metric per model of a (combined) model on a local frame (reference core.py:1572-1693).  Each partition's
    features and label are ingested as transform() ingests them, in groups of up to TRANSFORM_GROUP_ROWS rows; each
    group is one device evaluation pass (the model's third transform function) that returns every model's
    accumulators; the accumulators merge on the host in partition and group order.  The label goes to the device as
    float32, as the fits read it: a float64 label that float32 cannot hold is scored at its float32 rounding.
    A BinaryClassificationEvaluator needs every row's score at once: each group's pass appends every model's scores
    and the label bits to device buffers sized for the whole frame (checked against the free device memory before the
    first group), and one curve pass over them gives every model's area at the end."""
    from . import metrics
    from .sparkshim.sql import _batches_to_pdf_iter

    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError(f"{type(model).__name__}._transformEvaluate() of a pyspark DataFrame is not "
                                      "supported in this build; evaluate a local frame")
    info = _eval_metric_info(evaluator)
    construct, _, evaluate = model._get_cuml_transform_func(dataset, info)
    if evaluate is None:
        raise NotImplementedError(f"{type(model).__name__} has no single-pass evaluation")
    input_col, input_cols = model._get_input_columns()
    label_col = info["labelCol"]
    n_cols = int(model.n_cols)
    state: Dict[str, Any] = {}
    accs: Optional[List[Dict[str, Any]]] = None

    def run(group: List[pa.RecordBatch]) -> None:
        nonlocal accs
        import torch

        y = np.concatenate([np.asarray(b.column(label_col).to_numpy(zero_copy_only=False), dtype=np.float32)
                            for b in group]) if group else np.zeros(0, np.float32)
        m = state["model"]
        X = _ingest(m.ctx, _batches_to_pdf_iter(_select_features(group, input_col, input_cols),
                                                dataset.arrow_backed_pandas), n_cols, int(y.size))
        yd = torch.as_tensor(y).to(m.ctx.device)
        if binary:
            evaluate(m, X, yd, state["scores"], state["pos"], state["row0"])
            state["row0"] += int(y.size)
            accs = []   # a group ran; the metrics come from the curve pass at the end
            return
        got = evaluate(m, X, yd)
        accs = got if accs is None else [metrics.merge_all([a, b], info["classification"]) for a, b in zip(accs, got)]

    binary = info["binary"]
    for pid, part in enumerate(dataset._parts):
        if "model" not in state:
            gpu = _CumlCommon._set_gpu_device(BarrierTaskContext(pid, len(dataset._parts)), True, True)
            state["model"] = construct(gpu)
            if binary:
                state["scores"], state["pos"] = state["model"].ctx.binary_buffers(evaluate.n_models, dataset.count())
                state["row0"] = 0
        for group in _row_groups(part, 4 * n_cols + 4):   # X and the float32 label
            run(group)
        if accs is None:   # the first partition is empty: one pass over no rows still gives every model's accumulators
            run([])
    assert accs is not None
    if binary:
        return [float(v) for v in state["model"].ctx.eval_binary(state["scores"], state["pos"], info["numBins"],
                                                                  info["metric"])]
    if info["classification"]:
        return [metrics.multiclass_metric(a, info["metric"], info["metricLabel"], info["beta"]) for a in accs]
    return [metrics.regression_metric(a, info["metric"], info["throughOrigin"]) for a in accs]


def _class_accs(res: Dict[str, Any]) -> List[Dict[str, Any]]:
    """Per-model accumulators of one Context.eval_* result."""
    if "reg" in res:
        return [{"n": res["n"], "reg": r} for r in res["reg"]]
    return [{"n": res["n"], "label_count": res["label_count"], "tp": t, "fp": f, "loss": float(l)}
            for t, f, l in zip(res["tp"], res["fp"], res["loss"])]


def _parse_conf_bool(v: str) -> bool:
    if v not in ("true", "false"):
        raise ValueError(v)
    return v == "true"


def _parse_conf_verbose(v: str) -> Union[int, bool]:
    try:
        i = int(v)
    except ValueError:
        return _parse_conf_bool(v)
    if not 0 <= i <= 6:
        raise ValueError(v)
    return i


def _parse_conf_pos_int(v: str) -> int:
    i = int(v)
    if i <= 0:
        raise ValueError(v)
    return i


_CONF_PARAMS = (
    ("verbose", "spark.rapids.ml.verbose", _parse_conf_verbose, "a boolean or an integer between 0 and 6"),
    ("float32_inputs", "spark.rapids.ml.float32_inputs", _parse_conf_bool, "a boolean"),
    ("num_workers", "spark.rapids.ml.num_workers", _parse_conf_pos_int, "an integer greater than 0"),
)


def _active_session_conf() -> Any:
    """The conf of the active session, without creating one: the live SparkSession under pyspark, else the LocalSession."""
    if HAVE_PYSPARK:
        try:
            from pyspark.sql import SparkSession

            active = SparkSession.getActiveSession()
            if active is not None:
                return active.conf
        except Exception:
            pass
    from .sparkshim.sql import LocalSession

    return LocalSession._active.conf if LocalSession._active is not None else None


def _spark_context_active() -> bool:
    if not HAVE_PYSPARK:
        return False
    try:
        from pyspark import SparkContext

        return SparkContext._active_spark_context is not None
    except Exception:
        return False


# Local-filesystem writer / reader producing and accepting the SAME directory layout as pyspark's DefaultParamsWriter and
# the reference's _CumlEstimatorWriter / _CumlModelWriter (core.py:268-355): path/metadata/part-00000 holds one JSON
# object {class, timestamp, sparkVersion, uid, paramMap, defaultParamMap, _cuml_params, _num_workers, _float32_inputs};
# a model adds path/data/part-00000 = json.dumps(model attributes); Hadoop-style _SUCCESS markers beside both.  A
# directory written by the reference therefore loads here and vice versa (class names are not compared, as in the
# reference's readers, which call DefaultParamsReader.loadMetadata without an expected class).
class _Writer:
    def __init__(self, inst: Any, model_attributes: Optional[Dict[str, Any]]):
        self.inst = inst
        self.model_attributes = model_attributes
        self._overwrite = False

    def overwrite(self) -> "_Writer":
        self._overwrite = True
        return self

    def save(self, path: str) -> None:
        _save_metadata(self.inst, path, self._overwrite)
        if self.model_attributes is not None:
            _write_part(os.path.join(path, "data"), json.dumps(self.model_attributes))


class _Reader:
    def __init__(self, cls: Any, is_model: bool):
        self.cls = cls
        self.is_model = is_model

    def load(self, path: str) -> Any:
        meta = _load_metadata(path)
        if self.is_model:
            inst = self.cls(**json.loads(_read_part(os.path.join(path, "data"))))
        else:
            inst = self.cls()
        _reset_uid(inst, meta["uid"])
        _set_params_from_metadata(inst, meta)
        return inst


def _reset_uid(inst: Any, uid: str) -> None:
    if hasattr(inst, "_resetUid"):   # pyspark Params: re-parents the Param objects as well
        inst._resetUid(uid)
    else:
        inst.uid = uid


def _write_part(dirname: str, text: str) -> None:
    os.makedirs(dirname, exist_ok=True)
    with open(os.path.join(dirname, "part-00000"), "w") as f:
        f.write(text + "\n")
    open(os.path.join(dirname, "_SUCCESS"), "w").close()


def _read_part(dirname: str) -> str:
    parts = sorted(f for f in os.listdir(dirname) if f.startswith("part-"))
    if not parts:
        raise IOError(f"no part file under {dirname}")
    for name in parts:   # saveAsTextFile of a one-element RDD may leave empty parts beside the one that has the line
        with open(os.path.join(dirname, name)) as f:
            text = f.read().strip()
        if text:
            return text.splitlines()[0]
    raise IOError(f"empty part files under {dirname}")


def _spark_version() -> str:
    if HAVE_PYSPARK:
        try:
            import pyspark

            return str(pyspark.__version__)
        except Exception:
            pass
    return "3.5.0"   # what DefaultParamsReader parses with majorMinorVersion(); no Spark is involved in a local save


def _save_metadata(inst: Any, path: str, overwrite: bool, extra: Optional[Dict[str, Any]] = None) -> None:
    import time

    if os.path.exists(path) and not overwrite:
        raise IOError(f"Path {path} already exists. To overwrite it, use write().overwrite().save(path).")
    meta = {
        "class": inst.__module__ + "." + inst.__class__.__name__,
        "timestamp": int(time.time() * 1000),
        "sparkVersion": _spark_version(),
        "uid": inst.uid,
        "paramMap": {p.name: v for p, v in inst._paramMap.items()},
        "defaultParamMap": {p.name: v for p, v in inst._defaultParamMap.items()},
        "_cuml_params": inst._cuml_params,
        "_num_workers": inst._num_workers,
        "_float32_inputs": inst._float32_inputs,
    }
    if extra:
        meta.update(extra)
    _write_part(os.path.join(path, "metadata"), json.dumps(meta, separators=(",", ":")))


def _load_metadata(path: str) -> Dict[str, Any]:
    return json.loads(_read_part(os.path.join(path, "metadata")))


def _set_params_from_metadata(inst: Any, meta: Dict[str, Any]) -> None:
    for name, v in meta.get("defaultParamMap", {}).items():
        if inst.hasParam(name):
            inst._setDefault(**{name: v})
    for name, v in meta.get("paramMap", {}).items():
        if inst.hasParam(name):
            inst._set(**{name: v})
    inst._cuml_params = meta["_cuml_params"]
    inst._num_workers = meta["_num_workers"]
    inst._float32_inputs = meta["_float32_inputs"]


class _CumlModel(ModelBase, _CumlParams, _CumlCommon):
    """reference: core.py:1356-1753 (KMeans-relevant subset)."""

    def __init__(self, *, dtype: Optional[str] = None, n_cols: Optional[int] = None, **model_attributes: Any) -> None:
        super().__init__()
        self._initialize_cuml_params()
        self.dtype = dtype
        self.n_cols = n_cols
        self._model_attributes = model_attributes
        self._model_attributes["dtype"] = dtype
        self._model_attributes["n_cols"] = n_cols

    def _get_model_attributes(self) -> Optional[Dict[str, Any]]:
        return self._model_attributes

    @abstractmethod
    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None) -> Tuple[Callable, Callable, Optional[Callable]]:
        raise NotImplementedError

    @abstractmethod
    def _out_schema(self, input_schema: Any) -> Any:
        raise NotImplementedError

    # -- persistence (core.py:310-355): metadata as the estimator + path/data = json.dumps(model attributes) --
    def save(self, path: str, overwrite: bool = False) -> None:
        """pyspark.ml.util.MLWritable.save: a shortcut of write().save(path) — an existing path is an error unless
        write().overwrite() (or overwrite=True here) is used."""
        w = self.write()
        (w.overwrite() if overwrite else w).save(path)

    def write(self) -> Any:
        if _spark_context_active():
            from . import spark_binding

            return spark_binding.make_writer(self, self._get_model_attributes())
        return _Writer(self, self._get_model_attributes())

    @classmethod
    def read(cls) -> Any:
        if _spark_context_active():
            from . import spark_binding

            return spark_binding.make_reader(cls, True)
        return _Reader(cls, True)

    @classmethod
    def load(cls, path: str) -> "_CumlModel":
        return cls.read().load(path)

    if not HAVE_PYSPARK:   # pyspark.ml.Transformer.transform(dataset, params) -> self._transform(dataset) otherwise
        def transform(self, dataset: LocalDataFrame) -> LocalDataFrame:
            return self._transform(dataset)

    # the model attributes that _combine turns into one list entry per model
    _combined_attrs: Tuple[str, ...] = ()

    @classmethod
    def _combine(cls, models: List["_CumlModel"]) -> "_CumlModel":
        """One model holding every model's `_combined_attrs`, for the single-pass evaluation (reference
        classification.py:1557-1572); its other attributes and its params are the first model's."""
        assert len(models) > 0 and all(isinstance(m, cls) for m in models)
        first = models[0]
        attrs = dict(first._get_model_attributes() or {})
        for name in cls._combined_attrs:
            attrs[name] = [m._get_model_attributes()[name] for m in models]
        out = cls(**attrs)
        first._copyValues(out)
        first._copy_cuml_params(out)
        return out

    def _transformEvaluate(self, dataset: Any, evaluator: Any, params: Optional[Dict[Any, Any]] = None) -> List[float]:
        """The evaluator's metric for every model of this (combined) model on a local frame, one device pass per
        ingest group (reference core.py:1572-1693)."""
        return _transform_evaluate_internal(self.copy(params) if params else self, dataset, evaluator)


def _no_spark_transform(model: Any, dataset: Any) -> None:
    """transform() of a pyspark DataFrame is a pandas_udf of one output column: other models refuse it."""
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError(f"{type(model).__name__}.transform() of a pyspark DataFrame is not supported in "
                                      "this build; transform a local frame")


class _CumlModelWithColumns(_CumlModel):
    """reference: core.py:1797-1941 — keeps the input columns and appends the output column."""

    def _output_col_name(self) -> str:
        """The column transform() appends: predictionCol here, outputCol for a feature transformer."""
        return self.getOrDefault("predictionCol")

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        """The (column name, Arrow type) of each column transform() appends, in order: one per output of the grouped
        transform function."""
        return [(self._output_col_name(), self._out_schema(None))]

    def _grouped_transform(self, predict: Callable[[Any, Any], Sequence[Any]], row_bytes: int,
                           sparse: bool = False) -> _GroupedTransform:
        """This model's grouped transform function: `predict(device_model, X)` returns one CUDA tensor per column of
        _transform_outputs(); `row_bytes` is the device bytes a row takes (sparse: X is a device CSR, see
        _GroupedTransform)."""
        return _GroupedTransform(predict, int(self.n_cols), row_bytes, [t for _, t in self._transform_outputs()],
                                 sparse)

    def _transform(self, dataset: Any) -> Any:
        from .sparkshim.sql import _batches_to_pdf_iter

        outputs = self._transform_outputs()
        if len(outputs) > 1:
            _no_spark_transform(self, dataset)
        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):   # pandas_udf + withColumn (core.py:1846-1878)
                return spark_binding.transform_with_pandas_udf(
                    self, dataset, alias.data, lambda ctx, local: _CumlCommon._set_gpu_device(ctx, local, True))
        input_col, input_cols = self._get_input_columns()
        construct, transform, _ = self._get_cuml_transform_func(dataset)
        cols: List[List[List[pa.Array]]] = [[] for _ in outputs]   # output -> partition -> one array per batch
        model = None
        for pid, part in enumerate(dataset._parts):
            if part and model is None:   # on the GPU of the first partition with a batch
                model = construct(_CumlCommon._set_gpu_device(BarrierTaskContext(pid, len(dataset._parts)), True, True))
            frames = _batches_to_pdf_iter(_select_features(part, input_col, input_cols), dataset.arrow_backed_pandas)
            per: List[List[pa.Array]] = [[] for _ in outputs]
            for res in _iter_transform(transform, model, frames):
                for arrs, r, (_, out_type) in zip(per, res, outputs):
                    arrs.append(_transform_result_array(r, out_type))
            for c, arrs in zip(cols, per):
                c.append(arrs)
        if model is not None:
            model.close()
        out = dataset
        for (name, _), parts in zip(outputs, cols):
            out = out.with_appended_column(name, parts)
        return out


class _CumlModelWithPredictionCol(_CumlModelWithColumns):
    """reference: core.py:1944-1967."""

    def setPredictionCol(self, value: str) -> "_CumlModelWithPredictionCol":
        self._set_params(predictionCol=value)
        return self

    @property
    def numFeatures(self) -> int:
        """Number of features the model was trained on (reference core.py:1961-1967)."""
        return int(self.n_cols) if self.n_cols is not None else -1
