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
import uuid
from abc import abstractmethod
from collections import namedtuple
from typing import Any, Callable, Dict, Iterator, List, Optional, Sequence, Tuple, Union

import numpy as np
import pandas as pd
import pyarrow as pa

from .params import _CumlParams
from .sparkshim import (HAVE_PYSPARK, BarrierTaskContext, EstimatorBase, LocalDataFrame, ModelBase, Params, Row,
                        get_session)
from .utils import DeviceRowAppender, arrow_list_column_buffers, get_logger

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


def _features_from_pdf(pdf: pd.DataFrame, multi_col_names: Optional[List[str]], appender: DeviceRowAppender,
                       logger: Any) -> int:
    """One Arrow batch -> rows of the device matrix.  Fast path: the Arrow child buffer, zero-copy.
    Compat path (classic Spark conversion: object column of ndarrays): host stacking, as core.py:916 does."""
    n_b = int(pdf.shape[0])
    if n_b == 0:
        return 0
    if multi_col_names:
        cols = []
        for c in multi_col_names:
            a = pdf[c].to_numpy()
            if a.dtype == np.float64 or a.dtype == np.float32 or a.dtype.kind == "i":
                cols.append(np.ascontiguousarray(a))
            else:
                cols.append(np.ascontiguousarray(a, dtype=np.float32))
        dt = cols[0].dtype
        cols = [c if c.dtype == dt else c.astype(dt) for c in cols]
        appender.append_columns(cols)
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
        cols = [np.ascontiguousarray(df[c].to_numpy()) for c in df.columns]
        dt = cols[0].dtype
        app.append_columns([c if c.dtype == dt else c.astype(dt) for c in cols])
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


_ARROW_SCALARS = {"int": pa.int32(), "float": pa.float32(), "double": pa.float64()}


def _transform_result_array(res: Any, out_type: str) -> pa.Array:
    """One transform result (a pandas Series) as the Arrow array of the model's output type: "int" or "array<float>" /
    "array<double>" (one fixed-width vector per row)."""
    if out_type.startswith("array<"):
        elem = _ARROW_SCALARS[out_type[len("array<"):-1]]
        rows = list(res)
        width = len(rows[0]) if rows else 0
        vals = np.asarray(rows, dtype=elem.to_pandas_dtype()).reshape(-1) if rows else np.zeros(0, elem.to_pandas_dtype())
        offsets = np.arange(0, len(rows) * width + 1, max(width, 1), dtype=np.int32)[: len(rows) + 1]
        return pa.ListArray.from_arrays(pa.array(offsets), pa.array(vals, type=elem))
    return pa.array(np.asarray(res), type=_ARROW_SCALARS[out_type])



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
        """-> (selected/cast dataframe, multi_col_names, dimension, feature dtype)."""
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
            df, multi_col_names, dimension, _ = spark_binding.pre_process_data(self, dataset, alias.data)
            is_local = spark_binding.is_local(dataset)
        else:
            df, multi_col_names, dimension, _ = self._pre_process_data(dataset)
            if df.getNumPartitions() != num_workers:
                df = df.repartition(num_workers)   # core.py:771-772
            is_local = True   # the local frame runs on this host: partition id doubles as the GPU id (core.py:377-384)
        params: Dict[str, Any] = {param_alias.cuml_init: dict(self.cuml_params), param_alias.fit_multiple_params: None}
        extra_cols = [c for c in (alias.label, alias.row_number) if c in df.columns]
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
                appender = DeviceRowAppender(cc.handle, dimension)
                sizes: List[int] = []
                # label / row-number columns the pre-processed frame carries (kneighbors): host arrays, per batch
                extra: Dict[str, List[np.ndarray]] = {c: [] for c in extra_cols}
                for pdf in pdf_iter:
                    sizes.append(_features_from_pdf(pdf, multi_col_names, appender, logger))
                    for c in extra_cols:
                        extra[c].append(np.asarray(pdf[c].to_numpy(), dtype=np.int64))
                if len(sizes) == 0 or all(sz == 0 for sz in sizes):
                    raise RuntimeError(
                        "A python worker received no data.  Please increase amount of data or use fewer workers.")
                X = appender.finish()
                slots = [np.concatenate(extra[c]) if c in extra else None for c in (alias.label, alias.row_number)]
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
            """pyspark.ml.Estimator.fitMultiple: (index, model) per param map, one fit each — what the reference falls back
            to for KMeans (`_enable_fit_multiple_in_single_pass` is False there, core.py:1172-1228)."""
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


TRANSFORM_GROUP_ROWS = 1 << 20    # rows labelled per device pass when the transform function can take several batches ...
TRANSFORM_GROUP_BYTES = 2 << 30   # ... and the cap on the device matrix they form (transform function's `row_bytes`)


def _iter_transform(transform_internal: Callable, get_model: Callable[[], Any], frames: Iterator[Any]) -> Iterator[Any]:
    """One result per input frame, in order.  When the model's transform function offers `.many` (KMeans), consecutive
    frames are grouped up to TRANSFORM_GROUP_ROWS rows and labelled in one device pass; otherwise frame by frame, as the
    reference does (core.py:1900-1915)."""
    many = getattr(transform_internal, "many", None)
    if many is None:
        for f in frames:
            yield transform_internal(get_model(), f)
        return
    row_bytes = max(1, int(getattr(transform_internal, "row_bytes", 1)))
    limit = max(1, min(TRANSFORM_GROUP_ROWS, TRANSFORM_GROUP_BYTES // row_bytes))
    group: List[Any] = []
    rows = 0
    for f in frames:
        group.append(f)
        rows += len(f)
        if rows >= limit:
            yield from many(get_model(), group)
            group, rows = [], 0
    if group:
        yield from many(get_model(), group)


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


class _CumlModelWithColumns(_CumlModel):
    """reference: core.py:1797-1941 — keeps the input columns and appends the output column."""

    def _output_col_name(self) -> str:
        """The column transform() appends: predictionCol here, outputCol for a feature transformer."""
        return self.getOrDefault("predictionCol")

    def _transform(self, dataset: Any) -> Any:
        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):   # pandas_udf + withColumn (core.py:1846-1878)
                return spark_binding.transform_with_pandas_udf(
                    self, dataset, alias.data, lambda ctx, local: _CumlCommon._set_gpu_device(ctx, local, True))
        input_col, input_cols = self._get_input_columns()
        construct, transform_internal, _ = self._get_cuml_transform_func(dataset)
        pred_name = self._output_col_name()
        out_type = self._out_schema(dataset.schema)
        n_cols = self.n_cols
        out_parts: List[List[pa.Array]] = []
        state: Dict[str, Any] = {}
        for pid, part in enumerate(dataset._parts):
            def frames(part: Any = part, pid: int = pid) -> Iterator[Any]:
                from .sparkshim.sql import _batches_to_pdf_iter

                def selected() -> Iterator[pa.RecordBatch]:   # feature columns only, renamed at the Arrow level (zero-copy)
                    for batch in part:
                        if "model" not in state:
                            gpu = _CumlCommon._set_gpu_device(BarrierTaskContext(pid, len(dataset._parts)), True, True)
                            state["model"] = construct(gpu)
                        if input_cols:
                            yield batch.select(list(input_cols))
                        else:
                            yield batch.select([input_col]).rename_columns([alias.data])

                return _batches_to_pdf_iter(selected(), dataset.arrow_backed_pandas)

            out_parts.append([_transform_result_array(res, out_type)
                              for res in _iter_transform(transform_internal, lambda: state["model"], frames())])
        if "model" in state and hasattr(state["model"], "close"):
            state["model"].close()
        assert n_cols is None or n_cols > 0
        return dataset.with_appended_column(pred_name, out_parts)


class _CumlModelWithPredictionCol(_CumlModelWithColumns):
    """reference: core.py:1944-1967."""

    def setPredictionCol(self, value: str) -> "_CumlModelWithPredictionCol":
        self._set_params(predictionCol=value)
        return self

    @property
    def numFeatures(self) -> int:
        """Number of features the model was trained on (reference core.py:1961-1967)."""
        return int(self.n_cols) if self.n_cols is not None else -1
