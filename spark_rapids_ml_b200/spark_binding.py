"""The real-pyspark side of the Spark<->worker boundary (SURVEY.md 8b "B1").  Imported only when `import pyspark`
succeeds; with a LocalDataFrame (this image: no pyspark / JVM) core.py drives the same worker function through the
shim instead.

What the reference does at these call sites, reproduced here against the public pyspark API:
  * pre-processing      core.py:463-562   select / cast the feature column(s); VectorUDT -> array via
                                          pyspark.ml.functions.vector_to_array (:523-525); dimension from first()
  * barrier fit stage   core.py:1005-1013 dataset.mapInPandas(_train_udf, schema).rdd.barrier().mapPartitions(identity)
  * local-mode probe    core.py:377-384 / utils._is_local: master URL "local..." -> partition id doubles as the GPU id
  * transform           core.py:1846-1878 a pandas_udf over struct(*feature columns), appended with withColumn
  * persistence         core.py:268-355   MLWriter / MLReader over DefaultParamsWriter.saveMetadata / DefaultParamsReader
                                          (+ sc.parallelize([json]).saveAsTextFile(path/data) for a model)
"""
from __future__ import annotations

from typing import Any, Callable, Iterator, List, Optional, Tuple

import pandas as pd


def is_spark_dataframe(obj: Any) -> bool:
    try:
        from pyspark.sql import DataFrame
    except Exception:
        return False
    return isinstance(obj, DataFrame)


def is_local(dataset: Any) -> bool:
    """reference utils._is_local: Spark local mode (one host, partition id == GPU id)."""
    try:
        master = dataset.sparkSession.sparkContext.master
    except Exception:
        return True
    return str(master).startswith("local")


def pre_process_data(est: Any, dataset: Any, data_alias: str) -> Tuple[Any, Optional[List[str]], int, str]:
    """-> (selected/cast DataFrame, multi_col_names, dimension, element type) — reference core.py:463-562."""
    from pyspark.ml.functions import vector_to_array
    from pyspark.ml.linalg import VectorUDT
    from pyspark.sql.functions import col
    from pyspark.sql.types import ArrayType, DoubleType, FloatType

    input_col, input_cols = est._get_input_columns()
    f32 = bool(est._float32_inputs)
    if input_col is not None:
        dtype = dataset.schema[input_col].dataType
        if isinstance(dtype, VectorUDT):
            feat = vector_to_array(col(input_col), "float32" if f32 else "float64").alias(data_alias)   # :523-525
            inner = "float" if f32 else "double"
        elif isinstance(dtype, ArrayType):
            elem = dtype.elementType
            if isinstance(elem, DoubleType) and f32:
                feat = col(input_col).cast(ArrayType(FloatType())).alias(data_alias)                    # :489-495
                inner = "float"
            elif isinstance(elem, (FloatType, DoubleType)):
                feat = col(input_col).alias(data_alias)
                inner = "float" if isinstance(elem, FloatType) else "double"
            else:
                feat = col(input_col).cast(ArrayType(FloatType() if f32 else DoubleType())).alias(data_alias)
                inner = "float" if f32 else "double"
        else:
            raise ValueError("Unsupported input type.")
        df = dataset.select(feat)
        first = df.first()
        if first is None:
            raise RuntimeError("A python worker received no data.  Please increase amount of data or use fewer workers.")
        return df, None, len(first[data_alias]), inner
    assert input_cols is not None
    want = FloatType() if f32 else DoubleType()
    df = dataset.select(*[col(c).cast(want).alias(c) for c in input_cols])                              # :543-557
    return df, list(input_cols), len(input_cols), "float" if f32 else "double"


def run_barrier_fit(df: Any, train_udf: Callable[[Iterator[pd.DataFrame]], Iterator[pd.DataFrame]], out_schema: Any,
                    num_workers: int) -> List[Any]:
    """One barrier task per GPU (reference core.py:771-772, 1005-1013); returns the collected model rows."""
    if df.rdd.getNumPartitions() != num_workers:
        df = df.repartition(num_workers)
    pipelined_rdd = df.mapInPandas(train_udf, schema=out_schema).rdd.barrier().mapPartitions(lambda x: x)
    pipelined_rdd = try_stage_level_scheduling(pipelined_rdd, df)
    return pipelined_rdd.collect()


def _version_tuple(v: str) -> Tuple[int, ...]:
    out = []
    for part in str(v).split(".")[:3]:
        digits = "".join(ch for ch in part if ch.isdigit())
        out.append(int(digits) if digits else 0)
    return tuple(out + [0] * (3 - len(out)))


def stage_level_scheduling_plan(spark_version: str, conf_get: Callable[[str], Optional[str]], is_local_mode: bool,
                                plugins: str = "", rapids_sql_enabled: str = "true") -> Tuple[Optional[Tuple[int, float]], str]:
    """Decide whether the training stage gets its own task resource profile (reference core.py:637-740): so that each
    barrier task lands on a different executor and owns its GPU while ETL stages keep their fractional GPU amounts.
    -> ((task_cpus, task_gpus) or None, reason).  Pure function of the Spark version and confs: unit-tested without Spark."""
    if is_local_mode:
        return None, "local mode: the partition id selects the GPU"
    ver = _version_tuple(spark_version)
    if ver < (3, 4, 0):
        return None, "stage-level scheduling requires Spark 3.4.0+"
    master = conf_get("spark.master") or ""
    if ver < (3, 5, 1) and not (master.startswith("spark://") or master.startswith("local-cluster")):
        return None, "Spark %s: stage-level scheduling requires standalone or local-cluster mode" % spark_version
    cores, gpus = conf_get("spark.executor.cores"), conf_get("spark.executor.resource.gpu.amount")
    if cores is None or gpus is None:
        return None, "spark.executor.cores and spark.executor.resource.gpu.amount must be set"
    if int(cores) == 1:
        return None, "spark.executor.cores = 1: one task at a time anyway"
    if int(float(gpus)) > 1:
        return None, "spark.executor.resource.gpu.amount > 1: left to the user's configuration"
    task_gpu = conf_get("spark.task.resource.gpu.amount")
    if task_gpu is not None and float(task_gpu) == float(gpus):
        return None, "spark.task.resource.gpu.amount equals the executor's: already one task per GPU"
    # more than half of the executor's cores => two training tasks never share an executor; with the RAPIDS SQL plugin
    # active the training task takes the whole executor so that no ETL task runs beside it
    sql_plugin = "com.nvidia.spark.SQLPlugin" in (plugins or "") and str(rapids_sql_enabled).lower() == "true"
    task_cpus = int(cores) if sql_plugin else int(cores) // 2 + 1
    return (task_cpus, 1.0), "training tasks require cores=%d, gpu=1.0" % task_cpus


def try_stage_level_scheduling(rdd: Any, dataset: Any) -> Any:
    """rdd.withResources(profile) when stage_level_scheduling_plan says so; any surprise leaves the RDD as it is."""
    try:
        session = dataset.sparkSession
        sc = session.sparkContext
        sconf = sc.getConf()
        plan, _ = stage_level_scheduling_plan(str(session.version), lambda k: sconf.get(k), is_local(dataset),
                                              session.conf.get("spark.plugins", " "),
                                              session.conf.get("spark.rapids.sql.enabled", "true"))
        if plan is None:
            return rdd
        from pyspark.resource.profile import ResourceProfileBuilder
        from pyspark.resource.requests import TaskResourceRequests

        treqs = TaskResourceRequests().cpus(plan[0]).resource("gpu", plan[1])
        return rdd.withResources(ResourceProfileBuilder().require(treqs).build)
    except Exception:
        return rdd


def current_barrier_context() -> Any:
    """Inside a Spark barrier task: pyspark.BarrierTaskContext.get()."""
    from pyspark import BarrierTaskContext

    return BarrierTaskContext.get()


def transform_with_pandas_udf(model: Any, dataset: Any, data_alias: str, set_gpu: Callable[[Any, bool], int]) -> Any:
    """reference core.py:1797-1941 for a single output column: pandas_udf over struct(features) + withColumn."""
    from pyspark.ml.functions import vector_to_array
    from pyspark.ml.linalg import VectorUDT
    from pyspark.sql.functions import col, pandas_udf, struct

    input_col, input_cols = model._get_input_columns()
    construct, transform_internal, _ = model._get_cuml_transform_func(dataset)
    local = is_local(dataset)
    if input_col is not None:
        dtype = dataset.schema[input_col].dataType
        if isinstance(dtype, VectorUDT):
            select_cols = [vector_to_array(col(input_col), "float32" if model._float32_inputs else "float64").alias(data_alias)]
        else:
            select_cols = [col(input_col).alias(data_alias)]
    else:
        select_cols = [col(c) for c in (input_cols or [])]

    @pandas_udf(model._out_schema(dataset.schema))   # "int" (KMeans), "array<float>" (PCA)
    def predict_udf(iterator: Iterator[pd.DataFrame]) -> Iterator[pd.Series]:
        from pyspark import TaskContext

        gpu = set_gpu(TaskContext.get(), local)
        device_model = construct(gpu)
        try:
            from .core import _iter_transform   # groups consecutive batches into one device pass where possible

            yield from _iter_transform(transform_internal, lambda: device_model, iterator)
        finally:
            if hasattr(device_model, "close"):
                device_model.close()

    return dataset.withColumn(model._output_col_name(), predict_udf(struct(*select_cols)))


def _extra_metadata(inst: Any) -> dict:
    return {"_cuml_params": inst._cuml_params, "_num_workers": inst._num_workers, "_float32_inputs": inst._float32_inputs}


def make_writer(inst: Any, model_attributes: Optional[dict]) -> Any:
    """MLWriter for an estimator (model_attributes None) or a model — reference core.py:268-288, 310-332."""
    import json
    import os

    from pyspark.ml.util import DefaultParamsWriter, MLWriter

    class _B2kWriter(MLWriter):
        def saveImpl(self, path: str) -> None:
            DefaultParamsWriter.saveMetadata(inst, path, self.sc, extraMetadata=_extra_metadata(inst))
            if model_attributes is not None:
                self.sc.parallelize([json.dumps(model_attributes)], 1).saveAsTextFile(os.path.join(path, "data"))

    return _B2kWriter()


def make_reader(cls: Any, is_model: bool) -> Any:
    """MLReader for an estimator or a model class — reference core.py:291-307, 335-355."""
    import json
    import os

    from pyspark.ml.util import DefaultParamsReader, MLReader

    class _B2kReader(MLReader):
        def load(self, path: str) -> Any:
            metadata = DefaultParamsReader.loadMetadata(path, self.sc)
            if is_model:
                attrs = json.loads(self.sc.textFile(os.path.join(path, "data")).collect()[0])
                inst = cls(**attrs)
            else:
                inst = cls()
            inst._resetUid(metadata["uid"])
            DefaultParamsReader.getAndSetParams(inst, metadata)
            inst._cuml_params = metadata["_cuml_params"]
            inst._num_workers = metadata["_num_workers"]
            inst._float32_inputs = metadata["_float32_inputs"]
            return inst

    return _B2kReader()
