"""Spark-Param <-> backend-param plumbing (mirrors the reference's params.py:162-707 semantics; written
against sparkshim.Params when pyspark is absent).

  _param_mapping()           Spark Param name -> backend param name | "" (ignored, warn) | None (unsupported)
  _param_value_mapping()     backend param name -> value mapper (None result = unsupported value)
  _get_cuml_params_default() backend defaults
  cuml_params / num_workers / _set_params / clear / _use_cpu_fallback     as in the reference
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple, TypeVar, Union

from .sparkshim import Param, Params, TypeConverters, get_session
from .utils import get_logger

P = TypeVar("P", bound="_CumlParams")


class HasFeaturesCols(Params):
    """reference: params.py:69-88 — multi-column (scalar) feature input."""

    featuresCols = Param("parent", "featuresCols", "features column names for multi-column input.",
                         TypeConverters.toListString)

    def getFeaturesCols(self) -> List[str]:
        return self.getOrDefault(self.featuresCols)


class HasFeaturesCol(Params):
    featuresCol = Param("parent", "featuresCol", "features column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(featuresCol="features")


class HasPredictionCol(Params):
    predictionCol = Param("parent", "predictionCol", "prediction column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(predictionCol="prediction")

    def getPredictionCol(self) -> str:
        return self.getOrDefault(self.predictionCol)


class HasVerboseParam(Params):
    """reference: params.py:144-159."""

    verbose = Param("parent", "verbose", "logging level (bool or 0..6).")

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(verbose=False)


class _KMeansParams(HasFeaturesCol, HasPredictionCol):
    """pyspark.ml.clustering._KMeansParams stand-in: the Spark-side Params with Spark's defaults
    (k=2, initMode='k-means||', initSteps=2, tol=1e-4, maxIter=20, distanceMeasure='euclidean')."""

    k = Param("parent", "k", "The number of clusters to create. Must be > 1.", TypeConverters.toInt)
    initMode = Param("parent", "initMode", 'The initialization algorithm: "random" or "k-means||".',
                     TypeConverters.toString)
    initSteps = Param("parent", "initSteps", "The number of steps for k-means|| initialization mode.",
                      TypeConverters.toInt)
    tol = Param("parent", "tol", "the convergence tolerance for iterative algorithms (>= 0).", TypeConverters.toFloat)
    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    distanceMeasure = Param("parent", "distanceMeasure", "the distance measure: 'euclidean' or 'cosine'.",
                            TypeConverters.toString)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)
    solver = Param("parent", "solver", "The solver algorithm for optimization.", TypeConverters.toString)
    maxBlockSizeInMB = Param("parent", "maxBlockSizeInMB", "maximum memory in MB for stacking input data.",
                             TypeConverters.toFloat)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(k=2, initMode="k-means||", initSteps=2, tol=1e-4, maxIter=20,
                         distanceMeasure="euclidean", solver="auto", maxBlockSizeInMB=0.0)

    def getK(self) -> int:
        return self.getOrDefault(self.k)

    def getInitMode(self) -> str:
        return self.getOrDefault(self.initMode)

    def getInitSteps(self) -> int:
        return self.getOrDefault(self.initSteps)

    def getTol(self) -> float:
        return self.getOrDefault(self.tol)

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getSeed(self) -> int:
        return self.getOrDefault(self.seed)

    def getDistanceMeasure(self) -> str:
        return self.getOrDefault(self.distanceMeasure)


class HasInputCol(Params):
    inputCol = Param("parent", "inputCol", "input column name.", TypeConverters.toString)


class HasInputCols(Params):
    """reference: params.py:91-107 — multi-column (scalar) input of a feature transformer."""

    inputCols = Param("parent", "inputCols", "input column names.", TypeConverters.toListString)

    def getInputCols(self) -> List[str]:
        return self.getOrDefault(self.inputCols)


class HasIDCol(Params):
    """reference: params.py:127-141 — the column that identifies each row (k-NN items and queries)."""

    idCol = Param("parent", "idCol", "id column name.", TypeConverters.toString)

    def getIdCol(self) -> Optional[str]:
        return self.getOrDefault(self.idCol)


class HasLabelCol(Params):
    labelCol = Param("parent", "labelCol", "label column name.", TypeConverters.toString)

    def getLabelCol(self) -> str:
        return self.getOrDefault(self.labelCol)


class HasOutputCol(Params):
    outputCol = Param("parent", "outputCol", "output column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(outputCol=self.uid + "__output")   # pyspark's HasOutputCol default

    def getOutputCol(self) -> str:
        return self.getOrDefault(self.outputCol)


class _PCAParams(HasInputCol, HasOutputCol):
    """pyspark.ml.feature._PCAParams stand-in: k (no default), inputCol, outputCol."""

    k = Param("parent", "k", "the number of principal components (> 0).", TypeConverters.toInt)

    def getK(self) -> int:
        return self.getOrDefault(self.k)


class _CumlClass(object):
    """reference: params.py:162-257."""

    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {}

    @classmethod
    def _param_value_mapping(cls) -> Dict[str, Callable[[Any], Union[None, str, float, int]]]:
        return {}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        raise NotImplementedError

    def _pyspark_class(self) -> Optional[type]:
        return None


class _CumlParams(_CumlClass, HasVerboseParam, Params):
    """reference: params.py:260-707."""

    _cuml_params: Dict[str, Any] = {}
    _num_workers: Optional[int] = None
    _float32_inputs: bool = True
    _fallback_enabled: bool = False

    def __init__(self) -> None:
        super().__init__()
        self.logger = get_logger(self.__class__)
        fb = get_session().conf.get("spark.rapids.ml.cpu.fallback.enabled", "false")
        if fb not in ("true", "false"):
            raise ValueError(f"unknown value {fb} for spark.rapids.ml.cpu.fallback.enabled")
        self._fallback_enabled = fb == "true"

    @property
    def cuml_params(self) -> Dict[str, Any]:
        return self._cuml_params

    @property
    def num_workers(self) -> int:
        inferred = self._infer_num_workers()
        if self._num_workers is not None:
            if inferred < self._num_workers:
                raise ValueError(
                    f"The num_workers ({self._num_workers}) should be less than or equal to total GPUs ({inferred})")
            return self._num_workers
        return inferred

    @num_workers.setter
    def num_workers(self, value: int) -> None:
        self._num_workers = value

    def _infer_num_workers(self) -> int:
        """reference: params.py:556-588 infers GPUs from the Spark cluster; locally: visible CUDA devices
        (>= 1 so that param plumbing is testable on a CPU box)."""
        conf = get_session().conf.get("spark.rapids.ml.num_workers.local", None)
        if conf is not None:
            return int(conf)
        try:
            import torch

            n = torch.cuda.device_count()
        except Exception:
            n = 0
        return max(1, n)

    def copy(self: P, extra: Optional[Dict[Param, Any]] = None) -> P:
        that = super().copy(extra)  # type: ignore[misc]
        that._cuml_params = dict(self._cuml_params)
        if extra:
            for p, v in extra.items():
                if that.hasParam(p.name):
                    that._set_cuml_param(p.name, v, silent=True)
        return that

    def _initialize_cuml_params(self) -> None:
        self._cuml_params = self._get_cuml_params_default()
        for spark_param in self._param_mapping().keys():
            if self.hasParam(spark_param) and self.hasDefault(spark_param):
                self._set_cuml_param(spark_param, self.getOrDefault(spark_param))

    def _set_params(self: P, **kwargs: Any) -> P:
        param_map = self._param_mapping()
        for spark_param, cuml_param in param_map.items():
            if spark_param != cuml_param and spark_param in kwargs and cuml_param in kwargs:
                raise ValueError(f"'{cuml_param}' is an alias of '{spark_param}', set one or the other.")
        for k, v in kwargs.items():
            if k in ("featuresCol", "inputCol") and self.hasParam(k):   # a list selects the multi-column param
                if isinstance(v, str):
                    self._set(**{k: v})
                elif isinstance(v, list):
                    self._set(**{k + "s": v})
            elif self.hasParam(k):
                self._set(**{k: v})
                self._set_cuml_param(k, v, silent=self._fallback_enabled)
            elif k in self.cuml_params:
                self._cuml_params[k] = v
                for spark_param, cuml_param in param_map.items():
                    if k == cuml_param and self.hasParam(spark_param):
                        try:
                            self._set(**{spark_param: v})
                        except TypeError:
                            pass
            elif k == "num_workers":
                self._num_workers = v
            elif k == "float32_inputs":
                self._float32_inputs = v
            else:
                raise ValueError(f"Unsupported param '{k}'.")
        return self

    def clear(self, param: Param) -> None:
        super().clear(param)
        cuml_param = self._param_mapping().get(param.name)
        if cuml_param:
            self._set_cuml_value(cuml_param, self.getOrDefault(param.name))

    def _copy_cuml_params(self: P, to: P) -> P:
        to._cuml_params = dict(self._cuml_params)
        to._num_workers = self._num_workers
        to._float32_inputs = self._float32_inputs
        return to

    def _get_input_columns(self) -> Tuple[Optional[str], Optional[List[str]]]:
        """reference: params.py:521-554."""
        for multi, single in (("featuresCols", "featuresCol"), ("inputCols", "inputCol")):
            if self.hasParam(multi) and self.isDefined(multi):
                return None, self.getOrDefault(multi)
            if self.hasParam(single) and self.isDefined(single):
                return self.getOrDefault(single), None
        raise ValueError("Please set inputCol(s) or featuresCol(s)")

    def _get_cuml_param(self, spark_param: str, silent: bool = True) -> Optional[str]:
        param_map = self._param_mapping()
        if spark_param in param_map:
            cuml_param = param_map[spark_param]
            if cuml_param is None:
                if not silent:
                    raise ValueError(f"Spark Param '{spark_param}' is not supported by cuML.")
            elif cuml_param == "":
                if not silent:
                    print(f"WARNING: Spark Param '{spark_param}' is not used by cuML.")
                cuml_param = None
            return cuml_param
        if spark_param in self.cuml_params:
            return spark_param
        return None

    def _set_cuml_param(self, spark_param: str, spark_value: Any, silent: bool = True) -> None:
        cuml_param = self._get_cuml_param(spark_param, silent)
        if cuml_param is not None:
            try:
                self._set_cuml_value(cuml_param, spark_value)
            except ValueError:
                if not self._fallback_enabled:
                    ref = cuml_param + " or " + spark_param if cuml_param != spark_param else spark_param
                    raise ValueError(f"{ref} given an invalid or unsupported value {spark_value}")

    def _get_cuml_mapping_value(self, k: str, v: Any) -> Any:
        value_map = self._param_value_mapping()
        if k not in value_map:
            return v
        mapped = value_map[k](v)
        if mapped is None:
            raise ValueError(f"Value '{v}' for '{k}' param is unsupported")
        return mapped

    def _set_cuml_value(self, k: str, v: Any) -> None:
        self._cuml_params[k] = self._get_cuml_mapping_value(k, v)

    def _use_cpu_fallback(self, params: Optional[Dict[Param, Any]] = None) -> bool:
        """reference: params.py:690-707.  Reports whether the reference WOULD fall back to pyspark.ml on CPU;
        this build has no CPU path, so callers raise instead of falling back."""
        mapping, vmap = self._param_mapping(), self._param_value_mapping()
        fallback = False
        for param, value in (params if params else self.extractParamMap()).items():
            if param.name in mapping:
                mapped = mapping[param.name]
                if (not mapped and mapped is None and (self.isSet(param) or params)) or (
                        mapped and mapped in vmap and vmap[mapped](value) is None):
                    get_logger(self.__class__).warning(
                        f"Setting Spark Param '{param.name}' to '{value}' is not supported on GPU.")
                    fallback = True
        return fallback
