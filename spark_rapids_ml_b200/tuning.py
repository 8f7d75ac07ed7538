"""K-fold cross validation on local frames: every fold fits the whole param grid from one ingest (fitMultiple), packs
the fitted models into one (_combine) and scores all of them in one device pass over the validation rows
(_transformEvaluate), as the reference's CrossValidator does (python tuning.py:92-157).

Folds (a local rule: Spark's rand(seed) cannot be reproduced without the JVM): without foldCol, row r of the frame in
global order is in validation fold floor(k u_r), u = numpy.random.default_rng(seed).random(n); with foldCol, the
column gives the fold and a value outside [0, k) is an error.  The folds run in order on one GPU; `parallelism` is
accepted and has no effect.
"""
from __future__ import annotations

import itertools
import json
import os
import zlib
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa

from .sparkshim import HAVE_PYSPARK, Param, Params, TypeConverters, keyword_only


class ParamGridBuilder:
    """pyspark.ml.tuning.ParamGridBuilder: the product of the grids, the first addGrid varying slowest."""

    def __init__(self) -> None:
        self._grid: Dict[Any, List[Any]] = {}

    def addGrid(self, param: Any, values: Sequence[Any]) -> "ParamGridBuilder":
        self._grid[param] = list(values)
        return self

    def baseOn(self, *args: Any) -> "ParamGridBuilder":
        pairs = args[0].items() if len(args) == 1 and isinstance(args[0], dict) else args
        for p, v in pairs:
            self._grid[p] = [v]
        return self

    def build(self) -> List[Dict[Any, Any]]:
        keys = list(self._grid)
        return [dict(zip(keys, vals)) for vals in itertools.product(*(self._grid[k] for k in keys))]


def _row_count(df: Any) -> int:
    return sum(b.num_rows for p in df._parts for b in p)


def fold_ids(df: Any, k: int, seed: int, fold_col: Optional[str] = None) -> np.ndarray:
    """The validation fold of every row of a local frame, in global row order."""
    if fold_col:
        f = np.concatenate([np.asarray(b.column(fold_col).to_numpy(zero_copy_only=False)) for p in df._parts
                            for b in p]) if _row_count(df) else np.zeros(0)
        if f.size and (np.any(f < 0) or np.any(f >= k) or np.any(f != np.floor(f))):
            bad = f[(f < 0) | (f >= k) | (f != np.floor(f))][0]
            raise ValueError(f"Fold number must be in range [0, {k}), but got {bad}.")
        return f.astype(np.int64)
    u = np.random.default_rng(seed).random(_row_count(df))
    return np.minimum((k * u).astype(np.int64), k - 1)


def _take(df: Any, mask: np.ndarray, drop: Optional[str], parts: int) -> Any:
    table = df._table()
    t = table.filter(pa.array(mask))
    if drop:
        t = t.drop([drop])
    from .sparkshim.sql import _split_table

    return df._derive(_split_table(t, max(1, parts), df.sparkSession.max_records_per_batch), t.schema)


def k_fold(df: Any, k: int, seed: int, fold_col: Optional[str], parts: int) -> List[Any]:
    """[(train, validation)] per fold; the training frames are split into `parts` partitions."""
    ids = fold_ids(df, k, seed, fold_col)
    return [(_take(df, ids != i, fold_col, parts), _take(df, ids == i, fold_col, df.getNumPartitions()))
            for i in range(k)]


class _CrossValidatorParams(Params):
    estimator = Param("parent", "estimator", "estimator to be cross-validated")
    estimatorParamMaps = Param("parent", "estimatorParamMaps", "estimator param maps")
    evaluator = Param("parent", "evaluator", "evaluator used to select hyper-parameters that maximize the validator "
                      "metric")
    numFolds = Param("parent", "numFolds", "number of folds for cross validation", TypeConverters.toInt)
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    parallelism = Param("parent", "parallelism", "the number of threads to use when running parallel algorithms "
                        "(no effect here: the folds share one GPU and run in order)", TypeConverters.toInt)
    collectSubModels = Param("parent", "collectSubModels", "whether to collect a list of sub-models trained during "
                             "tuning.", TypeConverters.identity)
    foldCol = Param("parent", "foldCol", "Param for the column name of user specified fold number.",
                    TypeConverters.toString)

    def _cv_defaults(self) -> None:
        self._setDefault(numFolds=3, seed=zlib.crc32(b"CrossValidator") & 0x7FFFFFFF, parallelism=1,
                         collectSubModels=False, foldCol="")

    def getEstimator(self) -> Any:
        return self.getOrDefault("estimator")

    def getEstimatorParamMaps(self) -> List[Dict[Any, Any]]:
        return self.getOrDefault("estimatorParamMaps")

    def getEvaluator(self) -> Any:
        return self.getOrDefault("evaluator")

    def getNumFolds(self) -> int:
        return self.getOrDefault("numFolds")

    def getSeed(self) -> int:
        return self.getOrDefault("seed")

    def getParallelism(self) -> int:
        return self.getOrDefault("parallelism")

    def getCollectSubModels(self) -> bool:
        return bool(self.getOrDefault("collectSubModels"))

    def getFoldCol(self) -> str:
        return self.getOrDefault("foldCol")


class CrossValidator(_CrossValidatorParams):
    """K-fold cross validation over a param grid; see the module docstring for the fold rule.

    >>> from spark_rapids_ml_b200.classification import LogisticRegression
    >>> from spark_rapids_ml_b200.evaluation import MulticlassClassificationEvaluator
    >>> from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder
    >>> lr = LogisticRegression()
    >>> grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.1]).build()
    >>> cv = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=MulticlassClassificationEvaluator())
    >>> cv.fit(df).avgMetrics
    """

    @keyword_only
    def __init__(self, *, estimator: Any = None, estimatorParamMaps: Optional[List[Dict[Any, Any]]] = None,
                 evaluator: Any = None, numFolds: int = 3, seed: Optional[int] = None, parallelism: int = 1,
                 collectSubModels: bool = False, foldCol: str = "") -> None:
        super().__init__()
        self._cv_defaults()
        self._set(**{k: v for k, v in self._input_kwargs.items() if v is not None})

    def setParams(self, **kwargs: Any) -> "CrossValidator":
        return self._set(**{k: v for k, v in kwargs.items() if v is not None})

    def setNumFolds(self, value: int) -> "CrossValidator":
        return self._set(numFolds=value)

    def setSeed(self, value: int) -> "CrossValidator":
        return self._set(seed=value)

    def setFoldCol(self, value: str) -> "CrossValidator":
        return self._set(foldCol=value)

    def setCollectSubModels(self, value: bool) -> "CrossValidator":
        return self._set(collectSubModels=value)

    def _check(self) -> None:
        k = self.getNumFolds()
        if k < 2:
            raise ValueError(f"numFolds must be >= 2, got {k}")
        est, eva = self.getEstimator(), self.getEvaluator()
        if not (hasattr(est, "_supportsTransformEvaluate") and est._supportsTransformEvaluate(eva)):
            raise NotImplementedError(f"CrossValidator of {type(est).__name__} with {type(eva).__name__} is not "
                                      "supported: this build has no CPU fallback")

    def fit(self, dataset: Any, params: Optional[Dict[Any, Any]] = None) -> "CrossValidatorModel":
        if params:
            return self.copy(params).fit(dataset)
        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):
                raise NotImplementedError("CrossValidator.fit() of a pyspark DataFrame is not supported in this build; "
                                          "fit a local frame")
        self._check()
        est, eva = self.getEstimator(), self.getEvaluator()
        if hasattr(est, "_check_tuning_input"):   # input the single-pass evaluation cannot read, refused before any fit
            est._check_tuning_input(dataset)
        maps = list(self.getEstimatorParamMaps())
        k = self.getNumFolds()
        parts = int(est.num_workers) if getattr(est, "num_workers", None) else dataset.getNumPartitions()
        folds = k_fold(dataset, k, self.getSeed(), self.getFoldCol() or None, parts)
        metrics_all: List[List[float]] = []
        sub_models: Optional[List[List[Any]]] = [] if self.getCollectSubModels() else None
        for train, valid in folds:
            models = [m for _, m in sorted(est.fitMultiple(train, maps), key=lambda t: t[0])]
            combined = models[0]._combine(models)
            metrics_all.append(list(combined._transformEvaluate(valid, eva)))
            if sub_models is not None:
                sub_models.append(models)
        avg = list(np.mean(metrics_all, axis=0))
        std = list(np.std(metrics_all, axis=0))
        best = int(np.argmax(avg) if eva.isLargerBetter() else np.argmin(avg))
        best_model = est.fit(dataset, maps[best])
        model = CrossValidatorModel(best_model, [float(a) for a in avg], sub_models, [float(s) for s in std])
        return self._copyValues(model)

    def write(self) -> "_CVWriter":
        return _CVWriter(self)

    def save(self, path: str) -> None:
        self.write().save(path)

    @classmethod
    def read(cls) -> "_CVReader":
        return _CVReader(cls)

    @classmethod
    def load(cls, path: str) -> "CrossValidator":
        return cls.read().load(path)


class CrossValidatorModel(_CrossValidatorParams):
    """The best model refitted on the whole frame, the fold-averaged metrics per param map (avgMetrics, stdMetrics) and,
    with collectSubModels, every fold's models.  transform() delegates to bestModel."""

    def __init__(self, bestModel: Any = None, avgMetrics: Optional[List[float]] = None,
                 subModels: Optional[List[List[Any]]] = None, stdMetrics: Optional[List[float]] = None) -> None:
        super().__init__()
        self._cv_defaults()
        self.bestModel = bestModel
        self.avgMetrics = list(avgMetrics or [])
        self.stdMetrics = list(stdMetrics or [])
        self.subModels = subModels

    def transform(self, dataset: Any, params: Optional[Dict[Any, Any]] = None) -> Any:
        return self.bestModel.transform(dataset) if not params else self.bestModel.copy(params).transform(dataset)

    def write(self) -> "_CVWriter":
        return _CVWriter(self)

    def save(self, path: str) -> None:
        self.write().save(path)

    @classmethod
    def read(cls) -> "_CVReader":
        return _CVReader(cls)

    @classmethod
    def load(cls, path: str) -> "CrossValidatorModel":
        return cls.read().load(path)


# ---- persistence: metadata JSON + estimator/, evaluator/ and bestModel/ written by their own writers ----
def _class_path(obj: Any) -> str:
    return f"{type(obj).__module__}.{type(obj).__name__}"


def _import(path: str) -> Any:
    import importlib

    mod, name = path.rsplit(".", 1)
    return getattr(importlib.import_module(mod), name)


def _save_params_obj(obj: Any, path: str) -> None:
    """An evaluator (no writer of its own here): its class and param values as JSON."""
    os.makedirs(path, exist_ok=True)
    vals = {p.name: v for p, v in obj._paramMap.items()}
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"class": _class_path(obj), "uid": obj.uid, "paramMap": vals}, f)


def _load_params_obj(path: str) -> Any:
    with open(os.path.join(path, "metadata.json")) as f:
        meta = json.load(f)
    obj = _import(meta["class"])()
    obj._set(**meta["paramMap"])
    return obj


class _CVWriter:
    def __init__(self, inst: Any) -> None:
        self.inst = inst
        self._overwrite = False

    def overwrite(self) -> "_CVWriter":
        self._overwrite = True
        return self

    def save(self, path: str) -> None:
        if os.path.exists(path) and not self._overwrite:
            raise FileExistsError(f"Path {path} already exists; use write().overwrite().save(path)")
        os.makedirs(path, exist_ok=True)
        inst = self.inst
        est = inst.getEstimator()
        maps = [[{"param": p.name, "value": v} for p, v in pm.items()] for pm in inst.getEstimatorParamMaps()]
        meta: Dict[str, Any] = {
            "class": _class_path(inst), "uid": inst.uid,
            "paramMap": {p.name: v for p, v in inst._paramMap.items()
                         if p.name not in ("estimator", "estimatorParamMaps", "evaluator")},
            "estimatorParamMaps": maps, "estimatorClass": _class_path(est), "evaluatorClass": _class_path(inst.getEvaluator())}
        if isinstance(inst, CrossValidatorModel):
            meta.update(avgMetrics=inst.avgMetrics, stdMetrics=inst.stdMetrics, bestModelClass=_class_path(inst.bestModel))
            inst.bestModel.write().overwrite().save(os.path.join(path, "bestModel"))
        with open(os.path.join(path, "metadata.json"), "w") as f:
            json.dump(meta, f)
        est.write().overwrite().save(os.path.join(path, "estimator"))
        _save_params_obj(inst.getEvaluator(), os.path.join(path, "evaluator"))


class _CVReader:
    def __init__(self, cls: Any) -> None:
        self.cls = cls

    def load(self, path: str) -> Any:
        with open(os.path.join(path, "metadata.json")) as f:
            meta = json.load(f)
        est = _import(meta["estimatorClass"]).load(os.path.join(path, "estimator"))
        eva = _load_params_obj(os.path.join(path, "evaluator"))
        maps = [{est.getParam(e["param"]): e["value"] for e in pm} for pm in meta["estimatorParamMaps"]]
        if self.cls is CrossValidatorModel or meta["class"].endswith("CrossValidatorModel"):
            best = _import(meta["bestModelClass"]).load(os.path.join(path, "bestModel"))
            out: Any = CrossValidatorModel(best, meta["avgMetrics"], None, meta["stdMetrics"])
        else:
            out = CrossValidator()
        out._set(**meta["paramMap"])
        out._set(estimator=est, estimatorParamMaps=maps, evaluator=eva)
        return out
