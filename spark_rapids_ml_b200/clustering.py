"""KMeans / KMeansModel — the reference's PySpark-ML Estimator/Model surface for the distributed KMeans.fit()
path (python/src/spark_rapids_ml/clustering.py:84-604), with the cuML calls replaced by libb2kmeans
(hand-written sm_90a CUDA behind include/b2kmeans.h).

Same names, argument meaning and error behaviour as the reference:
  KMeansClass._param_mapping / _param_value_mapping / _get_cuml_params_default      clustering.py:84-141
  _KMeansCumlParams (featuresCol/featuresCols handling, seed default)                clustering.py:144-186
  KMeans (keyword-only ctor, setters, _get_cuml_fit_func, _out_schema,
          _create_pyspark_model, _merge_model_chunks)                                clustering.py:189-502
  KMeansModel (clusterCenters, hasSummary, predict, _get_cuml_transform_func)        clustering.py:505-604
  KMeans.fitMultiple / KMeansModel._transformEvaluate: CrossValidator(KMeans, ClusteringEvaluator), which the
  reference hands to pyspark's CrossValidator (GPU fits, CPU silhouette); here every fold's grid fits from one ingest
  and its models are scored in one device silhouette pass (b2k_silhouette_multi)
  DBSCANClass, _DBSCANCumlParams, DBSCAN (lazy fit), DBSCANModel.transform             clustering.py:607-1186
  GaussianMixture / BisectingKMeans: Spark's estimators of those names, which the reference lacks

Differences that are deliberate: no CPU fallback (cpu() / single-vector predict need a JVM and raise), and the
fit function receives a DEVICE matrix from the worker scaffold instead of host arrays to concatenate.  DBSCAN: every
rank returns the labels of its own rows (the reference's come from rank 0 only), and transform of a pyspark DataFrame
raises NotImplementedError.
"""
from __future__ import annotations

import functools
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pyarrow as pa

from .core import (FitInputType, _CumlCaller, _CumlEstimator, _CumlModelWithPredictionCol, _DeviceModel,
                   _TunedEstimator, alias, param_alias)
from .params import HasFeaturesCol, HasFeaturesCols, HasIDCol, HasPredictionCol, P, _CumlClass, _CumlParams, _KMeansParams
from .sparkshim import HAVE_PYSPARK, Param, Row, TypeConverters, keyword_only
from .utils import get_logger


class KMeansClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        # reference: clustering.py:86-98 — None = unsupported on GPU, "" = accepted and ignored
        return {
            "distanceMeasure": None,
            "initMode": "init",
            "k": "n_clusters",
            "initSteps": "",
            "maxIter": "max_iter",
            "seed": "random_state",
            "tol": "tol",
            "weightCol": None,
            "solver": "",
            "maxBlockSizeInMB": "",
        }

    @classmethod
    def _param_value_mapping(cls) -> Dict[str, Callable[[Any], Union[None, str, float, int]]]:
        def tol_value_mapper(x: float) -> float:
            if x == 0.0:  # reference: clustering.py:113-123
                get_logger(cls).warning(
                    "tol=0 is not supported in cuml yet. "
                    + "It will be mapped to smallest positive float, i.e. numpy.finfo('float32').tiny.")
                return np.finfo("float32").tiny.item()
            return x

        def init_value_mapper(x: str) -> Optional[str]:
            return {"k-means||": "scalable-k-means++", "scalable-k-means++": "scalable-k-means++",
                    "random": "random"}.get(x)

        return {"tol": tol_value_mapper, "init": init_value_mapper}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        # reference: clustering.py:127-138 (the cuML KMeans signature defaults it pins in its tests)
        return {
            "n_clusters": 8,
            "max_iter": 300,
            "tol": 0.0001,
            "verbose": False,
            "random_state": None,
            "init": "scalable-k-means++",
            "n_init": "auto",
            "oversampling_factor": 2.0,
            "max_samples_per_batch": 32768,
        }

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.clustering.KMeans when pyspark is installed


class _KMeansCumlParams(_CumlParams, _KMeansParams, HasFeaturesCols):
    """Shared Spark Params of KMeans and KMeansModel (reference: clustering.py:144-186)."""

    def __init__(self) -> None:
        super().__init__()
        # restrict the default seed to a 32-bit signed integer, as the reference does for cuML
        self._setDefault(seed=hash(type(self).__name__) & 0x07FFFFFFF)

    def getFeaturesCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.featuresCols):
            return self.getFeaturesCols()
        if self.isDefined(self.featuresCol):
            return self.getOrDefault("featuresCol")
        raise RuntimeError("featuresCol is not set")

    def setFeaturesCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(featuresCol=value)
        else:
            self._set_params(featuresCols=value)
        return self

    def setFeaturesCols(self: P, value: List[str]) -> P:
        return self._set_params(featuresCols=value)

    def setPredictionCol(self: P, value: str) -> P:
        self._set_params(predictionCol=value)
        return self


class KMeans(KMeansClass, _TunedEstimator, _KMeansCumlParams):
    """KMeans on H100: one barrier task per GPU; each iteration is ONE fused pass over the device-resident
    partition (TMA -> wgmma 3xTF32 distance tile -> argmin, then per-cluster partial sums) followed by one NCCL
    allreduce of the [k*d sums | k counts] buffer.  Parameters as in the reference (clustering.py:197-236):

    k (default 2), initMode ("k-means||" | "random"), maxIter (20), tol (1e-4), seed, featuresCol (str for an
    array column, list of str for scalar columns), predictionCol, num_workers, verbose.

    >>> from spark_rapids_ml_b200.clustering import KMeans
    >>> df = session.createDataFrame([([0.0, 0.0],), ([1.0, 1.0],), ([9.0, 8.0],), ([8.0, 9.0],)], ["features"])
    >>> model = KMeans(k=2).setFeaturesCol("features").setMaxIter(10).fit(df)
    >>> sorted(c.tolist() for c in model.clusterCenters())
    [[0.5, 0.5], [8.5, 8.5]]
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", predictionCol: str = "prediction",
                 k: int = 2, initMode: str = "k-means||", tol: float = 0.0001, maxIter: int = 20,
                 seed: Optional[int] = None, num_workers: Optional[int] = None,
                 verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()   # session-wide defaults for arguments not passed (clustering.py:315)
        # if the user does not override it, n_init = 1 to match Spark behaviour (clustering.py:316-319)
        if "n_init" not in self._input_kwargs:
            self._input_kwargs["n_init"] = 1
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        if self._input_kwargs.get("seed", None) is None:
            self._input_kwargs.pop("seed", None)
        if self._input_kwargs.get("num_workers", None) is None:
            self._input_kwargs.pop("num_workers", None)
        self._set_params(**self._input_kwargs)

    def setInitMode(self, value: str) -> "KMeans":
        return self._set_params(initMode=value)

    def setK(self, value: int) -> "KMeans":
        return self._set_params(k=value)

    def setMaxIter(self, value: int) -> "KMeans":
        return self._set_params(maxIter=value)

    def setSeed(self, value: int) -> "KMeans":
        if value > 0x07FFFFFFF:
            raise ValueError("cuML seed value must be a 32-bit integer.")
        return self._set_params(seed=value)

    def setTol(self, value: float) -> "KMeans":
        return self._set_params(tol=value)

    def setWeightCol(self, value: str) -> "KMeans":
        raise ValueError("'weightCol' is not supported by cuML.")

    # every map is fitted in turn on the same device matrix
    _single_pass_params = frozenset(("k", "maxIter", "tol", "seed", "initMode"))

    def _settings(self) -> Dict[str, Any]:
        return dict(self.cuml_params)

    def _fit_array_order(self) -> str:
        return "C"

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        cls = self.__class__
        grid = self._fit_grid

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            if grid is None:
                return _fit_one(dfs, params)
            rows: Dict[str, List[Any]] = {}
            for init in grid:   # one fit per param map on the same device matrix, in map order
                for key, v in _fit_one(dfs, {**params, param_alias.cuml_init: init,
                                             param_alias.fit_multiple_params: True}).items():
                    rows.setdefault(key, []).extend(v)
            return rows

        def _fit_one(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for KMeansMG(handle, **cuml_init).fit(concated) — clustering.py:381-415
            ctx = params[param_alias.handle]
            init = dict(params[param_alias.cuml_init])
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            X = dfs[0][0]
            n_init = init.get("n_init", 1)
            out = ctx.kmeans_fit(
                X,
                int(init["n_clusters"]),
                init=init.get("init", "scalable-k-means++"),
                max_iter=int(init["max_iter"]),
                tol=float(init["tol"]),
                seed=int(init["random_state"]) if init.get("random_state") is not None else 0,
                oversampling_factor=float(init.get("oversampling_factor", 2.0)),
                n_init=1 if n_init == "auto" else int(n_init),
            )
            get_logger(cls).info(f"iterations: {out['n_iter_']}, inertia: {out['inertia_']}")
            all_centers = out["cluster_centers_"].cpu().numpy().astype(np.float64).tolist()
            n_cols = params[param_alias.num_cols]
            dtype_str = "float32"
            if params.get(param_alias.fit_multiple_params):
                return {"chunk_id": [0], "cluster_centers_": [all_centers], "n_cols": [n_cols], "dtype": [dtype_str]}
            # chunk the centers so that one model row stays under Spark's ~2 GB buffer limit (clustering.py:437-454)
            max_bytes_per_chunk = 1024 ** 3
            max_centers_per_chunk = max(1, max_bytes_per_chunk // (n_cols * 8))
            chunks = [all_centers[s:s + max_centers_per_chunk] for s in range(0, len(all_centers), max_centers_per_chunk)]
            return {"chunk_id": list(range(len(chunks))), "cluster_centers_": chunks,
                    "n_cols": [n_cols] * len(chunks), "dtype": [dtype_str] * len(chunks)}

        return _cuml_fit

    def _supportsTransformEvaluate(self, evaluator: Any) -> bool:
        """CrossValidator scores KMeans models with a ClusteringEvaluator's silhouette, either distance measure."""
        return _supports_silhouette(evaluator)

    def _out_schema(self) -> Any:
        # reference: clustering.py:458-468
        return "chunk_id int, cluster_centers_ array<array<double>>, n_cols int, dtype string"

    def _create_pyspark_model(self, result: Row) -> "KMeansModel":
        return KMeansModel(**result.asDict())

    def _merge_model_chunks(self, rows: List[Row], paramMaps: Optional[Sequence[Dict[Any, Any]]] = None) -> List[Row]:
        # reference: clustering.py:473-502
        def _one_model_row(chunk_rows: List[Row]) -> Row:
            srt = sorted(chunk_rows, key=lambda r: r["chunk_id"])
            merged: List[List[float]] = []
            for row in srt:
                merged.extend([list(map(float, c)) for c in row["cluster_centers_"]])
            return Row(cluster_centers_=merged, n_cols=int(srt[0]["n_cols"]), dtype=srt[0]["dtype"])

        if paramMaps is None:
            if len(rows) == 0:
                raise ValueError("Expected at least one fit result row but got none")
            return [_one_model_row(rows)]
        assert len(rows) == len(paramMaps)
        return [_one_model_row([r]) for r in rows]


class KMeansModel(KMeansClass, _CumlModelWithPredictionCol, _KMeansCumlParams):
    """reference: clustering.py:505-604."""

    def __init__(self, cluster_centers_: List[List[float]], n_cols: int, dtype: str):
        super().__init__(n_cols=n_cols, dtype=dtype, cluster_centers_=cluster_centers_)
        self.cluster_centers_ = cluster_centers_

    def cpu(self) -> Any:
        raise NotImplementedError("KMeansModel.cpu() builds a JVM pyspark.ml KMeansModel; no JVM/pyspark in this build")

    def clusterCenters(self) -> List[np.ndarray]:
        return [np.array(x) for x in self.cluster_centers_]

    @property
    def hasSummary(self) -> bool:
        return False

    def predict(self, value: Any) -> int:
        """The reference falls back to the JVM model for a single vector (clustering.py:555-559); here the single
        row goes through the same device kernel."""
        v = np.asarray(value.toArray() if hasattr(value, "toArray") else value, dtype=np.float32).reshape(1, -1)
        from . import _native
        import torch

        with _native.Context(torch.cuda.current_device() if torch.cuda.is_available() else 0) as ctx:
            C = torch.tensor(self.cluster_centers_, dtype=torch.float32, device=ctx.device)
            labels, _ = ctx.kmeans_assign(torch.from_numpy(v).to(ctx.device), C)
            return int(labels[0].item())

    def _out_schema(self, input_schema: Any = None) -> str:
        return "int"

    def _transform_array_order(self) -> str:
        return "C"

    def _center_sets(self) -> List[List[List[float]]]:
        """The centres of each model of this (combined) model."""
        c = self.cluster_centers_
        return [c] if len(c) == 0 or not isinstance(c[0][0], (list, tuple)) else list(c)  # type: ignore[list-item]

    _combined_attrs = ("cluster_centers_",)

    def _transformEvaluate(self, dataset: Any, evaluator: Any, params: Optional[Dict[Any, Any]] = None) -> List[float]:
        """The silhouette of every model of this (combined) model on a local frame, with the worker count and
        repartitioning that ClusteringEvaluator.evaluate uses: one barrier task per GPU ingests the features once,
        labels the rows with each model's centres as transform() does (b2k_kmeans_assign) and scores every model in one
        b2k_silhouette_multi call.  The evaluator's predictionCol is not read: the labels come from the models."""
        from .evaluation import _SilhouetteMultiCaller

        model = self.copy(params) if params else self
        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):
                raise NotImplementedError("KMeansModel._transformEvaluate() of a pyspark DataFrame is not supported in "
                                          "this build; evaluate a local frame")
        if not _supports_silhouette(evaluator):
            raise NotImplementedError(f"KMeansModel._transformEvaluate() does not support {type(evaluator).__name__}")
        if evaluator.isSet("weightCol") and evaluator.getOrDefault("weightCol"):
            raise NotImplementedError("weightCol is not supported by the device evaluation")
        ev_features, features = evaluator.getOrDefault("featuresCol"), model.getFeaturesCol()
        if list(np.atleast_1d(ev_features)) != list(np.atleast_1d(features)):
            raise NotImplementedError(f"the evaluator's featuresCol {ev_features!r} differs from the model's "
                                      f"featuresCol {features!r}: the device evaluation reads one features column")
        if dataset.count() == 0:
            raise ValueError("ClusteringEvaluator: the frame has no rows")
        caller = _SilhouetteMultiCaller(features, model._center_sets(), evaluator.getDistanceMeasure())
        res = caller._call_cuml_fit_func(dataset, partially_collect=True)
        rows = res if isinstance(res, list) else res.collect()
        return [float(v) for v in rows[0]["silhouette"]]

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        # the injected-centers predictor (clustering.py:582-596): b2k_kmeans_assign labels a group's rows
        construct = functools.partial(_DeviceModel, C=np.asarray(self.cluster_centers_, dtype=np.float32))
        transform = self._grouped_transform(lambda m, X: (m.ctx.kmeans_assign(X, m.arrays["C"])[0],),
                                            4 * int(self.n_cols or 1))
        return construct, transform, None


def _supports_silhouette(evaluator: Any) -> bool:
    if type(evaluator).__name__ != "ClusteringEvaluator":
        return False
    try:
        return (evaluator.getMetricName() == "silhouette" and
                evaluator.getDistanceMeasure() in ("squaredEuclidean", "cosine"))
    except Exception:
        return False


def _kmeans_grid_shares_ingest(paramMaps: Sequence[Dict[Any, Any]]) -> bool:
    """Whether KMeans.fitMultiple fits these maps from one ingest: every map changes only per-fit params."""
    return KMeans._shares_ingest(paramMaps)


# ---- DBSCAN (reference: clustering.py:607-1186) ----
class DBSCANClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"eps": 0.5, "min_samples": 5, "metric": "euclidean", "algorithm": "brute", "verbose": False,
                "max_mbytes_per_batch": None}

    def _pyspark_class(self) -> Optional[type]:
        return None   # pyspark.ml has no DBSCAN


class _DBSCANCumlParams(_CumlParams, HasFeaturesCol, HasFeaturesCols, HasIDCol, HasPredictionCol):
    """Shared Spark Params of DBSCAN and DBSCANModel (reference: clustering.py:626-730)."""

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(eps=0.5, min_samples=5, metric="euclidean", algorithm="brute", max_mbytes_per_batch=None,
                         idCol=alias.row_number)

    eps = Param("parent", "eps", "The maximum distance between 2 points such they reside in the same neighborhood.",
                TypeConverters.toFloat)
    min_samples = Param("parent", "min_samples", "The number of samples in a neighborhood such that this group can be "
                        "considered as an important core point (including the point itself).", TypeConverters.toInt)
    metric = Param("parent", "metric", "The metric to use when calculating distances between points.Spark Rapids ML "
                   "does not support the 'precomputed' mode from sklearn and cuML, please use those libraries instead.",
                   TypeConverters.toString)
    algorithm = Param("parent", "algorithm", "The algorithm to be used by for nearest neighbor computations.",
                      TypeConverters.toString)
    max_mbytes_per_batch = Param("parent", "max_mbytes_per_batch", "Calculate batch size using no more than this "
                                 "number of megabytes for the pairwise distance computation.", TypeConverters.toInt)

    def getFeaturesCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.featuresCols):
            return self.getFeaturesCols()
        if self.isDefined(self.featuresCol):
            return self.getOrDefault("featuresCol")
        raise RuntimeError("featuresCol is not set")

    def setFeaturesCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(featuresCol=value)
        else:
            self._set_params(featuresCols=value)
        return self

    def setFeaturesCols(self: P, value: List[str]) -> P:
        return self._set_params(featuresCols=value)

    def setPredictionCol(self: P, value: str) -> P:
        self._set_params(predictionCol=value)
        return self

    def setIdCol(self: P, value: str) -> P:
        self._set_params(idCol=value)
        return self


def _no_pyspark(dataset: Any) -> None:
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError("DBSCANModel.transform of a pyspark DataFrame is not supported yet; use a local "
                                      "frame")


class DBSCAN(DBSCANClass, _CumlEstimator, _DBSCANCumlParams):
    """DBSCAN on H100 (reference: clustering.py:733-934).  fit() is lazy and returns a DBSCANModel; the clustering runs
    in DBSCANModel.transform, one barrier task per GPU over the whole frame.  Parameters: eps (0.5), min_samples (5),
    metric ("euclidean" | "cosine"), algorithm ("brute" | "rbc": both run the same exact pass), max_mbytes_per_batch
    (accepted, unused: no pass here is batched by memory), featuresCol, predictionCol, idCol, num_workers, verbose.

    Labels follow include/b2kmeans.h: clusters are numbered by their lowest row; a border row that touches two clusters
    takes the cluster of its lowest adjacent core row, where scikit-learn and cuML take whichever expands first.

    >>> from spark_rapids_ml_b200.clustering import DBSCAN
    >>> df = session.createDataFrame([([1.0, 1.0],), ([1.0, 2.0],), ([5.0, 5.0],), ([5.0, 6.0],)], ["features"])
    >>> DBSCAN(eps=2.0, min_samples=2).fit(df).transform(df).collect()   # prediction 0, 0, 1, 1
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", predictionCol: str = "prediction",
                 eps: float = 0.5, min_samples: int = 5, metric: str = "euclidean", algorithm: str = "brute",
                 max_mbytes_per_batch: Optional[int] = None, num_workers: Optional[int] = None,
                 verbose: Union[int, bool] = False, idCol: str = alias.row_number, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        if self._input_kwargs.get("num_workers", None) is None:
            self._input_kwargs.pop("num_workers", None)
        self._set_params(**self._input_kwargs)
        self.cuml_params["calc_core_sample_indices"] = False   # core-sample indices are not supported

    def setEps(self: P, value: float) -> P:
        return self._set_params(eps=value)

    def getEps(self) -> float:
        return self.getOrDefault("eps")

    def setMinSamples(self: P, value: int) -> P:
        return self._set_params(min_samples=value)

    def getMinSamples(self) -> int:
        return self.getOrDefault("min_samples")

    def setMetric(self: P, value: str) -> P:
        return self._set_params(metric=value)

    def getMetric(self) -> str:
        return self.getOrDefault("metric")

    def setAlgorithm(self: P, value: str) -> P:
        return self._set_params(algorithm=value)

    def getAlgorithm(self) -> str:
        return self.getOrDefault("algorithm")

    def setMaxMbytesPerBatch(self: P, value: Optional[int]) -> P:
        return self._set_params(max_mbytes_per_batch=value)

    def getMaxMbytesPerBatch(self) -> Optional[int]:
        return self.getOrDefault("max_mbytes_per_batch")

    def _fit(self, dataset: Any) -> "DBSCANModel":
        if self.getMetric() == "precomputed":
            raise ValueError("Spark Rapids ML does not support the 'precomputed' mode from sklearn and cuML, please "
                             "use those libraries instead")
        _validate_dbscan_params(self)
        model = DBSCANModel(n_cols=0, dtype="")
        model._num_workers = self._num_workers
        model._float32_inputs = self._float32_inputs
        self._copyValues(model)
        self._copy_cuml_params(model)
        return model

    def _create_pyspark_model(self, result: Row) -> Any:
        raise NotImplementedError("DBSCAN does not support model creation from Row")

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None) -> Any:
        raise NotImplementedError("DBSCAN does not fit and generate model")

    def _out_schema(self) -> Any:
        raise NotImplementedError("DBSCAN does not output for fit and generate model")


def _validate_dbscan_params(p: Any) -> None:
    metric, algorithm = p.getOrDefault("metric"), p.getOrDefault("algorithm")
    if metric not in ("euclidean", "cosine"):
        raise ValueError(f"metric {metric!r} is not supported: use 'euclidean' or 'cosine'")
    if algorithm not in ("brute", "rbc"):
        raise ValueError(f"algorithm {algorithm!r} is not supported: use 'brute' or 'rbc'")


class DBSCANModel(DBSCANClass, _CumlModelWithPredictionCol, _CumlCaller, _DBSCANCumlParams):
    """reference: clustering.py:937-1186.  transform(frame) clusters the frame's rows (one barrier task per GPU, each
    rank's labels for its own rows) and appends the int32 predictionCol in the frame's row order, matching rows by idCol
    or, when the frame has no such column, by a monotonically increasing `unique_id`."""

    def __init__(self, n_cols: int, dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype)
        self._setDefault(idCol=alias.row_number)

    def _out_schema(self, input_schema: Any = None) -> Any:
        return f"{self._get_prediction_name()} int, {alias.row_number} long"

    def _get_prediction_name(self) -> str:
        return self.getOrDefault("predictionCol")

    def _require_nccl_ucx(self) -> Tuple[bool, bool]:
        return (True, False)

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None) -> Any:
        raise NotImplementedError("DBSCAN does not have a separate transform UDF")

    def _pre_process_data(self, dataset: Any) -> Tuple[Any, Optional[List[str]], int, str]:
        """The feature columns as for every estimator, plus the row id as alias.row_number (int64)."""
        df, multi_col_names, dimension, ftype = _CumlCaller._pre_process_data(self, dataset)
        id_col = self.getIdCol()
        df = df.with_appended_column(alias.row_number,
                                     [[b.column(id_col).cast(pa.int64()) for b in p] for p in dataset._parts])
        return df, multi_col_names, dimension, ftype

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        pred_name = self._get_prediction_name()

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for DBSCANMG(handle).fit_predict (clustering.py:1049-1098); every rank returns its own rows
            ctx = params[param_alias.handle]
            X, _, row_number = dfs[0]
            init = params[param_alias.cuml_init]
            labels, _, _ = ctx.dbscan_fit(X, float(init["eps"]), int(init["min_samples"]), init["metric"])
            return {pred_name: labels.cpu().numpy(), alias.row_number: row_number}

        return _cuml_fit

    def _transform(self, dataset: Any) -> Any:
        _no_pyspark(dataset)
        _validate_dbscan_params(self)
        id_col = self.getIdCol()
        with_id = dataset if id_col in dataset.columns else dataset.with_monotonically_increasing_id(id_col)
        input_col, input_cols = self._get_input_columns()
        cols = [id_col] + ([input_col] if input_col is not None else list(input_cols))
        res = self._call_cuml_fit_func(with_id.select(cols).repartition(self.num_workers), partially_collect=False)
        table = res._table()
        got_ids = np.asarray(table.column(alias.row_number).to_numpy(), dtype=np.int64)
        got = np.asarray(table.column(self._get_prediction_name()).to_numpy(), dtype=np.int32)
        order = np.argsort(got_ids, kind="stable")
        got_ids, got = got_ids[order], got[order]
        if np.any(got_ids[1:] == got_ids[:-1]):
            raise ValueError(f"idCol '{id_col}' must identify each row: it has repeated values")
        out_parts = []
        for p in with_id._parts:
            arrs = []
            for b in p:
                ids = np.asarray(b.column(id_col).cast(pa.int64()).to_numpy(), dtype=np.int64)
                arrs.append(pa.array(got[np.searchsorted(got_ids, ids)], type=pa.int32()))
            out_parts.append(arrs)
        return dataset.with_appended_column(self._get_prediction_name(), out_parts)


# ---- GaussianMixture (pyspark.ml.clustering.GaussianMixture; the reference has no Gaussian mixture) ----
class GaussianMixtureClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        # None = unsupported, "" = accepted and ignored
        return {"k": "n_components", "maxIter": "max_iter", "tol": "tol", "seed": "random_state",
                "aggregationDepth": "", "weightCol": None}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_components": 2, "max_iter": 100, "tol": 0.01, "random_state": None, "verbose": False}

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.clustering.GaussianMixture when pyspark is installed


class _GaussianMixtureCumlParams(_CumlParams, HasFeaturesCol, HasFeaturesCols, HasPredictionCol):
    """Shared Spark Params of GaussianMixture and GaussianMixtureModel (Spark's defaults: k=2, maxIter=100, tol=0.01,
    probabilityCol='probability', aggregationDepth=2)."""

    k = Param("parent", "k", "Number of independent Gaussians in the mixture model. Must be > 1.", TypeConverters.toInt)
    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    tol = Param("parent", "tol", "the convergence tolerance for iterative algorithms (>= 0).", TypeConverters.toFloat)
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    probabilityCol = Param("parent", "probabilityCol", "Column name for predicted class conditional probabilities.",
                           TypeConverters.toString)
    aggregationDepth = Param("parent", "aggregationDepth", "suggested depth for treeAggregate (>= 2).",
                             TypeConverters.toInt)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(k=2, maxIter=100, tol=0.01, probabilityCol="probability", aggregationDepth=2)
        # the KMeans rule: a 32-bit signed seed from the class name
        self._setDefault(seed=hash(type(self).__name__) & 0x07FFFFFFF)

    def getK(self) -> int:
        return self.getOrDefault(self.k)

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getTol(self) -> float:
        return self.getOrDefault(self.tol)

    def getSeed(self) -> int:
        return self.getOrDefault(self.seed)

    def getProbabilityCol(self) -> str:
        return self.getOrDefault(self.probabilityCol)

    def getAggregationDepth(self) -> int:
        return self.getOrDefault(self.aggregationDepth)

    def getFeaturesCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.featuresCols):
            return self.getFeaturesCols()
        if self.isDefined(self.featuresCol):
            return self.getOrDefault("featuresCol")
        raise RuntimeError("featuresCol is not set")

    def setFeaturesCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(featuresCol=value)
        else:
            self._set_params(featuresCols=value)
        return self

    def setFeaturesCols(self: P, value: List[str]) -> P:
        return self._set_params(featuresCols=value)

    def setPredictionCol(self: P, value: str) -> P:
        return self._set_params(predictionCol=value)

    def setProbabilityCol(self: P, value: str) -> P:
        return self._set_params(probabilityCol=value)


class GaussianMixture(GaussianMixtureClass, _CumlEstimator, _GaussianMixtureCumlParams):
    """Gaussian mixture models (full covariances) by EM on H100, Spark's pyspark.ml.clustering.GaussianMixture.  One
    barrier task per GPU holds its partition on the device; each iteration is one E pass (the whitened quadratic forms
    of every row and component, on wgmma 3xTF32 where the shape allows), a moments pass and a weighted Gram pass in
    fp64, one NCCL allreduce and an fp64 update with one eigendecomposition per component on the host.  Parameters:
    k (2), maxIter (100), tol (0.01, on the total log-likelihood), seed, featuresCol (str for an array column, list of
    str for scalar columns), predictionCol, probabilityCol ("probability"), aggregationDepth (accepted, unused),
    num_workers, verbose.  weightCol is not supported.

    The start is Spark's rule (weights 1/k, the mean and diagonal variance of 5 sampled rows per component) with the
    rows drawn by the library's own seeded generator, so it differs from Spark's for the same seed.

    >>> from spark_rapids_ml_b200.clustering import GaussianMixture
    >>> model = GaussianMixture(k=2, seed=1).fit(df)
    >>> model.weights, model.summary.logLikelihood
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", predictionCol: str = "prediction",
                 k: int = 2, probabilityCol: str = "probability", tol: float = 0.01, maxIter: int = 100,
                 seed: Optional[int] = None, aggregationDepth: int = 2, weightCol: Optional[str] = None,
                 num_workers: Optional[int] = None, verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        for name in ("seed", "num_workers", "weightCol"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        if "weightCol" in self._input_kwargs:
            raise ValueError("'weightCol' is not supported by GaussianMixture on the GPU.")
        self._set_params(**self._input_kwargs)

    def setK(self, value: int) -> "GaussianMixture":
        return self._set_params(k=value)

    def setMaxIter(self, value: int) -> "GaussianMixture":
        return self._set_params(maxIter=value)

    def setTol(self, value: float) -> "GaussianMixture":
        return self._set_params(tol=value)

    def setSeed(self, value: int) -> "GaussianMixture":
        return self._set_params(seed=value)

    def setAggregationDepth(self, value: int) -> "GaussianMixture":
        return self._set_params(aggregationDepth=value)

    def setWeightCol(self, value: str) -> "GaussianMixture":
        raise ValueError("'weightCol' is not supported by GaussianMixture on the GPU.")

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        k, max_iter, tol = self.getK(), self.getMaxIter(), self.getTol()
        if isinstance(k, bool) or not isinstance(k, int) or k < 2:
            raise ValueError(f"k given invalid value {k} (must be > 1)")
        if max_iter < 0:
            raise ValueError(f"maxIter given invalid value {max_iter} (must be >= 0)")
        if not tol >= 0:
            raise ValueError(f"tol given invalid value {tol} (must be >= 0)")

    def _fit_array_order(self) -> str:
        return "C"

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        cls = self.__class__

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            ctx = params[param_alias.handle]
            init = params[param_alias.cuml_init]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            seed = init.get("random_state")
            out = ctx.gmm_fit(dfs[0][0], int(init["n_components"]), max_iter=int(init["max_iter"]),
                              tol=float(init["tol"]), seed=int(seed) if seed is not None else 0)
            get_logger(cls).info(f"iterations: {out['n_iter']}, log-likelihood: {out['log_likelihood']}")
            return {"weights_": [out["weights"].tolist()], "means_": [out["means"].tolist()],
                    "covs_": [out["covs"].tolist()], "cluster_sizes_": [out["cluster_sizes"].tolist()],
                    "log_likelihood_": [out["log_likelihood"]], "num_iters": [out["n_iter"]],
                    "n_cols": [params[param_alias.num_cols]], "dtype": ["float32"]}

        return _cuml_fit

    def _out_schema(self) -> Any:
        return ("weights_ array<double>, means_ array<array<double>>, covs_ array<array<array<double>>>, "
                "cluster_sizes_ array<long>, log_likelihood_ double, num_iters int, n_cols int, dtype string")

    def _create_pyspark_model(self, result: Row) -> "GaussianMixtureModel":
        r = result.asDict()
        return GaussianMixtureModel(
            weights_=[float(v) for v in r["weights_"]], means_=[[float(v) for v in m] for m in r["means_"]],
            covs_=[[[float(v) for v in row] for row in c] for c in r["covs_"]],
            cluster_sizes_=[int(v) for v in r["cluster_sizes_"]], log_likelihood_=float(r["log_likelihood_"]),
            num_iters=int(r["num_iters"]), n_cols=int(r["n_cols"]), dtype=str(r["dtype"]))


class GaussianMixtureSummary:
    """The training summary Spark's GaussianMixtureModel.summary holds: k, numIter, logLikelihood, clusterSizes."""

    def __init__(self, k: int, num_iter: int, log_likelihood: float, cluster_sizes: List[int]) -> None:
        self.k = k
        self.numIter = num_iter
        self.logLikelihood = log_likelihood
        self.clusterSizes = cluster_sizes


class GaussianMixtureModel(GaussianMixtureClass, _CumlModelWithPredictionCol, _GaussianMixtureCumlParams):
    """transform() appends predictionCol (int, the most probable component, the lower one on a tie) and probabilityCol
    (a double vector of the k component probabilities)."""

    def __init__(self, weights_: List[float], means_: List[List[float]], covs_: List[List[List[float]]],
                 cluster_sizes_: List[int], log_likelihood_: float, num_iters: int, n_cols: int, dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype, weights_=weights_, means_=means_, covs_=covs_,
                         cluster_sizes_=cluster_sizes_, log_likelihood_=log_likelihood_, num_iters=num_iters)
        self.weights_ = weights_
        self.means_ = means_
        self.covs_ = covs_
        self.cluster_sizes_ = cluster_sizes_
        self.log_likelihood_ = log_likelihood_
        self.num_iters = num_iters
        self._set_params(k=len(weights_))

    @property
    def weights(self) -> List[float]:
        return list(self.weights_)

    @property
    def gaussiansDF(self) -> Any:
        """A local frame with one row per component: mean (a double vector) and cov (a [d, d] double matrix)."""
        from .sparkshim import get_session

        table = pa.table({
            "mean": pa.array([list(m) for m in self.means_], type=pa.list_(pa.float64())),
            "cov": pa.array([[list(r) for r in c] for c in self.covs_], type=pa.list_(pa.list_(pa.float64()))),
        })
        return get_session().createDataFrame(table)

    @property
    def hasSummary(self) -> bool:
        return True

    @property
    def summary(self) -> GaussianMixtureSummary:
        return GaussianMixtureSummary(len(self.weights_), int(self.num_iters), float(self.log_likelihood_),
                                      list(self.cluster_sizes_))

    def predict(self, value: Any) -> int:
        raise NotImplementedError("GaussianMixtureModel.predict() of a single vector is not supported; use transform()")

    def predictProbability(self, value: Any) -> Any:
        raise NotImplementedError("GaussianMixtureModel.predictProbability() of a single vector is not supported; use "
                                  "transform()")

    def cpu(self) -> Any:
        raise NotImplementedError("GaussianMixtureModel.cpu() builds a JVM pyspark.ml model; no JVM/pyspark in this "
                                  "build")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "int"

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        return [(self.getOrDefault("predictionCol"), "int"), (self.getProbabilityCol(), "array<double>")]

    def _transform_array_order(self) -> str:
        return "C"

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        w = np.asarray(self.weights_, dtype=np.float64)
        mu = np.asarray(self.means_, dtype=np.float64)
        cov = np.asarray(self.covs_, dtype=np.float64)

        def _predict(m: Any, X: Any) -> Tuple[Any, Any]:
            prob, labels = m.ctx.gmm_predict(X, w, mu, cov)
            return labels, prob

        k = len(self.weights_)
        return _DeviceModel, self._grouped_transform(_predict, 4 * int(self.n_cols) + 8 * k + 4), None


# ---- BisectingKMeans (pyspark.ml.clustering.BisectingKMeans; the reference has no bisecting k-means) ----
class BisectingKMeansClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        # None = unsupported, "" = accepted and ignored (distanceMeasure: only "euclidean", checked by the params)
        return {"k": "n_clusters", "maxIter": "max_iter", "seed": "random_state",
                "minDivisibleClusterSize": "min_divisible_cluster_size", "distanceMeasure": "", "weightCol": None}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_clusters": 4, "max_iter": 20, "random_state": None, "min_divisible_cluster_size": 1.0,
                "verbose": False}

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.clustering.BisectingKMeans when pyspark is installed


def _check_bkm_distance(value: Any) -> None:
    if value != "euclidean":
        raise ValueError(f"distanceMeasure {value!r} is not supported by BisectingKMeans on the GPU: use 'euclidean'")


class _BisectingKMeansCumlParams(_CumlParams, HasFeaturesCol, HasFeaturesCols, HasPredictionCol):
    """Shared Spark Params of BisectingKMeans and BisectingKMeansModel (Spark's defaults: k=4, maxIter=20,
    minDivisibleClusterSize=1.0, distanceMeasure='euclidean')."""

    k = Param("parent", "k", "The desired number of leaf clusters. Must be > 1.", TypeConverters.toInt)
    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    minDivisibleClusterSize = Param("parent", "minDivisibleClusterSize",
                                    "The minimum number of points (if >= 1.0) or the minimum proportion of points "
                                    "(if < 1.0) of a divisible cluster.", TypeConverters.toFloat)
    distanceMeasure = Param("parent", "distanceMeasure", "the distance measure. Supported options: 'euclidean'.",
                            TypeConverters.toString)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(k=4, maxIter=20, minDivisibleClusterSize=1.0, distanceMeasure="euclidean")
        # the KMeans rule: a 32-bit signed seed from the class name
        self._setDefault(seed=hash(type(self).__name__) & 0x07FFFFFFF)

    def getK(self) -> int:
        return self.getOrDefault(self.k)

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getSeed(self) -> int:
        return self.getOrDefault(self.seed)

    def getMinDivisibleClusterSize(self) -> float:
        return self.getOrDefault(self.minDivisibleClusterSize)

    def getDistanceMeasure(self) -> str:
        return self.getOrDefault(self.distanceMeasure)

    def getFeaturesCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.featuresCols):
            return self.getFeaturesCols()
        if self.isDefined(self.featuresCol):
            return self.getOrDefault("featuresCol")
        raise RuntimeError("featuresCol is not set")

    def setFeaturesCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(featuresCol=value)
        else:
            self._set_params(featuresCols=value)
        return self

    def setFeaturesCols(self: P, value: List[str]) -> P:
        return self._set_params(featuresCols=value)

    def setPredictionCol(self: P, value: str) -> P:
        return self._set_params(predictionCol=value)


class BisectingKMeans(BisectingKMeansClass, _CumlEstimator, _BisectingKMeansCumlParams):
    """Bisecting k-means on H100, Spark's pyspark.ml.clustering.BisectingKMeans (euclidean).  One barrier task per GPU
    holds its partition on the device.  Level by level, the largest divisible clusters are split in two: each
    iteration is one device pass over the rows of the clusters being split (every row against its cluster's two
    children, fp64 sums folded in a fixed order), one NCCL allreduce and the new children; the host decides the next
    level once per level.  Parameters: k (4), maxIter (20, iterations per level), seed, minDivisibleClusterSize (1.0:
    a count when >= 1, else a fraction of the rows), distanceMeasure ("euclidean" only), featuresCol (str for an array
    column, list of str for scalar columns), predictionCol, num_workers, verbose.  weightCol is not supported.

    A split starts from the library's own seeded generator, so the tree differs from Spark's for the same seed; ties
    between equally large divisible clusters go to the lower node index.

    >>> from spark_rapids_ml_b200.clustering import BisectingKMeans
    >>> model = BisectingKMeans(k=8, seed=1).fit(df)
    >>> model.clusterCenters(), model.summary.trainingCost
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", predictionCol: str = "prediction",
                 maxIter: int = 20, seed: Optional[int] = None, k: int = 4, minDivisibleClusterSize: float = 1.0,
                 distanceMeasure: str = "euclidean", weightCol: Optional[str] = None,
                 num_workers: Optional[int] = None, verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        for name in ("seed", "num_workers", "weightCol"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        if "weightCol" in self._input_kwargs:
            raise ValueError("'weightCol' is not supported by BisectingKMeans on the GPU.")
        if "distanceMeasure" in self._input_kwargs:
            _check_bkm_distance(self._input_kwargs["distanceMeasure"])
        self._set_params(**self._input_kwargs)

    def setK(self, value: int) -> "BisectingKMeans":
        return self._set_params(k=value)

    def setMaxIter(self, value: int) -> "BisectingKMeans":
        return self._set_params(maxIter=value)

    def setSeed(self, value: int) -> "BisectingKMeans":
        return self._set_params(seed=value)

    def setMinDivisibleClusterSize(self, value: float) -> "BisectingKMeans":
        return self._set_params(minDivisibleClusterSize=value)

    def setDistanceMeasure(self, value: str) -> "BisectingKMeans":
        _check_bkm_distance(value)
        return self._set_params(distanceMeasure=value)

    def setWeightCol(self, value: str) -> "BisectingKMeans":
        raise ValueError("'weightCol' is not supported by BisectingKMeans on the GPU.")

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        k, max_iter, mdcs = self.getK(), self.getMaxIter(), self.getMinDivisibleClusterSize()
        if isinstance(k, bool) or not isinstance(k, int) or k < 2:
            raise ValueError(f"k given invalid value {k} (must be > 1)")
        if max_iter < 1:
            raise ValueError(f"maxIter given invalid value {max_iter} (must be >= 1)")
        if not mdcs > 0:
            raise ValueError(f"minDivisibleClusterSize given invalid value {mdcs} (must be > 0)")
        _check_bkm_distance(self.getDistanceMeasure())

    def _fit_array_order(self) -> str:
        return "C"

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        cls = self.__class__

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            ctx = params[param_alias.handle]
            init = params[param_alias.cuml_init]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            seed = init.get("random_state")
            out = ctx.bkm_fit(dfs[0][0], int(init["n_clusters"]), max_iter=int(init["max_iter"]),
                              min_divisible=float(init["min_divisible_cluster_size"]),
                              seed=int(seed) if seed is not None else 0)
            get_logger(cls).info(f"levels: {out['n_levels']}, nodes: {len(out['node_index'])}, "
                                 f"training cost: {out['training_cost']}")
            return {"node_index_": [out["node_index"].tolist()], "node_centers_": [out["centers"].tolist()],
                    "node_sizes_": [out["sizes"].tolist()], "node_costs_": [out["costs"].tolist()],
                    "cluster_sizes_": [out["cluster_sizes"].tolist()], "training_cost_": [out["training_cost"]],
                    "num_iters": [int(init["max_iter"])], "n_cols": [params[param_alias.num_cols]],
                    "dtype": ["float32"]}

        return _cuml_fit

    def _out_schema(self) -> Any:
        return ("node_index_ array<long>, node_centers_ array<array<double>>, node_sizes_ array<long>, "
                "node_costs_ array<double>, cluster_sizes_ array<long>, training_cost_ double, num_iters int, "
                "n_cols int, dtype string")

    def _create_pyspark_model(self, result: Row) -> "BisectingKMeansModel":
        r = result.asDict()
        return BisectingKMeansModel(
            node_index_=[int(v) for v in r["node_index_"]],
            node_centers_=[[float(v) for v in c] for c in r["node_centers_"]],
            node_sizes_=[int(v) for v in r["node_sizes_"]], node_costs_=[float(v) for v in r["node_costs_"]],
            cluster_sizes_=[int(v) for v in r["cluster_sizes_"]], training_cost_=float(r["training_cost_"]),
            num_iters=int(r["num_iters"]), n_cols=int(r["n_cols"]), dtype=str(r["dtype"]))


class BisectingKMeansSummary:
    """The training summary Spark's BisectingKMeansModel.summary holds: k (the leaf count), numIter, clusterSizes and
    trainingCost."""

    def __init__(self, k: int, num_iter: int, cluster_sizes: List[int], training_cost: float) -> None:
        self.k = k
        self.numIter = num_iter
        self.clusterSizes = cluster_sizes
        self.trainingCost = training_cost


class BisectingKMeansModel(BisectingKMeansClass, _CumlModelWithPredictionCol, _BisectingKMeansCumlParams):
    """The cluster tree: node indices (root 1, children 2i and 2i + 1), centres, sizes and costs in depth-first order.
    transform() appends predictionCol (int): the leaf reached by descending from the root to the nearer child, leaves
    numbered in depth-first order as clusterCenters() lists them."""

    def __init__(self, node_index_: List[int], node_centers_: List[List[float]], node_sizes_: List[int],
                 node_costs_: List[float], cluster_sizes_: List[int], training_cost_: float, num_iters: int,
                 n_cols: int, dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype, node_index_=node_index_, node_centers_=node_centers_,
                         node_sizes_=node_sizes_, node_costs_=node_costs_, cluster_sizes_=cluster_sizes_,
                         training_cost_=training_cost_, num_iters=num_iters)
        self.node_index_ = node_index_
        self.node_centers_ = node_centers_
        self.node_sizes_ = node_sizes_
        self.node_costs_ = node_costs_
        self.cluster_sizes_ = cluster_sizes_
        self.training_cost_ = training_cost_
        self.num_iters = num_iters
        self._set_params(k=len(self._leaves()))

    def _leaves(self) -> List[int]:
        ids = set(self.node_index_)
        return [j for j, i in enumerate(self.node_index_) if 2 * i not in ids and 2 * i + 1 not in ids]

    def clusterCenters(self) -> List[np.ndarray]:
        return [np.asarray(self.node_centers_[j], dtype=np.float64) for j in self._leaves()]

    @property
    def hasSummary(self) -> bool:
        return True

    @property
    def summary(self) -> BisectingKMeansSummary:
        return BisectingKMeansSummary(len(self._leaves()), int(self.num_iters), list(self.cluster_sizes_),
                                      float(self.training_cost_))

    def computeCost(self, dataset: Any) -> float:
        """The sum of squared distances of the rows of `dataset` to the centres of the leaves they are predicted to."""
        from .core import _CumlCommon, _GroupedTransform, _iter_transform, _select_features
        from .sparkshim import BarrierTaskContext
        from .sparkshim.sql import _batches_to_pdf_iter

        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):
                raise NotImplementedError("BisectingKMeansModel.computeCost of a pyspark DataFrame is not supported "
                                          "yet; use a local frame")
        idx = np.asarray(self.node_index_, dtype=np.int64)
        cen = np.asarray(self.node_centers_, dtype=np.float64)
        transform = _GroupedTransform(lambda m, X: (m.ctx.bkm_predict(X, idx, cen, with_cost=True)[1],),
                                      int(self.n_cols), 4 * int(self.n_cols) + 12, ["double"])
        input_col, input_cols = self._get_input_columns()
        total, model = 0.0, None
        for pid, part in enumerate(dataset._parts):
            if part and model is None:
                model = _DeviceModel(_CumlCommon._set_gpu_device(BarrierTaskContext(pid, len(dataset._parts)), True,
                                                                 True))
            frames = _batches_to_pdf_iter(_select_features(part, input_col, input_cols), dataset.arrow_backed_pandas)
            for (c,) in _iter_transform(transform, model, frames):
                total += float(np.sum(c, dtype=np.float64))
        if model is not None:
            model.close()
        return total

    def predict(self, value: Any) -> int:
        raise NotImplementedError("BisectingKMeansModel.predict() of a single vector is not supported; use transform()")

    def cpu(self) -> Any:
        raise NotImplementedError("BisectingKMeansModel.cpu() builds a JVM pyspark.ml model; no JVM/pyspark in this "
                                  "build")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "int"

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        return [(self.getOrDefault("predictionCol"), "int")]

    def _transform_array_order(self) -> str:
        return "C"

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        idx = np.asarray(self.node_index_, dtype=np.int64)
        cen = np.asarray(self.node_centers_, dtype=np.float64)

        def _predict(m: Any, X: Any) -> Tuple[Any]:
            return (m.ctx.bkm_predict(X, idx, cen)[0],)

        return _DeviceModel, self._grouped_transform(_predict, 4 * int(self.n_cols) + 4), None
