"""KMeans / KMeansModel — the reference's PySpark-ML Estimator/Model surface for the distributed KMeans.fit()
path (python/src/spark_rapids_ml/clustering.py:84-604), with the cuML calls replaced by libb2kmeans
(hand-written sm_90a CUDA behind include/b2kmeans.h).

Same names, argument meaning and error behaviour as the reference:
  KMeansClass._param_mapping / _param_value_mapping / _get_cuml_params_default      clustering.py:84-141
  _KMeansCumlParams (featuresCol/featuresCols handling, seed default)                clustering.py:144-186
  KMeans (keyword-only ctor, setters, _get_cuml_fit_func, _out_schema,
          _create_pyspark_model, _merge_model_chunks)                                clustering.py:189-502
  KMeansModel (clusterCenters, hasSummary, predict, _get_cuml_transform_func)        clustering.py:505-604

Differences that are deliberate: no CPU fallback (cpu() / single-vector predict need a JVM and raise), and the
fit function receives a DEVICE matrix from the worker scaffold instead of host arrays to concatenate.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pandas as pd

from .core import (FitInputType, _append_transform_features, _CumlEstimator, _CumlModelWithPredictionCol,
                   _transform_context, param_alias)
from .params import HasFeaturesCols, P, _CumlClass, _CumlParams, _KMeansParams
from .sparkshim import Row, keyword_only
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


class KMeans(KMeansClass, _CumlEstimator, _KMeansCumlParams):
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

    def _fit_array_order(self) -> str:
        return "C"

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        cls = self.__class__

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
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

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        cluster_centers_ = self.cluster_centers_
        n_cols = self.n_cols

        class _DeviceKMeans:  # the injected-centers predictor (clustering.py:582-596)
            def __init__(self, gpu: int) -> None:
                import torch

                self.ctx = _transform_context(gpu)
                self.C = torch.tensor(cluster_centers_, dtype=torch.float32, device=self.ctx.device)

            def close(self) -> None:   # the context (pinned staging, scratch, copy threads) stays with the process
                self.C = None

        def _construct_kmeans(gpu: int = 0) -> Any:
            return _DeviceKMeans(gpu)

        def _transform_many(kmeans: Any, dfs: List[Union[pd.DataFrame, np.ndarray]]) -> List[pd.Series]:
            """Several input batches in ONE device pass: every batch is ingested into the same device matrix, one
            b2k_kmeans_assign labels all rows, one read-back, one Series per input batch (same order, same lengths).
            The per-batch host overhead (allocation, launches, a synchronising read-back) is what a 10 000-row Arrow batch
            costs most; core._iter_transform groups batches up to ~1 M rows."""
            from .utils import DeviceRowAppender

            sizes = [len(df) for df in dfs]
            total = sum(sizes)
            if total == 0:
                return [pd.Series([], dtype="int32") for _ in dfs]
            app = DeviceRowAppender(kmeans.ctx, n_cols, first_capacity=total)
            for df, n_b in zip(dfs, sizes):
                if n_b:
                    _append_transform_features(app, df, n_cols)
            X = app.finish()
            labels, _ = kmeans.ctx.kmeans_assign(X, kmeans.C)
            host = labels.cpu().numpy()
            out, o = [], 0
            for n_b in sizes:
                out.append(pd.Series(host[o:o + n_b]))
                o += n_b
            return out

        def _transform_internal(kmeans: Any, df: Union[pd.DataFrame, np.ndarray]) -> pd.Series:
            return _transform_many(kmeans, [df])[0]

        _transform_internal.many = _transform_many  # type: ignore[attr-defined]
        _transform_internal.row_bytes = 4 * int(n_cols or 1)  # type: ignore[attr-defined]
        return _construct_kmeans, _transform_internal, None
