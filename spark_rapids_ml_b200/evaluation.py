"""MulticlassClassificationEvaluator, RegressionEvaluator and BinaryClassificationEvaluator: pyspark.ml.evaluation's
when pyspark is present, else the local stand-ins of sparkshim.evaluation (Spark's params, defaults and
isLargerBetter(); evaluate() of a local frame in fp64 on the host).  All three feed the single-pass multi-model
evaluation of CrossValidator (tuning.py).

ClusteringEvaluator: Spark's silhouette of a clustering (KMeansModel or DBSCANModel output), computed on the device by
b2k_silhouette (include/b2kmeans.h) in one barrier task per GPU."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa

from .core import _CumlCaller, alias, param_alias
from .params import HasFeaturesCol, HasFeaturesCols
from .sparkshim import HAVE_PYSPARK

if HAVE_PYSPARK:
    from pyspark.ml.evaluation import (  # noqa: F401
        BinaryClassificationEvaluator,
        ClusteringEvaluator as _ClusteringEvaluatorBase,
        MulticlassClassificationEvaluator,
        RegressionEvaluator,
    )
else:
    from .sparkshim.evaluation import (  # noqa: F401
        BinaryClassificationEvaluator,
        ClusteringEvaluator as _ClusteringEvaluatorBase,
        MulticlassClassificationEvaluator,
        RegressionEvaluator,
    )

__all__ = ["MulticlassClassificationEvaluator", "RegressionEvaluator", "BinaryClassificationEvaluator",
           "ClusteringEvaluator"]


def _cluster_ids(col: Any, name: str) -> np.ndarray:
    """A prediction column (Arrow) as int64 cluster ids: integers, or floats holding integers in int64 range."""
    if col.null_count:
        raise ValueError(f"predictionCol '{name}' holds null values: cluster ids must be integers")
    a = np.asarray(col.to_numpy(zero_copy_only=False))
    if a.dtype.kind in "iub":
        return a.astype(np.int64)
    if a.dtype.kind != "f":
        raise ValueError(f"predictionCol '{name}' has type {a.dtype}: cluster ids must be integers")
    v = a.astype(np.float64)
    bad = ~np.isfinite(v) | (v != np.floor(v)) | (v < -2.0**63) | (v >= 2.0**63)
    if np.any(bad):
        raise ValueError(f"predictionCol '{name}' holds {float(v[bad][0])!r}: cluster ids must be integers in int64 range")
    return v.astype(np.int64)


class _SilhouetteCaller(_CumlCaller, HasFeaturesCol, HasFeaturesCols):
    """One barrier task per GPU over the frame's features and cluster ids, with the worker count and NCCL set-up of a
    fit; every rank calls Context.silhouette on its rows and rank 0's value is returned."""

    def __init__(self, features: Any, prediction: str, distance: str) -> None:
        super().__init__()
        self._set_params(featuresCol=features)
        self._prediction, self._distance = prediction, distance

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {}

    def _out_schema(self) -> Any:
        return "silhouette double"

    def _pre_process_data(self, dataset: Any) -> Tuple[Any, Optional[List[str]], int, str]:
        """The features as every estimator reads them, plus the cluster ids as alias.row_number (int64)."""
        if self._prediction not in dataset.columns:
            raise ValueError(f"prediction column '{self._prediction}' not found in {dataset.columns}")
        df, multi_col_names, dimension, ftype = _CumlCaller._pre_process_data(self, dataset)
        ids = [[pa.array(_cluster_ids(b.column(self._prediction), self._prediction), type=pa.int64()) for b in p]
               for p in dataset._parts]
        return df.with_appended_column(alias.row_number, ids), multi_col_names, dimension, ftype

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None) -> Any:
        distance = self._distance

        def _cuml_fit(dfs: Any, params: Dict[str, Any]) -> Dict[str, Any]:
            import torch

            X, _, ids = dfs[0]
            v = params[param_alias.handle].silhouette(X, torch.from_numpy(ids).to(X.device), distance)
            return {"silhouette": [v]}

        return _cuml_fit


class _SilhouetteMultiCaller(_SilhouetteCaller):
    """_SilhouetteCaller's barrier task for KMeansModel._transformEvaluate: the rows are labelled on the device with
    each centre set as KMeansModel.transform labels them (Context.kmeans_assign), then one Context.silhouette_multi
    call scores every set; rank 0's values are returned."""

    def __init__(self, features: Any, center_sets: List[Any], distance: str) -> None:
        super().__init__(features, "", distance)
        self._center_sets = [np.asarray(c, dtype=np.float32) for c in center_sets]

    def _out_schema(self) -> Any:
        return "silhouette array<double>"

    def _pre_process_data(self, dataset: Any) -> Tuple[Any, Optional[List[str]], int, str]:
        return _CumlCaller._pre_process_data(self, dataset)

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None) -> Any:
        distance, center_sets = self._distance, self._center_sets

        def _cuml_fit(dfs: Any, params: Dict[str, Any]) -> Dict[str, Any]:
            import torch

            ctx = params[param_alias.handle]
            X = dfs[0][0]
            ids = [ctx.kmeans_assign(X, torch.from_numpy(C).to(X.device))[0].to(torch.int64) for C in center_sets]
            return {"silhouette": [ctx.silhouette_multi(X, ids, distance)]}

        return _cuml_fit


class ClusteringEvaluator(_ClusteringEvaluatorBase):
    """pyspark.ml.evaluation.ClusteringEvaluator on the device: metricName "silhouette", distanceMeasure
    "squaredEuclidean" (default) or "cosine", featuresCol (an array column or a list of numeric columns, as
    KMeansModel.transform reads them), predictionCol.  evaluate(frame) runs one barrier task per GPU and returns Spark's
    silhouette (= scikit-learn's silhouette_score with metric "sqeuclidean" or "cosine").

    Deliberate differences from Spark:
      * D(i, c) is formed as ||x - mu_c||^2 + Psi_c in a frame shifted by the global mean; Spark's
        ||x||^2 + sum ||y||^2 / N - 2 x.sum y / N is equal in exact arithmetic but cancels on offset data.
      * features are read as float32, as transform() reads them.
      * predictions must be integers in int64 range (-1, DBSCAN's noise, is a cluster like any other); a null, NaN or
        fractional value raises ValueError naming the column.  Spark keys clusters by any double.
      * under "cosine" a zero row is an error (Spark's normalisation makes it NaN); a NaN or infinite feature is an
        error; so is an empty frame.
      * weightCol raises NotImplementedError; evaluate() of a pyspark DataFrame raises NotImplementedError (there is
        no CPU fallback).
    The result is within the bound stated in include/b2kmeans.h of the exact value, and the same bits for the same
    input, worker count and devices."""

    def isLargerBetter(self) -> bool:
        return True

    def _evaluate(self, dataset: Any) -> float:
        if self.isSet("weightCol") and self.getOrDefault("weightCol"):
            raise NotImplementedError("weightCol is not supported by the device evaluation")
        if HAVE_PYSPARK:
            from . import spark_binding

            if spark_binding.is_spark_dataframe(dataset):
                raise NotImplementedError("ClusteringEvaluator.evaluate() of a pyspark DataFrame is not supported in "
                                          "this build; evaluate a local frame")
        metric, distance = self.getOrDefault("metricName"), self.getOrDefault("distanceMeasure")
        if metric != "silhouette":
            raise ValueError(f"{self.uid} parameter metricName given invalid value {metric}.")
        if distance not in ("squaredEuclidean", "cosine"):
            raise ValueError(f"{self.uid} parameter distanceMeasure given invalid value {distance}.")
        if dataset.count() == 0:
            raise ValueError("ClusteringEvaluator: the frame has no rows")
        caller = _SilhouetteCaller(self.getOrDefault("featuresCol"), self.getOrDefault("predictionCol"), distance)
        res = caller._call_cuml_fit_func(dataset, partially_collect=True)
        rows = res if isinstance(res, list) else res.collect()
        return float(rows[0]["silhouette"])
