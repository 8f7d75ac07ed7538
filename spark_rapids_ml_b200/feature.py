"""PCA / PCAModel — the reference's PySpark-ML Estimator/Model surface for distributed PCA
(python/src/spark_rapids_ml/feature.py:61-459), with the cuML calls replaced by libb2kmeans (hand-written sm_90a CUDA
behind include/b2kmeans.h).

  PCAClass._param_mapping / _get_cuml_params_default                         feature.py:61-77
  _PCACumlParams (inputCol / inputCols / outputCol handling)                feature.py:80-118
  PCA (keyword-only ctor, setK, _get_cuml_fit_func, _out_schema)             feature.py:121-260
  PCAModel (mean, pc, explainedVariance, _get_cuml_transform_func)           feature.py:263-459

Semantics (b2k_pca_fit, include/b2kmeans.h): mean_ = sum x / n in fp64 over all ranks; covariance of the centred data
/ (n - 1); components_ [k][d] by descending eigenvalue, each signed so that its largest-|value| element (lowest index on
a tie) is positive (the reference compares signs agnostically, so cuML's sign is not pinned); explained_variance_ratio_
= eigenvalue / trace; singular_values_ = sqrt(eigenvalue (n - 1)).  Zero total variance gives zero ratios and singular
values and the first k unit vectors as components.  transform() outputs X . components^T as array<float>, with no mean
subtracted, as Spark's PCAModel does.  svd_solver and whiten are accepted and ignored.

Differences that are deliberate: no CPU fallback (cpu() needs a JVM and raises), and the fit function receives a DEVICE
matrix from the worker scaffold instead of host arrays.
"""
from __future__ import annotations

import itertools
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import pandas as pd

from .core import (FitInputType, _append_transform_features, _CumlEstimator, _CumlModelWithColumns,
                   _transform_context, param_alias)
from .params import HasInputCols, P, _CumlClass, _CumlParams, _PCAParams
from .sparkshim import Row, keyword_only


class PCAClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {"k": "n_components"}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_components": None, "svd_solver": "auto", "verbose": False, "whiten": False}

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.feature.PCA when pyspark is installed


class _PCACumlParams(_CumlParams, _PCAParams, HasInputCols):
    """Shared Spark Params of PCA and PCAModel (reference: feature.py:80-118)."""

    def setInputCol(self: P, value: Union[str, List[str]]) -> P:
        if isinstance(value, str):
            self._set_params(inputCol=value)
        else:
            self._set_params(inputCols=value)
        return self

    def setInputCols(self: P, value: List[str]) -> P:
        return self._set_params(inputCols=value)

    def setOutputCol(self: P, value: str) -> P:
        return self._set_params(outputCol=value)

    def getInputCol(self) -> Union[str, List[str]]:  # type: ignore[override]
        if self.isDefined(self.inputCols):
            return self.getOrDefault(self.inputCols)
        if self.isDefined(self.inputCol):
            return self.getOrDefault(self.inputCol)
        raise RuntimeError("inputCol is not set")


class PCA(PCAClass, _CumlEstimator, _PCACumlParams):
    """PCA on H100: one barrier task per GPU; a column-sum pass and a Gram-matrix pass of the centred data (TMA +
    wgmma 3xTF32, fp64 partials) over the device-resident partition, two fp64 NCCL allreduces, then an fp64 eigen step
    on the host.  Parameters as in the reference (feature.py:121-195): k, inputCol (str for an array column, list of
    str for scalar columns), outputCol, num_workers, verbose.

    >>> from spark_rapids_ml_b200.feature import PCA
    >>> df = session.createDataFrame([([1.0, 1.0],), ([2.0, 2.0],), ([3.0, 3.0],)], ["features"])
    >>> model = PCA(k=1, inputCol="features").fit(df)
    >>> model.mean, model.explained_variance_ratio_
    ([2.0, 2.0], [1.0])
    """

    @keyword_only
    def __init__(self, *, k: Optional[int] = None, inputCol: Optional[Union[str, List[str]]] = None,
                 outputCol: Optional[str] = None, num_workers: Optional[int] = None,
                 verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        for name in ("k", "inputCol", "outputCol", "num_workers"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        self._set_params(**self._input_kwargs)

    def setK(self, value: int) -> "PCA":
        return self._set_params(k=value)

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        k = self.cuml_params.get("n_components")
        if k is None:
            raise ValueError("k is not set: PCA needs the number of principal components (setK)")
        if isinstance(k, bool) or not isinstance(k, int) or k < 1:
            raise ValueError(f"k given invalid value {k} (must be > 0)")

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for PCAMG(handle, **cuml_init).fit(...) and the attribute reads — feature.py:196-242
            ctx = params[param_alias.handle]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            out = ctx.pca_fit(dfs[0][0], int(params[param_alias.cuml_init]["n_components"]))
            return {
                "mean_": [out["mean_"].tolist()],
                "components_": [out["components_"].tolist()],
                "explained_variance_ratio_": [out["explained_variance_ratio_"].tolist()],
                "singular_values_": [out["singular_values_"].tolist()],
                "n_cols": params[param_alias.num_cols],
                "dtype": "float32",
            }

        return _cuml_fit

    def _out_schema(self) -> Any:
        # reference: feature.py:244-257
        return ("mean_ array<double>, components_ array<array<double>>, explained_variance_ratio_ array<double>, "
                "singular_values_ array<double>, n_cols int, dtype string")

    def _create_pyspark_model(self, result: Row) -> "PCAModel":
        r = result.asDict()
        return PCAModel(mean_=list(r["mean_"]), components_=[list(c) for c in r["components_"]],
                        explained_variance_ratio_=list(r["explained_variance_ratio_"]),
                        singular_values_=list(r["singular_values_"]), n_cols=int(r["n_cols"]), dtype=str(r["dtype"]))


class PCAModel(PCAClass, _CumlModelWithColumns, _PCACumlParams):
    """reference: feature.py:263-459.  transform() appends outputCol = X . components^T (array<float>); the mean is not
    subtracted, as in Spark."""

    def __init__(self, mean_: List[float], components_: List[List[float]], explained_variance_ratio_: List[float],
                 singular_values_: List[float], n_cols: int, dtype: str):
        super().__init__(n_cols=n_cols, dtype=dtype, mean_=mean_, components_=components_,
                         explained_variance_ratio_=explained_variance_ratio_, singular_values_=singular_values_)
        self.mean_ = mean_
        self.components_ = components_
        self.explained_variance_ratio_ = explained_variance_ratio_
        self.singular_values_ = singular_values_
        self._set_params(n_components=len(components_))

    @property
    def mean(self) -> List[float]:
        return self.mean_

    @property
    def pc(self) -> Any:
        """The principal components, one per column: pyspark DenseMatrix [d, k] when pyspark.ml.linalg provides it,
        else a numpy array [d, k]."""
        num_rows, num_cols = len(self.components_), int(self.n_cols)
        try:
            from pyspark.ml.linalg import DenseMatrix
        except ImportError:
            return np.array(self.components_, dtype=np.float64).reshape(num_rows, num_cols).T
        values = list(itertools.chain.from_iterable(self.components_))
        return DenseMatrix(num_cols, num_rows, values, False)   # column major: flip rows/cols (feature.py:387-390)

    @property
    def explainedVariance(self) -> Any:
        """Proportion of the variance each component explains: pyspark DenseVector when available, else numpy."""
        try:
            from pyspark.ml.linalg import DenseVector
        except ImportError:
            return np.array(self.explained_variance_ratio_, dtype=np.float64)
        return DenseVector(self.explained_variance_ratio_)

    def cpu(self) -> Any:
        raise NotImplementedError("PCAModel.cpu() builds a JVM pyspark.ml PCAModel; no JVM/pyspark in this build")

    def _output_col_name(self) -> str:
        return self.getOrDefault("outputCol")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "array<float>"

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        components_ = self.components_
        n_cols = int(self.n_cols)

        class _DevicePCA:
            def __init__(self, gpu: int) -> None:
                import torch

                self.ctx = _transform_context(gpu)
                self.C = torch.tensor(components_, dtype=torch.float32, device=self.ctx.device)

            def close(self) -> None:   # the context stays with the process
                self.C = None

        def _construct_pca(gpu: int = 0) -> Any:
            return _DevicePCA(gpu)

        def _transform_many(pca: Any, dfs: List[Union[pd.DataFrame, np.ndarray]]) -> List[pd.Series]:
            """Several input batches in ONE device pass: every batch is ingested into the same device matrix, one
            b2k_pca_transform projects all rows, one read-back, one Series per input batch."""
            from .utils import DeviceRowAppender

            sizes = [len(df) for df in dfs]
            total = sum(sizes)
            if total == 0:
                return [pd.Series([], dtype=object) for _ in dfs]
            app = DeviceRowAppender(pca.ctx, n_cols, first_capacity=total)
            for df, n_b in zip(dfs, sizes):
                if n_b:
                    _append_transform_features(app, df, n_cols)
            host = pca.ctx.pca_transform(app.finish(), pca.C).cpu().numpy()
            out, o = [], 0
            for n_b in sizes:
                out.append(pd.Series(list(host[o:o + n_b])))
                o += n_b
            return out

        def _transform_internal(pca: Any, df: Union[pd.DataFrame, np.ndarray]) -> pd.Series:
            return _transform_many(pca, [df])[0]

        _transform_internal.many = _transform_many  # type: ignore[attr-defined]
        _transform_internal.row_bytes = 4 * (n_cols + len(components_))  # type: ignore[attr-defined]
        return _construct_pca, _transform_internal, None
