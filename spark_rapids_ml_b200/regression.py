"""LinearRegression / LinearRegressionModel — the reference's distributed linear regression surface
(python/src/spark_rapids_ml/regression.py:181-862), with the cuML calls replaced by libb2kmeans (hand-written sm_90a
CUDA behind include/b2kmeans.h).

  LinearRegressionClass (param and value mappings, cuML defaults)          regression.py:181-234
  _LinearRegressionCumlParams (featuresCol(s), labelCol, predictionCol)   regression.py:237-288
  LinearRegression (keyword-only ctor, setters, fit function, fitMultiple) regression.py:291-700
  LinearRegressionModel (coefficients, intercept, transform)              regression.py:703-862

Semantics (b2k_linreg_moments / b2k_linreg_solve): one pass over the data forms the fp64 means and centred second
moments of [X | y] (labels cast to float32); every solver setting is then solved from them on the host in fp64 —
Cholesky (minimum norm on singular systems) for OLS and ridge, coordinate descent for the lasso and the elastic net.
Standardization scales by the population standard deviations, as MLlib does, so the coefficients match MLlib's; the
penalty is in the units of the standardized label (lambda / sigma_y), as in the reference's cuML calls.  transform()
appends predictionCol = intercept + x . coefficients as a double column, accumulated in fp64.

Differences that are deliberate: the reference standardizes with the sample standard deviation (/(n - 1)), which
moves its answers 0.2 % - 7 % off MLlib's; d = 1 is fitted (the reference rejects it for OLS and ridge); a constant
label is handled as MLlib handles it (the reference divides by zero).  Without standardization the penalty is applied
in label units, as the reference does, where MLlib still scales it by sigma_y.  No CPU fallback: cpu(), predict(),
evaluate() and summary raise NotImplementedError; loss="huber", solver="l-bfgs" and weightCol raise.
"""
from __future__ import annotations

import functools
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np

from .core import FitInputType, _CumlModelWithPredictionCol, _DeviceModel, _TunedEstimator, param_alias
from .params import HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasPredictionCol, P, _CumlClass, _CumlParams
from .sparkshim import Param, Row, TypeConverters, keyword_only


class LinearRegressionClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {
            "aggregationDepth": "",
            "elasticNetParam": "l1_ratio",
            "epsilon": "",
            "fitIntercept": "fit_intercept",
            "loss": "loss",
            "maxBlockSizeInMB": "",
            "maxIter": "max_iter",
            "regParam": "alpha",
            "solver": "solver",
            "standardization": "normalize",
            "tol": "tol",
            "weightCol": None,
        }

    @classmethod
    def _param_value_mapping(cls) -> Dict[str, Callable[[Any], Union[None, str, float, int]]]:
        return {
            "loss": lambda x: {"squaredError": "squared_loss", "huber": None, "squared_loss": "squared_loss"}.get(x, None),
            "solver": lambda x: {"auto": "auto", "normal": "eig", "l-bfgs": None, "eig": "eig"}.get(x, None),
        }

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"algorithm": "auto", "fit_intercept": True, "copy_X": True, "normalize": False, "verbose": False,
                "alpha": 0.0001, "solver": "auto", "loss": "squared_loss", "l1_ratio": 0.15, "max_iter": 1000,
                "tol": 0.001, "shuffle": True}

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.regression.LinearRegression when pyspark is installed


class _LinearRegressionParams(HasFeaturesCol, HasLabelCol, HasPredictionCol):
    """pyspark.ml.regression._LinearRegressionParams stand-in, with Spark's defaults."""

    regParam = Param("parent", "regParam", "regularization parameter (>= 0).", TypeConverters.toFloat)
    elasticNetParam = Param("parent", "elasticNetParam", "the ElasticNet mixing parameter, in range [0, 1]. For alpha "
                            "= 0, the penalty is an L2 penalty. For alpha = 1, it is an L1 penalty.",
                            TypeConverters.toFloat)
    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    tol = Param("parent", "tol", "the convergence tolerance for iterative algorithms (>= 0).", TypeConverters.toFloat)
    fitIntercept = Param("parent", "fitIntercept", "whether to fit an intercept term.")
    standardization = Param("parent", "standardization", "whether to standardize the training features before fitting "
                            "the model.")
    solver = Param("parent", "solver", "The solver algorithm for optimization: auto, normal, l-bfgs.",
                   TypeConverters.toString)
    loss = Param("parent", "loss", "The loss function to be optimized: squaredError, huber.", TypeConverters.toString)
    epsilon = Param("parent", "epsilon", "The shape parameter to control the amount of robustness (> 1.0).",
                    TypeConverters.toFloat)
    aggregationDepth = Param("parent", "aggregationDepth", "suggested depth for treeAggregate (>= 2).",
                             TypeConverters.toInt)
    maxBlockSizeInMB = Param("parent", "maxBlockSizeInMB", "maximum memory in MB for stacking input data.",
                             TypeConverters.toFloat)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(labelCol="label", maxIter=100, regParam=0.0, elasticNetParam=0.0, tol=1e-6,
                         fitIntercept=True, standardization=True, solver="auto", loss="squaredError", epsilon=1.35,
                         aggregationDepth=2, maxBlockSizeInMB=0.0)

    def getRegParam(self) -> float:
        return self.getOrDefault(self.regParam)

    def getElasticNetParam(self) -> float:
        return self.getOrDefault(self.elasticNetParam)

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getTol(self) -> float:
        return self.getOrDefault(self.tol)

    def getFitIntercept(self) -> bool:
        return self.getOrDefault(self.fitIntercept)

    def getStandardization(self) -> bool:
        return self.getOrDefault(self.standardization)

    def getSolver(self) -> str:
        return self.getOrDefault(self.solver)

    def getLoss(self) -> str:
        return self.getOrDefault(self.loss)

    def getEpsilon(self) -> float:
        return self.getOrDefault(self.epsilon)


class _LinearRegressionCumlParams(_CumlParams, _LinearRegressionParams, HasFeaturesCols):
    """Shared Spark Params of LinearRegression and LinearRegressionModel (reference: regression.py:237-288)."""

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

    def setLabelCol(self: P, value: str) -> P:
        return self._set_params(labelCol=value)

    def setPredictionCol(self: P, value: str) -> P:
        return self._set_params(predictionCol=value)


class LinearRegression(LinearRegressionClass, _TunedEstimator, _LinearRegressionCumlParams):
    """Linear regression on H100 under the squared loss: OLS (regParam = 0), ridge (elasticNetParam = 0), lasso
    (elasticNetParam = 1) and the elastic net in between, with or without an intercept and standardization.  One barrier
    task per GPU runs one pass over the device-resident partition (column sums, then a wgmma Gram pass and a fused
    X^T y pass, fp64 partials) and two fp64 NCCL allreduces; the solve runs on the host in fp64 from the moments.
    Parameters as in the reference (regression.py:291-433): featuresCol (str for an array column, list of str for
    scalar columns), labelCol, predictionCol, maxIter (100), regParam (0.0), elasticNetParam (0.0), tol (1e-6),
    fitIntercept (True), standardization (True), solver ("auto" | "normal"), loss ("squaredError"), num_workers,
    verbose.

    >>> from spark_rapids_ml_b200.regression import LinearRegression
    >>> df = session.createDataFrame([([1.0, 0.0], 3.0), ([0.0, 1.0], 5.0), ([1.0, 1.0], 8.0), ([2.0, 1.0], 10.0)],
    ...                              "features array<float>, label float")
    >>> model = LinearRegression(regParam=0.0).fit(df)
    >>> model.coefficients, model.intercept   # ([2.0, 5.0], 1.0)
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", labelCol: str = "label",
                 predictionCol: str = "prediction", maxIter: int = 100, regParam: float = 0.0,
                 elasticNetParam: float = 0.0, tol: float = 1e-6, fitIntercept: bool = True,
                 standardization: bool = True, solver: str = "auto", loss: str = "squaredError",
                 num_workers: Optional[int] = None, verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        if self._input_kwargs.get("num_workers", None) is None:
            self._input_kwargs.pop("num_workers", None)
        self._set_params(**self._input_kwargs)

    # every map is solved from one moments pass over the data
    _single_pass_params = frozenset(("regParam", "elasticNetParam", "maxIter", "tol", "fitIntercept",
                                     "standardization"))

    def _settings(self) -> Dict[str, Any]:
        cp = self.cuml_params
        return {"reg": float(cp["alpha"]), "l1_ratio": float(cp["l1_ratio"]),
                "fit_intercept": bool(cp["fit_intercept"]), "standardization": bool(cp["normalize"]),
                "max_iter": int(cp["max_iter"]), "tol": float(cp["tol"])}

    def setMaxIter(self, value: int) -> "LinearRegression":
        return self._set_params(maxIter=value)

    def setRegParam(self, value: float) -> "LinearRegression":
        return self._set_params(regParam=value)

    def setElasticNetParam(self, value: float) -> "LinearRegression":
        return self._set_params(elasticNetParam=value)

    def setLoss(self, value: str) -> "LinearRegression":
        return self._set_params(loss=value)

    def setStandardization(self, value: bool) -> "LinearRegression":
        return self._set_params(standardization=value)

    def setTol(self, value: float) -> "LinearRegression":
        return self._set_params(tol=value)

    def setFitIntercept(self, value: bool) -> "LinearRegression":
        return self._set_params(fitIntercept=value)

    def setSolver(self, value: str) -> "LinearRegression":
        return self._set_params(solver=value)

    def setWeightCol(self, value: str) -> "LinearRegression":
        raise ValueError("'weightCol' is not supported by cuML.")

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        _check_solver_settings(self._settings())

    def _fit_label_col(self) -> Optional[str]:
        return self.getLabelCol()

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        grid = self._fit_grid or [self._settings()]

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for LinearRegressionMG / RidgeMG / CDMG(handle, ...).fit(...) and the coefficient rescaling —
            # regression.py:520-700; every solver setting is solved from one moments pass
            from . import _native

            ctx = params[param_alias.handle]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            X, y, _ = dfs[0]
            n_total, mean, moments = ctx.linreg_moments(X, y)
            out: Dict[str, List[Any]] = {"coef_": [], "intercept_": [], "n_cols": [], "dtype": []}
            for s in grid:
                coef, b, _ = _native.linreg_solve(mean, moments, n_total, **s)
                out["coef_"].append(coef.tolist())
                out["intercept_"].append(b)
                out["n_cols"].append(params[param_alias.num_cols])
                out["dtype"].append("float32")
            return out

        return _cuml_fit

    def _out_schema(self) -> Any:
        return "coef_ array<double>, intercept_ double, n_cols int, dtype string"

    def _create_pyspark_model(self, result: Row) -> "LinearRegressionModel":
        r = result.asDict()
        return LinearRegressionModel(coef_=list(r["coef_"]), intercept_=float(r["intercept_"]), n_cols=int(r["n_cols"]),
                                     dtype=str(r["dtype"]))

    def _supportsTransformEvaluate(self, evaluator: Any) -> bool:
        from .core import _supports_transform_evaluate

        return _supports_transform_evaluate(False, evaluator)


def _check_solver_settings(s: Dict[str, Any]) -> None:
    """The errors b2k_linreg_solve would return, raised on the driver before any task starts."""
    if not s["reg"] >= 0:
        raise ValueError(f"regParam given invalid value {s['reg']!r}")
    if not 0 <= s["l1_ratio"] <= 1:
        raise ValueError(f"elasticNetParam given invalid value {s['l1_ratio']!r}")
    if s["max_iter"] < 0:
        raise ValueError(f"maxIter given invalid value {s['max_iter']!r}")
    if not s["tol"] >= 0:
        raise ValueError(f"tol given invalid value {s['tol']!r}")


class LinearRegressionModel(LinearRegressionClass, _CumlModelWithPredictionCol, _LinearRegressionCumlParams):
    """reference: regression.py:703-862.  transform() appends predictionCol = intercept + x . coefficients (double)."""

    def __init__(self, coef_: List[float], intercept_: float, n_cols: int, dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype, coef_=coef_, intercept_=intercept_)
        self.coef_ = coef_
        self.intercept_ = intercept_

    @property
    def coefficients(self) -> Any:
        """pyspark DenseVector when pyspark.ml.linalg provides it, else a numpy array."""
        try:
            from pyspark.ml.linalg import DenseVector
        except ImportError:
            return np.array(self.coef_, dtype=np.float64)
        return DenseVector(self.coef_)

    @property
    def intercept(self) -> float:
        return float(self.intercept_)

    @property
    def scale(self) -> float:
        return 1.0

    @property
    def hasSummary(self) -> bool:
        return False

    @property
    def summary(self) -> Any:
        raise NotImplementedError("LinearRegressionModel has no training summary in this build")

    def evaluate(self, dataset: Any) -> Any:
        raise NotImplementedError("LinearRegressionModel.evaluate() is not supported in this build")

    def predict(self, value: Any) -> float:
        raise NotImplementedError("LinearRegressionModel.predict() of a single vector is not supported; use transform()")

    def cpu(self) -> Any:
        raise NotImplementedError("LinearRegressionModel.cpu() builds a JVM pyspark.ml model; no JVM/pyspark in this build")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "double"

    _combined_attrs = ("coef_", "intercept_")

    def _models(self) -> List[Tuple[List[float], float]]:
        if isinstance(self.intercept_, (list, tuple)):
            return [(list(c), float(b)) for c, b in zip(self.coef_, self.intercept_)]
        return [(list(self.coef_), float(self.intercept_))]

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        if eval_metric_info is not None:
            return self._eval_func(eval_metric_info)
        if isinstance(self.intercept_, (list, tuple)):
            raise NotImplementedError("transform() of a combined multi-model instance is not supported")
        intercept_ = float(self.intercept_)
        construct = functools.partial(_DeviceModel, w=np.asarray(self.coef_, dtype=np.float64))
        transform = self._grouped_transform(lambda m, X: (m.ctx.linreg_predict(X, m.arrays["w"], intercept_),),
                                            4 * int(self.n_cols) + 8)
        return construct, transform, None

    def _eval_func(self, info: Dict[str, Any]) -> Tuple[Callable, Any, Callable]:
        """(construct, None, evaluate): evaluate(device model, X, y) scores every model on one device pass
        (b2k_eval_linear, identity kind) and returns their accumulators."""
        from .core import _class_accs

        if info["classification"]:
            raise NotImplementedError("LinearRegressionModel is evaluated with a RegressionEvaluator")
        models = [{"kind": "identity", "W": np.asarray([c], dtype=np.float64), "b": [b]} for c, b in self._models()]

        def _evaluate(h: Any, X: Any, y: Any) -> List[Dict[str, Any]]:
            return _class_accs(h.ctx.eval_linear(X, y, models))

        return _DeviceModel, None, _evaluate


from .tree import _RandomForestEstimator, _RandomForestModel  # noqa: E402  (tree.py imports this module lazily)


class RandomForestRegressor(_RandomForestEstimator):
    """Random forest regression on H100 (reference regression.py:865-1048).  Every tree is grown from the variance
    histograms of all workers' rows, with one allreduce per histogram pass, so the forest does not depend on the number
    of workers.  Labels are resolved to max|y| 2^-24 (DESIGN.md §15).  Parameters as in the reference: featuresCol (str
    or list of str), labelCol, predictionCol, maxDepth (5), maxBins (32), minInstancesPerNode (1), minInfoGain (0.0),
    impurity ("variance"), numTrees (20), featureSubsetStrategy ("auto"), seed, bootstrap (True), num_workers,
    verbose.

    >>> from spark_rapids_ml_b200.regression import RandomForestRegressor
    >>> df = session.createDataFrame([([1.0, 2.0], 1.5), ([1.0, 3.0], 2.5), ([2.0, 1.0], 0.5), ([3.0, 1.0], 0.0)],
    ...                              "features array<float>, label float")
    >>> RandomForestRegressor(numTrees=3, bootstrap=False).fit(df).transform(df)
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", labelCol: str = "label",
                 predictionCol: str = "prediction", maxDepth: int = 5, maxBins: int = 32, minInstancesPerNode: int = 1,
                 minInfoGain: float = 0.0, maxMemoryInMB: int = 256, cacheNodeIds: bool = False,
                 checkpointInterval: int = 10, impurity: str = "variance", subsamplingRate: float = 1.0,
                 seed: Optional[int] = None, numTrees: int = 20, featureSubsetStrategy: str = "auto",
                 leafCol: str = "", minWeightFractionPerNode: float = 0.0, weightCol: Optional[str] = None,
                 bootstrap: Optional[bool] = True, num_workers: Optional[int] = None, verbose: Union[int, bool] = False,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)

    def _init_defaults(self) -> None:
        self._setDefault(impurity="variance")

    def _is_classification(self) -> bool:
        return False

    def _model_class(self) -> Any:
        return RandomForestRegressionModel


class RandomForestRegressionModel(_RandomForestModel):
    """reference: regression.py:1051-1147.  transform() appends predictionCol, the mean of the trees' leaf values in
    tree order."""

    def _init_defaults(self) -> None:
        self._setDefault(impurity="variance")

    def _is_classification(self) -> bool:
        return False

    def evaluate(self, dataset: Any) -> Any:
        raise NotImplementedError("RandomForestRegressionModel.evaluate() is not supported in this build")
