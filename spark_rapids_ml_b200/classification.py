"""LogisticRegression / LogisticRegressionModel — the reference's distributed logistic regression surface
(python/src/spark_rapids_ml/classification.py:679-1614), with the cuML calls replaced by libb2kmeans (hand-written sm_90a
CUDA behind include/b2kmeans.h).

  LogisticRegressionClass (param and value mappings, cuML defaults)            classification.py:679-747
  _LogisticRegressionCumlParams (featuresCol(s), label, prediction columns)    classification.py:750-819
  LogisticRegression (keyword-only ctor, setters, fit function, fitMultiple)   classification.py:822-1303
  LogisticRegressionModel (coefficients, intercepts, transform, _combine)      classification.py:1306-1614

Semantics (b2k_logreg_labels / b2k_logreg_fit): MLlib's objective, (1/n) sum of the logistic (binomial) or softmax
(multinomial) loss + regParam ((1 - elasticNetParam)/2 |V|^2 + elasticNetParam |V|_1), V the coefficients scaled by the
sample standard deviations of the features with standardization.  Every optimiser step is one fused pass over the
device-resident rows (margins, residuals and the gradient X^T R in one read of X, fp64) and one allreduce; L-BFGS /
OWL-QN runs on the host in fp64.  transform() appends rawPrediction and probability (double vectors) and prediction
(the class value of the largest margin, a double).

Differences that are deliberate: with regParam = 0 a multinomial fit centres its coefficients per feature, as MLlib
does (the reference reports wherever its solver stopped on a problem without a unique solution); the classes are the
sorted distinct label values and the prediction is the class value, not its index; labels must be below 1024.  No CPU
fallback: cpu(), predict(), predictRaw(), predictProbability() and evaluate() raise NotImplementedError; weightCol,
threshold(s), the coefficient / intercept bounds and enable_sparse_data_optim=True raise ValueError; there is no
training summary.

Sparse input (DESIGN §21): a local frame whose features are Spark vectors in their SQL layout, struct<type: tinyint,
size: int, indices: array<int>, values: array<double>>, sparse and dense rows mixed.  With enable_sparse_data_optim=None
(the default) and a sparse first row, the rows stay sparse: one device CSR per partition, a CSC copy built once per fit,
and every evaluation is a rows pass and a column pass over the stored entries, so d may reach 2^25 / K' - 1 (K' = 1
for a binomial fit, numClasses for a multinomial one: K' (d + 1) <= 2^25).  Otherwise (a dense first row, or enable_sparse_data_optim=False) the rows are densified
into the dense path.  Both solve the same problem.  transform() of a vector struct column runs the CSR predict, for a
model fitted either way; CrossValidator and _transformEvaluate of such a frame raise NotImplementedError.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pyarrow as pa

from .core import (FitInputType, _CumlEstimator, _CumlModelWithPredictionCol, _DeviceModel, _TunedEstimator, alias,
                   param_alias)
from .params import HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasPredictionCol, P, _CumlClass, _CumlParams
from .tree import _RandomForestEstimator, _RandomForestModel
from .sparkshim import HAVE_PYSPARK, LocalDataFrame, Param, Row, TypeConverters, keyword_only
from .utils import densify_vector_column, get_logger, is_vector_struct


class LogisticRegressionClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {
            "maxIter": "max_iter",
            "regParam": "C",
            "elasticNetParam": "l1_ratio",
            "tol": "tol",
            "fitIntercept": "fit_intercept",
            "threshold": None,
            "thresholds": None,
            "standardization": "standardization",
            "weightCol": None,
            "aggregationDepth": "",
            "family": "",
            "lowerBoundsOnCoefficients": None,
            "upperBoundsOnCoefficients": None,
            "lowerBoundsOnIntercepts": None,
            "upperBoundsOnIntercepts": None,
            "maxBlockSizeInMB": "",
        }

    @classmethod
    def _param_value_mapping(cls) -> Dict[str, Callable[[Any], Union[None, str, float, int]]]:
        return {"C": lambda x: 1 / x if x > 0.0 else (0.0 if x == 0.0 else None)}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"fit_intercept": True, "standardization": False, "verbose": False, "C": 1.0, "penalty": "l2",
                "l1_ratio": None, "max_iter": 1000, "tol": 0.0001}

    @classmethod
    def _reg_params_value_mapping(cls, reg_param: float, elasticNet_param: float) -> Tuple[Optional[str], float, float]:
        """Spark's (regParam, elasticNetParam) -> cuML's (penalty, C, l1_ratio)."""
        if reg_param == 0.0:
            return None, 0.0, elasticNet_param
        penalty = "l2" if elasticNet_param == 0.0 else "l1" if elasticNet_param == 1.0 else "elasticnet"
        return penalty, 1.0 / reg_param, elasticNet_param

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.classification.LogisticRegression when pyspark is installed


class _LogisticRegressionParams(HasFeaturesCol, HasLabelCol, HasPredictionCol):
    """pyspark.ml.classification._LogisticRegressionParams stand-in, with Spark's defaults."""

    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    regParam = Param("parent", "regParam", "regularization parameter (>= 0).", TypeConverters.toFloat)
    elasticNetParam = Param("parent", "elasticNetParam", "the ElasticNet mixing parameter, in range [0, 1]. For alpha "
                            "= 0, the penalty is an L2 penalty. For alpha = 1, it is an L1 penalty.",
                            TypeConverters.toFloat)
    tol = Param("parent", "tol", "the convergence tolerance for iterative algorithms (>= 0).", TypeConverters.toFloat)
    fitIntercept = Param("parent", "fitIntercept", "whether to fit an intercept term.")
    standardization = Param("parent", "standardization", "whether to standardize the training features before fitting "
                            "the model.")
    threshold = Param("parent", "threshold", "Threshold in binary classification prediction, in range [0, 1].",
                      TypeConverters.toFloat)
    thresholds = Param("parent", "thresholds", "Thresholds in multi-class classification to adjust the probability of "
                       "predicting each class.")
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)
    aggregationDepth = Param("parent", "aggregationDepth", "suggested depth for treeAggregate (>= 2).",
                             TypeConverters.toInt)
    family = Param("parent", "family", "The name of family which is a description of the label distribution to be used "
                   "in the model. Supported options: auto, binomial, multinomial", TypeConverters.toString)
    lowerBoundsOnCoefficients = Param("parent", "lowerBoundsOnCoefficients", "The lower bounds on coefficients.")
    upperBoundsOnCoefficients = Param("parent", "upperBoundsOnCoefficients", "The upper bounds on coefficients.")
    lowerBoundsOnIntercepts = Param("parent", "lowerBoundsOnIntercepts", "The lower bounds on intercepts.")
    upperBoundsOnIntercepts = Param("parent", "upperBoundsOnIntercepts", "The upper bounds on intercepts.")
    maxBlockSizeInMB = Param("parent", "maxBlockSizeInMB", "maximum memory in MB for stacking input data.",
                             TypeConverters.toFloat)
    probabilityCol = Param("parent", "probabilityCol", "Column name for predicted class conditional probabilities.",
                           TypeConverters.toString)
    rawPredictionCol = Param("parent", "rawPredictionCol", "raw prediction (a.k.a. confidence) column name.",
                             TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(labelCol="label", maxIter=100, regParam=0.0, elasticNetParam=0.0, tol=1e-6,
                         fitIntercept=True, threshold=0.5, standardization=True, aggregationDepth=2, family="auto",
                         maxBlockSizeInMB=0.0, probabilityCol="probability", rawPredictionCol="rawPrediction")

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getRegParam(self) -> float:
        return self.getOrDefault(self.regParam)

    def getElasticNetParam(self) -> float:
        return self.getOrDefault(self.elasticNetParam)

    def getTol(self) -> float:
        return self.getOrDefault(self.tol)

    def getFitIntercept(self) -> bool:
        return self.getOrDefault(self.fitIntercept)

    def getStandardization(self) -> bool:
        return self.getOrDefault(self.standardization)

    def getFamily(self) -> str:
        return self.getOrDefault(self.family)

    def getThreshold(self) -> float:
        return self.getOrDefault(self.threshold)

    def getProbabilityCol(self) -> str:
        return self.getOrDefault(self.probabilityCol)

    def getRawPredictionCol(self) -> str:
        return self.getOrDefault(self.rawPredictionCol)


class _LogisticRegressionCumlParams(_CumlParams, _LogisticRegressionParams, HasFeaturesCols):
    """Shared Spark Params of LogisticRegression and LogisticRegressionModel (reference: classification.py:750-819)."""

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

    def setProbabilityCol(self: P, value: str) -> P:
        return self._set_params(probabilityCol=value)

    def setRawPredictionCol(self: P, value: str) -> P:
        return self._set_params(rawPredictionCol=value)

    def setThreshold(self: P, value: float) -> P:
        return self._set_params(threshold=value)

    def setThresholds(self: P, value: List[float]) -> P:
        return self._set_params(thresholds=value)


def _check_settings(s: Dict[str, Any]) -> None:
    """The errors b2k_logreg_fit would return, raised on the driver before any task starts."""
    if s["max_iter"] < 0:
        raise ValueError(f"maxIter given invalid value {s['max_iter']}")
    if not s["reg"] >= 0:
        raise ValueError(f"C or regParam given an invalid or unsupported value {s['reg']!r}")
    if not 0 <= s["l1_ratio"] <= 1:
        raise ValueError(f"elasticNetParam given invalid value {s['l1_ratio']!r}")
    if not s["tol"] >= 0:
        raise ValueError(f"tol given invalid value {s['tol']!r}")


class LogisticRegression(LogisticRegressionClass, _TunedEstimator, _LogisticRegressionCumlParams):
    """Logistic regression on H100: binomial or multinomial, with no penalty, L2, L1 or the elastic net, with or without
    an intercept and standardization.  One barrier task per GPU holds its partition on the device; the label pass and
    a column-moments pass run once, then every L-BFGS / OWL-QN step evaluates the loss and gradient in one fused fp64
    pass over the rows and one NCCL allreduce.  Parameters as in the reference (classification.py:822-955):
    featuresCol (str for an array column, list of str for scalar columns), labelCol, predictionCol, probabilityCol,
    rawPredictionCol, maxIter (100), regParam (0.0), elasticNetParam (0.0), tol (1e-6), fitIntercept (True),
    standardization (True), family ("auto"), num_workers, verbose.

    >>> from spark_rapids_ml_b200.classification import LogisticRegression
    >>> df = session.createDataFrame([([1.0, 2.0], 1.0), ([1.0, 3.0], 1.0), ([2.0, 1.0], 0.0), ([3.0, 1.0], 0.0)],
    ...                              "features array<float>, label float")
    >>> LogisticRegression(regParam=0.01).fit(df).coefficients   # [-2.48197, 2.48197]
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", labelCol: str = "label",
                 predictionCol: str = "prediction", probabilityCol: str = "probability",
                 rawPredictionCol: str = "rawPrediction", maxIter: int = 100, regParam: float = 0.0,
                 elasticNetParam: float = 0.0, tol: float = 1e-6, fitIntercept: bool = True,
                 standardization: bool = True, enable_sparse_data_optim: Optional[bool] = None,
                 float32_inputs: bool = True, num_workers: Optional[int] = None, verbose: Union[int, bool] = False,
                 **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._set_cuml_reg_params()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        self._sparse_data_optim = self._input_kwargs.pop("enable_sparse_data_optim", None)
        if self._sparse_data_optim:
            raise ValueError("enable_sparse_data_optim=True is not supported by spark_rapids_ml_b200's "
                             "LogisticRegression; leave it at None (the default) to fit sparse vectors as CSR")
        if self._input_kwargs.get("num_workers", None) is None:
            self._input_kwargs.pop("num_workers", None)
        self._set_params(**self._input_kwargs)

    # every map is fitted from one ingest, one label pass and one moments pass, then optimised on its own
    _single_pass_params = frozenset(("regParam", "elasticNetParam", "maxIter", "tol", "fitIntercept",
                                     "standardization", "family"))

    def _settings(self) -> Dict[str, Any]:
        family = self.getFamily().lower()
        if family not in ("auto", "binomial", "multinomial"):
            raise ValueError(f"family given invalid value {self.getFamily()}")
        return {"reg": float(self.getRegParam()), "l1_ratio": float(self.getElasticNetParam()),
                "tol": float(self.getTol()), "max_iter": int(self.getMaxIter()),
                "fit_intercept": bool(self.getFitIntercept()), "standardization": bool(self.getStandardization()),
                "family": family}

    def _set_cuml_reg_params(self) -> "LogisticRegression":
        penalty, C, l1_ratio = self._reg_params_value_mapping(self.getRegParam(), self.getElasticNetParam())
        self._cuml_params["penalty"] = penalty
        self._cuml_params["C"] = C
        self._cuml_params["l1_ratio"] = l1_ratio
        return self

    def _set_params(self, **kwargs: Any) -> "LogisticRegression":
        super()._set_params(**kwargs)
        if "regParam" in kwargs or "elasticNetParam" in kwargs:
            self._set_cuml_reg_params()
        return self

    def setMaxIter(self, value: int) -> "LogisticRegression":
        return self._set_params(maxIter=value)

    def setRegParam(self, value: float) -> "LogisticRegression":
        return self._set_params(regParam=value)

    def setElasticNetParam(self, value: float) -> "LogisticRegression":
        return self._set_params(elasticNetParam=value)

    def setTol(self, value: float) -> "LogisticRegression":
        return self._set_params(tol=value)

    def setFitIntercept(self, value: bool) -> "LogisticRegression":
        return self._set_params(fitIntercept=value)

    def setStandardization(self, value: bool) -> "LogisticRegression":
        return self._set_params(standardization=value)

    def setFamily(self, value: str) -> "LogisticRegression":
        return self._set_params(family=value)

    def setWeightCol(self, value: str) -> "LogisticRegression":
        raise ValueError("'weightCol' is not supported by cuML.")

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        _check_settings(self._settings())

    def _fit_label_col(self) -> Optional[str]:
        return self.getLabelCol()

    def _pre_process_features(self, dataset: LocalDataFrame) -> Tuple[LocalDataFrame, Optional[List[str]], int, str]:
        """A vector struct column: kept as vectors for the CSR path ("csr") when enable_sparse_data_optim is None and
        the first row is sparse, else densified to array<float> (the reference's rule, core.py:507-521).  Other feature
        columns as for every estimator."""
        col = _vector_column(dataset, self.getFeaturesCol())
        if col is None:
            return super()._pre_process_features(dataset)
        df = dataset.select(col).withColumnRenamed(col, alias.data)
        first = df.first()
        if first is None:
            raise RuntimeError("A python worker received no data.  Please increase amount of data or use fewer workers.")
        v = first[alias.data]
        if v is None:
            raise ValueError("null feature rows are not supported")
        sparse = v["type"] == 0
        dimension = int(v["size"]) if sparse else len(v["values"])
        if getattr(self, "_sparse_data_optim", None) is None and sparse:
            return df, None, dimension, "csr"
        parts = [[pa.RecordBatch.from_arrays([densify_vector_column(b.column(0), dimension)], names=[alias.data])
                  for b in p] for p in df._parts]
        return df._derive(parts, pa.schema([pa.field(alias.data, pa.list_(pa.float32()))])), None, dimension, "float"

    def _check_tuning_input(self, dataset: Any) -> None:
        """CrossValidator's single-pass evaluation reads dense rows: a vector struct frame is refused before any fit."""
        if isinstance(dataset, LocalDataFrame) and _vector_column(dataset, self.getFeaturesCol()) is not None:
            raise NotImplementedError("CrossValidator of LogisticRegression on sparse input (a vector struct features "
                                      "column) is not supported: the single-pass evaluation kernels read dense rows")

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        grid = self._fit_grid or [self._settings()]

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for LogisticRegressionMG(handle, ...).fit(...) per param map, the rescaling and the intercept
            # centring — classification.py:984-1192; one label pass and one moments pass serve every map
            ctx = params[param_alias.handle]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            X, y, _ = dfs[0]
            classes, counts, _n = ctx.logreg_labels(y)
            if isinstance(X, tuple):   # the device CSR (indptr, indices, values) of a sparse frame
                fits = ctx.logreg_fit_csr(X, params[param_alias.num_cols], y, classes, counts, grid)
            else:
                fits = ctx.logreg_fit(X, y, classes, counts, grid)
            out: Dict[str, List[Any]] = {"coef_": [], "intercept_": [], "classes_": [], "n_cols": [], "dtype": [],
                                         "num_iters": []}
            for coef, icpt, iters in fits:
                out["coef_"].append(coef.tolist())
                out["intercept_"].append(icpt.tolist())
                out["classes_"].append(classes.tolist())
                out["n_cols"].append(params[param_alias.num_cols])
                out["dtype"].append("float32")
                out["num_iters"].append(iters)
            return out

        return _cuml_fit

    def _out_schema(self) -> Any:
        return ("coef_ array<array<double>>, intercept_ array<double>, classes_ array<double>, n_cols int, "
                "dtype string, num_iters int")

    def _create_pyspark_model(self, result: Row) -> "LogisticRegressionModel":
        r = result.asDict()
        if len(r["classes_"]) == 1:
            if self.getFitIntercept() is False:
                raise ValueError("All labels belong to a single class and fitIntercept=false. This is not supported.  "
                                 "Please use fitIntercept=true.")
            self.logger.warning("All labels are the same value and fitIntercept=true, so the coefficients will be "
                                "zeros. Training is not needed.")
        return LogisticRegressionModel(coef_=[list(c) for c in r["coef_"]], intercept_=list(r["intercept_"]),
                                       classes_=list(r["classes_"]), n_cols=int(r["n_cols"]), dtype=str(r["dtype"]),
                                       num_iters=int(r["num_iters"]))

    def _supportsTransformEvaluate(self, evaluator: Any) -> bool:
        from .core import _supports_transform_evaluate

        return _supports_transform_evaluate(True, evaluator)


class LogisticRegressionModel(LogisticRegressionClass, _CumlModelWithPredictionCol, _LogisticRegressionCumlParams):
    """reference: classification.py:1306-1614.  transform() appends rawPredictionCol and probabilityCol (double
    vectors) and predictionCol (double)."""

    def __init__(self, coef_: Union[List[List[float]], List[List[List[float]]]],
                 intercept_: Union[List[float], List[List[float]]], classes_: List[float], n_cols: int, dtype: str,
                 num_iters: int) -> None:
        super().__init__(dtype=dtype, n_cols=n_cols, coef_=coef_, intercept_=intercept_, classes_=classes_,
                         num_iters=num_iters)
        self.coef_ = coef_
        self.intercept_ = intercept_
        self.classes_ = classes_
        self._num_classes = len(self.classes_)
        self.num_iters = num_iters

    def _get_num_models(self) -> int:
        return 1 if isinstance(self.intercept_[0], float) else len(self.intercept_)

    @property
    def coefficients(self) -> Any:
        """pyspark DenseVector when pyspark.ml.linalg provides it, else a numpy array."""
        if isinstance(self.coef_[0][0], float):
            if len(self.coef_) == 1:
                return _dense(self.coef_[0])
            raise Exception("Multinomial models contain a matrix of coefficients, use coefficientMatrix instead.")
        raise Exception("coefficients not defined for multi-model instance")

    @property
    def intercept(self) -> float:
        if isinstance(self.intercept_[0], float):
            if len(self.intercept_) == 1:
                return self.intercept_[0]  # type: ignore[return-value]
            raise Exception("Multinomial models contain a vector of intercepts, use interceptVector instead.")
        raise Exception("intercept not defined for multi-model instance")

    @property
    def coefficientMatrix(self) -> Any:
        """pyspark DenseMatrix when pyspark.ml.linalg provides it, else a numpy array [numCoefficientSets, numFeatures]."""
        if isinstance(self.coef_[0][0], float):
            rows, cols = len(self.coef_), len(self.coef_[0])
            flat = [float(c) for row in self.coef_ for c in row]  # type: ignore[union-attr]
            try:
                from pyspark.ml.linalg import DenseMatrix
            except ImportError:
                return np.array(flat, dtype=np.float64).reshape(rows, cols)
            return DenseMatrix(numRows=rows, numCols=cols, values=flat, isTransposed=True)
        raise Exception("coefficientMatrix not defined for multi-model instance")

    @property
    def interceptVector(self) -> Any:
        """Spark's interceptVector.compressed: sparse when 1.5 (nnz + 1) < size (pyspark vectors when available)."""
        if isinstance(self.intercept_[0], float):
            nnz = int(np.count_nonzero(self.intercept_))
            size = len(self.intercept_)
            if 1.5 * (nnz + 1.0) < size:
                try:
                    from pyspark.ml.linalg import Vectors
                except ImportError:
                    return _SparseIntercepts(size, {i: float(v) for i, v in enumerate(self.intercept_) if v != 0})
                return Vectors.sparse(size, {i: float(v) for i, v in enumerate(self.intercept_)})
            return _dense(self.intercept_)  # type: ignore[arg-type]
        raise Exception("interceptVector not defined for multi-model instance")

    @property
    def numClasses(self) -> int:
        return self._num_classes

    @property
    def hasSummary(self) -> bool:
        return False

    @property
    def summary(self) -> Any:
        raise RuntimeError("No training summary available for this %s" % self.__class__.__name__)

    def predict(self, value: Any) -> float:
        raise NotImplementedError("LogisticRegressionModel.predict() of a single vector is not supported; use transform()")

    def predictRaw(self, value: Any) -> Any:
        raise NotImplementedError("LogisticRegressionModel.predictRaw() of a single vector is not supported; use "
                                  "transform()")

    def predictProbability(self, value: Any) -> Any:
        raise NotImplementedError("LogisticRegressionModel.predictProbability() of a single vector is not supported; "
                                  "use transform()")

    def evaluate(self, dataset: Any) -> Any:
        raise NotImplementedError("LogisticRegressionModel.evaluate() is not supported in this build")

    def cpu(self) -> Any:
        raise NotImplementedError("LogisticRegressionModel.cpu() builds a JVM pyspark.ml model; no JVM/pyspark in this "
                                  "build")

    _combined_attrs = ("coef_", "intercept_")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "double"

    def _device_model(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        if self._get_num_models() != 1:
            raise NotImplementedError("transform() of a combined multi-model instance is not supported")
        W = np.asarray(self.coef_, dtype=np.float64)
        b = np.asarray(self.intercept_, dtype=np.float64)
        cls = np.asarray(self.classes_, dtype=np.float64)
        if W.shape[0] == 1 and cls.size == 1:   # one label seen: the binomial model of that label
            cls = np.array([0.0, 1.0])
        return W, b, cls

    def _eval_models(self) -> List[Dict[str, Any]]:
        """Each model of this (combined) instance as b2k_eval_linear takes it, with the class values transform() uses."""
        n = self._get_num_models()
        coefs = [self.coef_] if n == 1 else list(self.coef_)
        icpts = [self.intercept_] if n == 1 else list(self.intercept_)
        out = []
        for c, i in zip(coefs, icpts):
            W = np.asarray(c, dtype=np.float64)
            b = np.asarray(i, dtype=np.float64).reshape(-1)
            cls = np.asarray(self.classes_, dtype=np.float64)
            if W.shape[0] == 1 and cls.size == 1:
                cls = np.array([0.0, 1.0])
            kp = int(W.shape[0])
            out.append({"kind": "logistic" if kp == 1 else "softmax", "W": W, "b": b,
                        "class_values": cls[:2] if kp == 1 else cls[:kp]})
        return out

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        if eval_metric_info is not None:
            from .core import _class_accs

            if not eval_metric_info["classification"]:
                raise NotImplementedError("LogisticRegressionModel is evaluated with a MulticlassClassificationEvaluator")
            models = self._eval_models()
            eps = eval_metric_info["eps"]

            if eval_metric_info["binary"]:
                def _scores(h: Any, X: Any, y: Any, scores: Any, pos: Any, row0: int) -> None:
                    h.ctx.binary_scores_linear(X, y, models, scores, pos, row0)

                _scores.n_models = len(models)  # type: ignore[attr-defined]
                return _DeviceModel, None, _scores  # type: ignore[return-value]

            def _evaluate(h: Any, X: Any, y: Any) -> List[Dict[str, Any]]:
                return _class_accs(h.ctx.eval_linear(X, y, models, eps))

            return _DeviceModel, None, _evaluate  # type: ignore[return-value]
        W, b, cls = self._device_model()
        class_values = cls[:max(2, W.shape[0])]
        out_bytes = 8 * (2 * max(2, W.shape[0]) + 1)
        if isinstance(dataset, LocalDataFrame) and _vector_column(dataset, self.getFeaturesCol()) is not None:
            d = int(self.n_cols)
            transform = self._grouped_transform(lambda m, X: m.ctx.logreg_predict_csr(X, d, W, b, class_values),
                                                8 + out_bytes, sparse=True)
        else:
            transform = self._grouped_transform(lambda m, X: m.ctx.logreg_predict(X, W, b, class_values),
                                                4 * int(self.n_cols) + out_bytes)
        return _DeviceModel, transform, None

    def _transformEvaluate(self, dataset: Any, evaluator: Any, params: Optional[Dict[Any, Any]] = None) -> List[float]:
        if isinstance(dataset, LocalDataFrame) and _vector_column(dataset, self.getFeaturesCol()) is not None:
            raise NotImplementedError("LogisticRegressionModel._transformEvaluate() of sparse input (a vector struct "
                                      "features column) is not supported: the single-pass evaluation kernels read "
                                      "dense rows")
        return super()._transformEvaluate(dataset, evaluator, params)

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        return [(self.getRawPredictionCol(), "array<double>"), (self.getProbabilityCol(), "array<double>"),
                (self.getOrDefault("predictionCol"), "double")]


def _vector_column(dataset: LocalDataFrame, col: Any) -> Optional[str]:
    """The features column when it is a single vector struct column of the frame, else None."""
    if not isinstance(col, str) or dataset.schema is None or col not in dataset.columns:
        return None
    return col if is_vector_struct(dataset.schema.field(col).type) else None


def _dense(values: Sequence[float]) -> Any:
    try:
        from pyspark.ml.linalg import DenseVector
    except ImportError:
        return np.array(values, dtype=np.float64)
    return DenseVector(list(values))


class _SparseIntercepts:
    """A sparse vector (size, {index: value}) without pyspark: toArray() gives the dense values."""

    def __init__(self, size: int, values: Dict[int, float]) -> None:
        self.size = size
        self.values = values

    def toArray(self) -> np.ndarray:
        a = np.zeros(self.size, dtype=np.float64)
        for i, v in self.values.items():
            a[i] = v
        return a


class RandomForestClassifier(_RandomForestEstimator):
    """Random forest classification on H100 (reference classification.py:285-498).  Every tree is grown from the gini
    or entropy histograms of all workers' rows, with one allreduce per histogram pass, so the forest does not depend on
    the number of workers.  Parameters as in the reference: featuresCol (str or list of str), labelCol, predictionCol,
    probabilityCol, rawPredictionCol, maxDepth (5), maxBins (32), minInstancesPerNode (1), minInfoGain (0.0), impurity
    ("gini"), numTrees (20), featureSubsetStrategy ("auto"), seed, bootstrap (True), num_workers, verbose.  Labels are
    the class indices 0, 1, ...; numClasses = max label + 1.

    >>> from spark_rapids_ml_b200.classification import RandomForestClassifier
    >>> df = session.createDataFrame([([1.0, 2.0], 1.0), ([1.0, 3.0], 1.0), ([2.0, 1.0], 0.0), ([3.0, 1.0], 0.0)],
    ...                              "features array<float>, label float")
    >>> RandomForestClassifier(numTrees=3, bootstrap=False).fit(df).transform(df)
    """

    probabilityCol = Param("parent", "probabilityCol", "Column name for predicted class conditional probabilities.",
                           TypeConverters.toString)
    rawPredictionCol = Param("parent", "rawPredictionCol", "raw prediction (a.k.a. confidence) column name.",
                             TypeConverters.toString)

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", labelCol: str = "label",
                 predictionCol: str = "prediction", probabilityCol: str = "probability",
                 rawPredictionCol: str = "rawPrediction", maxDepth: int = 5, maxBins: int = 32,
                 minInstancesPerNode: int = 1, minInfoGain: float = 0.0, maxMemoryInMB: int = 256,
                 cacheNodeIds: bool = False, checkpointInterval: int = 10, impurity: str = "gini", numTrees: int = 20,
                 featureSubsetStrategy: str = "auto", seed: Optional[int] = None, subsamplingRate: float = 1.0,
                 leafCol: str = "", minWeightFractionPerNode: float = 0.0, weightCol: Optional[str] = None,
                 bootstrap: Optional[bool] = True, num_workers: Optional[int] = None, verbose: Union[int, bool] = False,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)

    def _init_defaults(self) -> None:
        self._setDefault(impurity="gini", probabilityCol="probability", rawPredictionCol="rawPrediction")

    def _is_classification(self) -> bool:
        return True

    def _model_class(self) -> Any:
        return RandomForestClassificationModel

    def setProbabilityCol(self, value: str) -> "RandomForestClassifier":
        return self._set_params(probabilityCol=value)

    def setRawPredictionCol(self, value: str) -> "RandomForestClassifier":
        return self._set_params(rawPredictionCol=value)


class RandomForestClassificationModel(_RandomForestModel):
    """reference: classification.py:501-676.  transform() appends rawPredictionCol (the sum of the trees' leaf
    probabilities), probabilityCol (raw normalised) and predictionCol (the class of the largest raw value)."""

    probabilityCol = RandomForestClassifier.probabilityCol
    rawPredictionCol = RandomForestClassifier.rawPredictionCol

    def _init_defaults(self) -> None:
        self._setDefault(impurity="gini", probabilityCol="probability", rawPredictionCol="rawPrediction")

    def _is_classification(self) -> bool:
        return True

    @property
    def numClasses(self) -> int:
        return self._num_classes

    def setProbabilityCol(self, value: str) -> "RandomForestClassificationModel":
        return self._set_params(probabilityCol=value)

    def setRawPredictionCol(self, value: str) -> "RandomForestClassificationModel":
        return self._set_params(rawPredictionCol=value)

    def predictRaw(self, value: Any) -> Any:
        raise NotImplementedError("predictRaw() of a single vector is not supported; use transform()")

    def predictProbability(self, value: Any) -> Any:
        raise NotImplementedError("predictProbability() of a single vector is not supported; use transform()")

    def evaluate(self, dataset: Any) -> Any:
        raise NotImplementedError("RandomForestClassificationModel.evaluate() is not supported in this build")


# ---- MultilayerPerceptronClassifier (pyspark.ml.classification; the reference has no multilayer perceptron) ----
class MultilayerPerceptronClassifierClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        # None = unsupported, "" = accepted and ignored
        return {"layers": "layers", "maxIter": "max_iter", "tol": "tol", "seed": "random_state", "blockSize": "",
                "solver": "solver", "stepSize": "step_size", "initialWeights": "initial_weights", "thresholds": None}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"layers": None, "max_iter": 100, "tol": 1e-6, "random_state": None, "solver": "l-bfgs",
                "step_size": 0.03, "initial_weights": None, "verbose": False}

    def _pyspark_class(self) -> Optional[type]:
        return None  # pyspark.ml.classification.MultilayerPerceptronClassifier when pyspark is installed


def _to_int_list(v: Any) -> List[int]:
    return [int(x) for x in v]


def _to_float_list(v: Any) -> List[float]:
    return [float(x) for x in np.asarray(v, dtype=np.float64).reshape(-1)]


class _MultilayerPerceptronCumlParams(_CumlParams, HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasPredictionCol):
    """Shared Spark Params of MultilayerPerceptronClassifier and its model (Spark's defaults: maxIter=100, tol=1e-6,
    blockSize=128, solver='l-bfgs', stepSize=0.03, rawPredictionCol='rawPrediction', probabilityCol='probability')."""

    layers = Param("parent", "layers", "Sizes of layers from input layer to output layer.", _to_int_list)
    maxIter = Param("parent", "maxIter", "max number of iterations (>= 0).", TypeConverters.toInt)
    tol = Param("parent", "tol", "the convergence tolerance for iterative algorithms (>= 0).", TypeConverters.toFloat)
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    blockSize = Param("parent", "blockSize", "block size for stacking input data in matrices (accepted; the loss is "
                      "averaged over rows).", TypeConverters.toInt)
    solver = Param("parent", "solver", "The solver algorithm for optimization. Supported options: l-bfgs, gd.",
                   TypeConverters.toString)
    stepSize = Param("parent", "stepSize", "Step size to be used for each iteration of optimization (> 0).",
                     TypeConverters.toFloat)
    initialWeights = Param("parent", "initialWeights", "The initial weights of the model.", _to_float_list)
    rawPredictionCol = Param("parent", "rawPredictionCol", "raw prediction (a.k.a. confidence) column name.",
                             TypeConverters.toString)
    probabilityCol = Param("parent", "probabilityCol", "Column name for predicted class conditional probabilities.",
                           TypeConverters.toString)
    thresholds = Param("parent", "thresholds", "Thresholds in multi-class classification (not supported).",
                       _to_float_list)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(maxIter=100, tol=1e-6, blockSize=128, solver="l-bfgs", stepSize=0.03, labelCol="label",
                         predictionCol="prediction", rawPredictionCol="rawPrediction", probabilityCol="probability")
        # the KMeans rule: a 32-bit signed seed from the class name
        self._setDefault(seed=hash(type(self).__name__) & 0x07FFFFFFF)

    def getLayers(self) -> List[int]:
        return list(self.getOrDefault(self.layers))

    def getMaxIter(self) -> int:
        return self.getOrDefault(self.maxIter)

    def getTol(self) -> float:
        return self.getOrDefault(self.tol)

    def getSeed(self) -> int:
        return self.getOrDefault(self.seed)

    def getBlockSize(self) -> int:
        return self.getOrDefault(self.blockSize)

    def getSolver(self) -> str:
        return self.getOrDefault(self.solver)

    def getStepSize(self) -> float:
        return self.getOrDefault(self.stepSize)

    def getInitialWeights(self) -> Optional[List[float]]:
        return list(self.getOrDefault(self.initialWeights)) if self.isDefined(self.initialWeights) else None

    def getRawPredictionCol(self) -> str:
        return self.getOrDefault(self.rawPredictionCol)

    def getProbabilityCol(self) -> str:
        return self.getOrDefault(self.probabilityCol)

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

    def setRawPredictionCol(self: P, value: str) -> P:
        return self._set_params(rawPredictionCol=value)

    def setProbabilityCol(self: P, value: str) -> P:
        return self._set_params(probabilityCol=value)

    def setThresholds(self: P, value: List[float]) -> P:
        raise ValueError("'thresholds' is not supported by MultilayerPerceptronClassifier on the GPU.")


def _mlp_n_weights(layers: Sequence[int]) -> int:
    return sum(int(layers[i]) * (int(layers[i - 1]) + 1) for i in range(1, len(layers)))


def _refuse_pyspark(dataset: Any, who: str) -> None:
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError(f"{who} of a pyspark DataFrame is not supported yet; use a local frame")


class MultilayerPerceptronClassifier(MultilayerPerceptronClassifierClass, _CumlEstimator,
                                     _MultilayerPerceptronCumlParams):
    """Multilayer perceptron classification on H100, Spark's pyspark.ml.classification.MultilayerPerceptronClassifier:
    sigmoid hidden layers, a softmax output layer and the cross-entropy loss, trained by L-BFGS (default) or full-batch
    gradient descent.  Every solver step is one evaluation of the loss and its gradient over the device-resident rows
    (the layer products and the gradient sums on wgmma 3xTF32 when d % 4 == 0, else in fp64) and one NCCL allreduce.
    Parameters: layers (required: [numFeatures, hidden..., numClasses]), maxIter (100), tol (1e-6), seed, blockSize
    (128; accepted, no effect: the loss is averaged over rows, not within blocks), solver ("l-bfgs" | "gd"), stepSize
    (0.03, gd only), initialWeights (Spark's flat layout), featuresCol / featuresCols, labelCol, predictionCol,
    rawPredictionCol, probabilityCol, num_workers, verbose.

    Deliberate differences from Spark: without initialWeights the start comes from the library's seeded generator, not
    XORShiftRandom; a fractional label is an error (Spark truncates it).  thresholds, sparse input, a pyspark DataFrame
    and CrossValidator / fitMultiple in one pass are not supported.

    >>> from spark_rapids_ml_b200.classification import MultilayerPerceptronClassifier
    >>> model = MultilayerPerceptronClassifier(layers=[4, 8, 3], seed=1).fit(df)
    >>> model.transform(df)
    """

    @keyword_only
    def __init__(self, *, featuresCol: Union[str, List[str]] = "features", labelCol: str = "label",
                 predictionCol: str = "prediction", maxIter: int = 100, tol: float = 1e-6, seed: Optional[int] = None,
                 layers: Optional[List[int]] = None, blockSize: int = 128, stepSize: float = 0.03,
                 solver: str = "l-bfgs", initialWeights: Optional[Any] = None, probabilityCol: str = "probability",
                 rawPredictionCol: str = "rawPrediction", thresholds: Optional[List[float]] = None,
                 num_workers: Optional[int] = None, verbose: Union[int, bool] = False, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        for name in ("seed", "num_workers", "layers", "initialWeights", "thresholds"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        if "thresholds" in self._input_kwargs:
            raise ValueError("'thresholds' is not supported by MultilayerPerceptronClassifier on the GPU.")
        if "initialWeights" in self._input_kwargs:
            self._input_kwargs["initialWeights"] = [float(v) for v in np.asarray(self._input_kwargs["initialWeights"],
                                                                                 dtype=np.float64).reshape(-1)]
        self._set_params(**self._input_kwargs)

    def setLayers(self, value: List[int]) -> "MultilayerPerceptronClassifier":
        return self._set_params(layers=value)

    def setMaxIter(self, value: int) -> "MultilayerPerceptronClassifier":
        return self._set_params(maxIter=value)

    def setTol(self, value: float) -> "MultilayerPerceptronClassifier":
        return self._set_params(tol=value)

    def setSeed(self, value: int) -> "MultilayerPerceptronClassifier":
        return self._set_params(seed=value)

    def setBlockSize(self, value: int) -> "MultilayerPerceptronClassifier":
        return self._set_params(blockSize=value)

    def setSolver(self, value: str) -> "MultilayerPerceptronClassifier":
        return self._set_params(solver=value)

    def setStepSize(self, value: float) -> "MultilayerPerceptronClassifier":
        return self._set_params(stepSize=value)

    def setInitialWeights(self, value: Any) -> "MultilayerPerceptronClassifier":
        return self._set_params(initialWeights=[float(v) for v in np.asarray(value, dtype=np.float64).reshape(-1)])

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        if not self.isDefined(self.layers):
            raise ValueError("layers must be set: [numFeatures, hidden layer sizes..., numClasses]")
        layers = self.getLayers()
        if len(layers) < 2:
            raise ValueError(f"layers given invalid value {layers} (must have at least 2 entries)")
        if any(v < 1 for v in layers):
            raise ValueError(f"layers given invalid value {layers} (every entry must be > 0)")
        if self.getMaxIter() < 0:
            raise ValueError(f"maxIter given invalid value {self.getMaxIter()}")
        if not self.getTol() >= 0:
            raise ValueError(f"tol given invalid value {self.getTol()}")
        if self.getBlockSize() < 1:
            raise ValueError(f"blockSize given invalid value {self.getBlockSize()}")
        if self.getSolver() not in ("l-bfgs", "gd"):
            raise ValueError(f"solver given invalid value {self.getSolver()} (supported: l-bfgs, gd)")
        if not self.getStepSize() > 0:
            raise ValueError(f"stepSize given invalid value {self.getStepSize()}")
        w0 = self.getInitialWeights()
        if w0 is not None and len(w0) != _mlp_n_weights(layers):
            raise ValueError(f"initialWeights has {len(w0)} values; layers {layers} need {_mlp_n_weights(layers)}")

    def _fit_label_col(self) -> Optional[str]:
        return self.getLabelCol()

    def _fit_array_order(self) -> str:
        return "C"

    def _fit(self, dataset: Any) -> "MultilayerPerceptronClassificationModel":
        _refuse_pyspark(dataset, "MultilayerPerceptronClassifier.fit")
        if isinstance(dataset, LocalDataFrame) and _vector_column(dataset, self.getFeaturesCol()) is not None:
            raise NotImplementedError("MultilayerPerceptronClassifier on sparse input (a vector struct features column) "
                                      "is not supported")
        self._validate_parameters()
        return super()._fit(dataset)  # type: ignore[return-value]

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        cls = self.__class__
        layers = self.getLayers()
        w0 = self.getInitialWeights()

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            ctx = params[param_alias.handle]
            init = params[param_alias.cuml_init]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            X, y, _ = dfs[0]
            d = params[param_alias.num_cols]
            if layers[0] != d:
                raise ValueError(f"layers[0] = {layers[0]} must equal the number of features {d}")
            seed = init.get("random_state")
            out = ctx.mlp_fit(X, y, layers, solver=str(init["solver"]), max_iter=int(init["max_iter"]),
                              tol=float(init["tol"]), step_size=float(init["step_size"]),
                              seed=int(seed) if seed is not None else 0, initial_weights=w0)
            get_logger(cls).info(f"iterations: {out['n_iter']}, loss: {out['objective_history'][-1:]}")
            return {"weights_": [out["weights"].tolist()], "layers_": [list(layers)],
                    "objective_history_": [out["objective_history"].tolist()],
                    "n_cols": [d], "dtype": ["float32"]}

        return _cuml_fit

    def _out_schema(self) -> Any:
        return "weights_ array<double>, layers_ array<int>, objective_history_ array<double>, n_cols int, dtype string"

    def _create_pyspark_model(self, result: Row) -> "MultilayerPerceptronClassificationModel":
        r = result.asDict()
        return MultilayerPerceptronClassificationModel(
            weights_=[float(v) for v in r["weights_"]], layers_=[int(v) for v in r["layers_"]],
            objective_history_=[float(v) for v in r["objective_history_"]], n_cols=int(r["n_cols"]),
            dtype=str(r["dtype"]))


class MultilayerPerceptronClassificationTrainingSummary:
    """The training summary Spark's MultilayerPerceptronClassificationModel.summary() holds: objectiveHistory (F at
    each accepted iterate) and totalIterations (its length, as Spark reports it)."""

    def __init__(self, objective_history: List[float]) -> None:
        self.objectiveHistory = list(objective_history)
        self.totalIterations = len(objective_history)


class MultilayerPerceptronClassificationModel(MultilayerPerceptronClassifierClass, _CumlModelWithPredictionCol,
                                              _MultilayerPerceptronCumlParams):
    """transform() appends rawPredictionCol (the last layer's affine output, a double vector), probabilityCol (its
    softmax) and predictionCol (the index of the largest raw value, the lower one on a tie, a double)."""

    def __init__(self, weights_: List[float], layers_: List[int], objective_history_: List[float], n_cols: int,
                 dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype, weights_=weights_, layers_=layers_,
                         objective_history_=objective_history_)
        self.weights_ = weights_
        self.layers_ = layers_
        self.objective_history_ = objective_history_
        self._set_params(layers=list(layers_))

    @property
    def weights(self) -> Any:
        return _dense(self.weights_)

    @property
    def numFeatures(self) -> int:
        return int(self.layers_[0])

    @property
    def numClasses(self) -> int:
        return int(self.layers_[-1])

    @property
    def hasSummary(self) -> bool:
        return True

    def summary(self) -> MultilayerPerceptronClassificationTrainingSummary:
        return MultilayerPerceptronClassificationTrainingSummary(self.objective_history_)

    def predict(self, value: Any) -> float:
        raise NotImplementedError("MultilayerPerceptronClassificationModel.predict() of a single vector is not "
                                  "supported; use transform()")

    def predictRaw(self, value: Any) -> Any:
        raise NotImplementedError("MultilayerPerceptronClassificationModel.predictRaw() of a single vector is not "
                                  "supported; use transform()")

    def predictProbability(self, value: Any) -> Any:
        raise NotImplementedError("MultilayerPerceptronClassificationModel.predictProbability() of a single vector is "
                                  "not supported; use transform()")

    def cpu(self) -> Any:
        raise NotImplementedError("MultilayerPerceptronClassificationModel.cpu() builds a JVM pyspark.ml model; no "
                                  "JVM/pyspark in this build")

    def _transform_array_order(self) -> str:
        return "C"

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        return [(self.getRawPredictionCol(), "array<double>"), (self.getProbabilityCol(), "array<double>"),
                (self.getOrDefault("predictionCol"), "double")]

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        _refuse_pyspark(dataset, "MultilayerPerceptronClassificationModel.transform")
        if isinstance(dataset, LocalDataFrame) and _vector_column(dataset, self.getFeaturesCol()) is not None:
            raise NotImplementedError("MultilayerPerceptronClassificationModel.transform of sparse input (a vector "
                                      "struct features column) is not supported")
        layers = list(self.layers_)
        w = np.asarray(self.weights_, dtype=np.float64)
        C = layers[-1]
        return _DeviceModel, self._grouped_transform(lambda m, X: m.ctx.mlp_predict(X, layers, w),
                                                     4 * int(self.n_cols) + 8 * (2 * C + 1)), None
