"""Local stand-ins for pyspark.ml.evaluation's MulticlassClassificationEvaluator, RegressionEvaluator and
BinaryClassificationEvaluator: Spark's params, defaults and isLargerBetter(); evaluate() of a local frame reads the
label, prediction (probability, rawPrediction) columns and computes in fp64 on the host (spark_rapids_ml_b200.metrics)."""
from __future__ import annotations

from typing import Any, Dict, Optional

import numpy as np

from .params import Param, Params, TypeConverters, keyword_only


class _Evaluator(Params):
    labelCol = Param("parent", "labelCol", "label column name.", TypeConverters.toString)
    predictionCol = Param("parent", "predictionCol", "prediction column name.", TypeConverters.toString)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)
    metricName = Param("parent", "metricName", "metric name in evaluation", TypeConverters.toString)

    def _init(self, kwargs: Dict[str, Any]) -> None:
        super().__init__()
        self._setDefault(labelCol="label", predictionCol="prediction")
        self._set(**{k: v for k, v in kwargs.items() if v is not None})

    def getLabelCol(self) -> str:
        return self.getOrDefault("labelCol")

    def getPredictionCol(self) -> str:
        return self.getOrDefault("predictionCol")

    def getMetricName(self) -> str:
        return self.getOrDefault("metricName")

    def setMetricName(self, value: str) -> "_Evaluator":
        return self._set(metricName=value)

    def setLabelCol(self, value: str) -> "_Evaluator":
        return self._set(labelCol=value)

    def setPredictionCol(self, value: str) -> "_Evaluator":
        return self._set(predictionCol=value)

    def _column(self, dataset: Any, name: str) -> Any:
        if self.isSet("weightCol") and self.getOrDefault("weightCol"):
            raise NotImplementedError("weightCol is not supported by this evaluator")
        return dataset.select(name).toPandas()[name]

    def evaluate(self, dataset: Any, params: Optional[Dict[Param, Any]] = None) -> float:
        return (self.copy(params) if params else self)._evaluate(dataset)

    def _evaluate(self, dataset: Any) -> float:
        raise NotImplementedError

    def isLargerBetter(self) -> bool:
        raise NotImplementedError


class MulticlassClassificationEvaluator(_Evaluator):
    """pyspark.ml.evaluation.MulticlassClassificationEvaluator: metricName (default "f1"), metricLabel (0.0), beta
    (1.0), eps (1e-15, logLoss), probabilityCol ("probability")."""

    metricLabel = Param("parent", "metricLabel", "The class whose metric will be computed in truePositiveRateByLabel|"
                        "falsePositiveRateByLabel|precisionByLabel|recallByLabel|fMeasureByLabel.",
                        TypeConverters.toFloat)
    beta = Param("parent", "beta", "The beta value used in weightedFMeasure|fMeasureByLabel.", TypeConverters.toFloat)
    eps = Param("parent", "eps", "log-loss is undefined for p=0, so the probability of the label is clipped "
                "below at eps: -log(max(p, eps)).", TypeConverters.toFloat)
    probabilityCol = Param("parent", "probabilityCol", "Column name for predicted class conditional probabilities.",
                           TypeConverters.toString)

    @keyword_only
    def __init__(self, *, predictionCol: str = "prediction", labelCol: str = "label", metricName: str = "f1",
                 weightCol: Optional[str] = None, metricLabel: float = 0.0, beta: float = 1.0,
                 probabilityCol: str = "probability", eps: float = 1e-15) -> None:
        self._init({})
        self._setDefault(metricName="f1", metricLabel=0.0, beta=1.0, eps=1e-15, probabilityCol="probability")
        self._set(**{k: v for k, v in self._input_kwargs.items() if v is not None})

    def getMetricLabel(self) -> float:
        return self.getOrDefault("metricLabel")

    def getBeta(self) -> float:
        return self.getOrDefault("beta")

    def getEps(self) -> float:
        return self.getOrDefault("eps")

    def getProbabilityCol(self) -> str:
        return self.getOrDefault("probabilityCol")

    def isLargerBetter(self) -> bool:
        return self.getMetricName() not in ("weightedFalsePositiveRate", "falsePositiveRateByLabel", "logLoss",
                                            "hammingLoss")

    def _evaluate(self, dataset: Any) -> float:
        from .. import metrics

        name = self.getMetricName()
        if name not in metrics.MULTICLASS_METRICS:
            raise ValueError(f"Unsupported metric name, found {name}")
        y = np.asarray(self._column(dataset, self.getLabelCol()), dtype=np.float64)
        p = np.asarray(self._column(dataset, self.getPredictionCol()), dtype=np.float64)
        probs = None
        if name == "logLoss":
            col = list(self._column(dataset, self.getProbabilityCol()))
            probs = np.asarray([np.asarray(v, dtype=np.float64) for v in col]) if col else np.zeros((0, 1))
        acc = metrics.class_accumulators(y, p, probs, self.getEps())
        return metrics.multiclass_metric(acc, name, self.getMetricLabel(), self.getBeta())


class RegressionEvaluator(_Evaluator):
    """pyspark.ml.evaluation.RegressionEvaluator: metricName (default "rmse"), throughOrigin (False)."""

    throughOrigin = Param("parent", "throughOrigin", "whether the regression is through the origin.",
                          TypeConverters.identity)

    @keyword_only
    def __init__(self, *, predictionCol: str = "prediction", labelCol: str = "label", metricName: str = "rmse",
                 weightCol: Optional[str] = None, throughOrigin: bool = False) -> None:
        self._init({})
        self._setDefault(metricName="rmse", throughOrigin=False)
        self._set(**{k: v for k, v in self._input_kwargs.items() if v is not None})

    def getThroughOrigin(self) -> bool:
        return bool(self.getOrDefault("throughOrigin"))

    def isLargerBetter(self) -> bool:
        return self.getMetricName() in ("r2", "var")

    def _evaluate(self, dataset: Any) -> float:
        from .. import metrics

        name = self.getMetricName()
        if name not in metrics.REGRESSION_METRICS:
            raise ValueError(f"Unsupported metric name, found {name}")
        y = np.asarray(self._column(dataset, self.getLabelCol()), dtype=np.float64)
        p = np.asarray(self._column(dataset, self.getPredictionCol()), dtype=np.float64)
        return metrics.regression_metric(metrics.reg_accumulators(y, p), name, self.getThroughOrigin())


class BinaryClassificationEvaluator(_Evaluator):
    """pyspark.ml.evaluation.BinaryClassificationEvaluator: metricName ("areaUnderROC" default, or "areaUnderPR"),
    rawPredictionCol ("rawPrediction"), numBins (1000, >= 0).  The score of a row is element 1 of a vector
    rawPrediction, or the value of a double one; the row is positive when its label > 0.5.  Spark down-samples the
    curve to numBins points per partition of its sorted scores; here the whole ordered list is one partition, so with
    numBins > 0 and more than 2 numBins distinct scores the value can differ from Spark's on a multi-partition RDD."""

    rawPredictionCol = Param("parent", "rawPredictionCol", "raw prediction (a.k.a. confidence) column name.",
                             TypeConverters.toString)
    numBins = Param("parent", "numBins", "Number of bins to down-sample the curves (ROC curve, PR curve) in area "
                    "computation. If 0, no down-sampling will occur. Must be >= 0.", TypeConverters.toInt)

    @keyword_only
    def __init__(self, *, rawPredictionCol: str = "rawPrediction", labelCol: str = "label",
                 metricName: str = "areaUnderROC", weightCol: Optional[str] = None, numBins: int = 1000) -> None:
        self._init({})
        self._setDefault(metricName="areaUnderROC", rawPredictionCol="rawPrediction", numBins=1000)
        self._set(**{k: v for k, v in self._input_kwargs.items() if v is not None})

    def _set(self, **kwargs: Any) -> "BinaryClassificationEvaluator":
        if kwargs.get("numBins") is not None and TypeConverters.toInt(kwargs["numBins"]) < 0:
            raise ValueError(f"numBins must be >= 0, got {kwargs['numBins']}")
        return super()._set(**kwargs)

    def getRawPredictionCol(self) -> str:
        return self.getOrDefault("rawPredictionCol")

    def setRawPredictionCol(self, value: str) -> "BinaryClassificationEvaluator":
        return self._set(rawPredictionCol=value)

    def getNumBins(self) -> int:
        return int(self.getOrDefault("numBins"))

    def setNumBins(self, value: int) -> "BinaryClassificationEvaluator":
        return self._set(numBins=value)

    def isLargerBetter(self) -> bool:
        return True

    def _evaluate(self, dataset: Any) -> float:
        from .. import metrics

        name = self.getMetricName()
        if name not in metrics.BINARY_METRICS:
            raise ValueError(f"Unsupported metric name, found {name}")
        y = np.asarray(self._column(dataset, self.getLabelCol()), dtype=np.float64)
        raw = list(self._column(dataset, self.getRawPredictionCol()))
        if raw and np.ndim(raw[0]) == 0:
            s = np.asarray(raw, dtype=np.float64)
        else:
            if any(len(v) < 2 for v in raw):
                raise ValueError(f"{self.getRawPredictionCol()} holds a vector of fewer than 2 elements: the binary "
                                 "score is element 1")
            s = np.asarray([v[1] for v in raw], dtype=np.float64)
        return metrics.binary_metric(s, y, name, self.getNumBins())


class ClusteringEvaluator(_Evaluator):
    """pyspark.ml.evaluation.ClusteringEvaluator's params: featuresCol ("features"), predictionCol ("prediction"),
    metricName ("silhouette", the only one), distanceMeasure ("squaredEuclidean" or "cosine"), weightCol.  Values
    outside those sets raise ValueError with Spark's ParamValidators wording.  evaluate() is spark_rapids_ml_b200.
    evaluation.ClusteringEvaluator's (on the device)."""

    featuresCol = Param("parent", "featuresCol", "features column name.", TypeConverters.identity)
    distanceMeasure = Param("parent", "distanceMeasure", "The distance measure. Supported options: "
                            "'squaredEuclidean' and 'cosine'.", TypeConverters.toString)
    _ALLOWED = {"metricName": ("silhouette",), "distanceMeasure": ("squaredEuclidean", "cosine")}

    @keyword_only
    def __init__(self, *, predictionCol: str = "prediction", featuresCol: Any = "features",
                 metricName: str = "silhouette", distanceMeasure: str = "squaredEuclidean",
                 weightCol: Optional[str] = None) -> None:
        self._init({})
        self._setDefault(featuresCol="features", metricName="silhouette", distanceMeasure="squaredEuclidean")
        self._set(**{k: v for k, v in self._input_kwargs.items() if v is not None})

    def _set(self, **kwargs: Any) -> "ClusteringEvaluator":
        for name, allowed in self._ALLOWED.items():
            v = kwargs.get(name)
            if v is not None and v not in allowed:
                raise ValueError(f"{self.uid} parameter {name} given invalid value {v}.")
        return super()._set(**kwargs)

    def getFeaturesCol(self) -> Any:
        return self.getOrDefault("featuresCol")

    def setFeaturesCol(self, value: Any) -> "ClusteringEvaluator":
        return self._set(featuresCol=value)

    def getDistanceMeasure(self) -> str:
        return self.getOrDefault("distanceMeasure")

    def setDistanceMeasure(self, value: str) -> "ClusteringEvaluator":
        return self._set(distanceMeasure=value)

    def setWeightCol(self, value: str) -> "ClusteringEvaluator":
        return self._set(weightCol=value)

    def isLargerBetter(self) -> bool:
        return True
