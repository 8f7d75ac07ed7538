"""The shared base of RandomForestClassifier / RandomForestRegressor (reference python/src/spark_rapids_ml/tree.py),
with cuML's per-worker forests replaced by libb2kmeans' b2k_rf_fit: every tree is grown from the exact integer
histograms of ALL workers' rows, level by level, with one allreduce per histogram pass (MLlib's design), so the forest
depends only on the rows in partition order and the params, not on the number of workers.  The semantics are written
in include/b2kmeans.h ("random forests") and DESIGN.md §15.

  _RandomForestClass (param and value mappings, cuML defaults)          tree.py:91-153
  _RandomForestCumlParams / _RandomForestEstimatorParams (setters)      tree.py:156-311
  _RandomForestEstimator (fit function, fitMultiple)                    tree.py:314-527
  _RandomForestModel (model_json, transform, persistence)               tree.py:530-

Models keep the forest as treelite-shaped JSON (model_json: {"trees": [{"num_nodes", "nodes": [...]}]}), the layout the
reference's utils.py:694-809 reads.  No treelite bytes are written, so the reference cannot load a model saved here; a
model the reference saved loads here through its model_json.  cpu(), trees, toDebugString, predict(), predictLeaf() and
transform() of a pyspark DataFrame raise NotImplementedError; weightCol and leafCol raise ValueError.
"""
from __future__ import annotations

import json
import math
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np

from .core import (FitInputType, _CumlModelWithPredictionCol, _DeviceModel, _TunedEstimator, _no_spark_transform,
                   param_alias)
from .params import HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasPredictionCol, P, _CumlClass, _CumlParams
from .sparkshim import Param, Row, TypeConverters

MAX_DEPTH = 16          # b2k_rf_fit's limit
MAX_BINS = (2, 256)     # bins are uint8


class _RandomForestClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {
            "maxBins": "n_bins",
            "maxDepth": "max_depth",
            "numTrees": "n_estimators",
            "impurity": "split_criterion",
            "featureSubsetStrategy": "max_features",
            "bootstrap": "bootstrap",
            "seed": "random_state",
            "minInstancesPerNode": "min_samples_leaf",
            "minInfoGain": "",
            "maxMemoryInMB": "",
            "cacheNodeIds": "",
            "checkpointInterval": "",
            "subsamplingRate": "",
            "minWeightFractionPerNode": "",
            "weightCol": None,
            "leafCol": None,
        }

    @classmethod
    def _param_value_mapping(cls) -> Dict[str, Callable[[Any], Union[None, str, float, int]]]:
        def _tree_mapping(feature_subset: str) -> Union[None, str, float, int]:
            num = _str_or_numerical(feature_subset)
            if isinstance(num, (int, float)):
                return num
            return {"onethird": 1 / 3.0, "all": 1.0, "auto": "auto", "sqrt": "sqrt", "log2": "log2"}.get(num, None)

        return {"max_features": _tree_mapping,
                "split_criterion": lambda v: {"gini": "gini", "entropy": "entropy", "variance": "mse"}.get(v, None)}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_streams": 4, "n_estimators": 100, "max_depth": 16, "max_features": "sqrt", "n_bins": 128,
                "bootstrap": True, "verbose": False, "min_samples_leaf": 1, "min_samples_split": 2, "max_samples": 1.0,
                "max_leaves": -1, "min_impurity_decrease": 0.0, "random_state": None, "max_batch_size": 4096}

    def _pyspark_class(self) -> Optional[type]:
        return None


def _str_or_numerical(s: str) -> Union[str, float, int]:
    """reference utils.py: '3' -> 3, '0.5' -> 0.5, anything else stays a string."""
    try:
        return int(s)
    except ValueError:
        try:
            return float(s)
        except ValueError:
            return s


class _RandomForestParams(HasFeaturesCol, HasLabelCol, HasPredictionCol):
    """pyspark.ml.tree._RandomForestParams stand-in, with Spark's defaults."""

    maxDepth = Param("parent", "maxDepth", "Maximum depth of the tree. (>= 0)", TypeConverters.toInt)
    maxBins = Param("parent", "maxBins", "Max number of bins for discretizing continuous features. Must be >=2.",
                    TypeConverters.toInt)
    minInstancesPerNode = Param("parent", "minInstancesPerNode", "Minimum number of instances each child must have "
                                "after split.", TypeConverters.toInt)
    minWeightFractionPerNode = Param("parent", "minWeightFractionPerNode", "Minimum fraction of the weighted sample "
                                     "count that each child must have after split.", TypeConverters.toFloat)
    minInfoGain = Param("parent", "minInfoGain", "Minimum information gain for a split to be considered at a tree "
                        "node.", TypeConverters.toFloat)
    maxMemoryInMB = Param("parent", "maxMemoryInMB", "Maximum memory in MB allocated to histogram aggregation.",
                          TypeConverters.toInt)
    cacheNodeIds = Param("parent", "cacheNodeIds", "If false, the algorithm will pass trees to executors to match "
                         "instances with nodes.")
    checkpointInterval = Param("parent", "checkpointInterval", "set checkpoint interval (>= 1) or disable checkpoint "
                               "(-1).", TypeConverters.toInt)
    impurity = Param("parent", "impurity", "Criterion used for information gain calculation (case-insensitive).",
                     TypeConverters.toString)
    numTrees = Param("parent", "numTrees", "Number of trees to train (>= 1).", TypeConverters.toInt)
    featureSubsetStrategy = Param("parent", "featureSubsetStrategy", "The number of features to consider for splits at "
                                  "each tree node.", TypeConverters.toString)
    subsamplingRate = Param("parent", "subsamplingRate", "Fraction of the training data used for learning each "
                            "decision tree, in range (0, 1].", TypeConverters.toFloat)
    bootstrap = Param("parent", "bootstrap", "Whether bootstrap samples are used when building trees.")
    seed = Param("parent", "seed", "random seed.", TypeConverters.toInt)
    weightCol = Param("parent", "weightCol", "weight column name.", TypeConverters.toString)
    leafCol = Param("parent", "leafCol", "Leaf indices column name.", TypeConverters.toString)

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(labelCol="label", maxDepth=5, maxBins=32, minInstancesPerNode=1, minWeightFractionPerNode=0.0,
                         minInfoGain=0.0, maxMemoryInMB=256, cacheNodeIds=False, checkpointInterval=10, numTrees=20,
                         featureSubsetStrategy="auto", subsamplingRate=1.0, bootstrap=True, leafCol="")

    def getMaxDepth(self) -> int:
        return self.getOrDefault(self.maxDepth)

    def getMaxBins(self) -> int:
        return self.getOrDefault(self.maxBins)

    def getMinInstancesPerNode(self) -> int:
        return self.getOrDefault(self.minInstancesPerNode)

    def getMinInfoGain(self) -> float:
        return self.getOrDefault(self.minInfoGain)

    def getImpurity(self) -> str:
        return self.getOrDefault(self.impurity)

    def getFeatureSubsetStrategy(self) -> str:
        return self.getOrDefault(self.featureSubsetStrategy)

    def getBootstrap(self) -> bool:
        return self.getOrDefault(self.bootstrap)

    def getSeed(self) -> int:
        return self.getOrDefault(self.seed)


class _RandomForestCumlParams(_CumlParams, _RandomForestParams, HasFeaturesCols):
    """Shared Spark Params of the estimators and models (reference: tree.py:156-255)."""

    def __init__(self) -> None:
        super().__init__()
        # restrict the default seed to a 32-bit signed integer, as the reference does
        self._setDefault(seed=_stable_hash(type(self).__name__) & 0x07FFFFFFF)
        self._init_defaults()

    def _init_defaults(self) -> None:
        """The defaults that differ between classification and regression (impurity, output columns)."""

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
        self._set(labelCol=value)
        return self

    def setPredictionCol(self: P, value: str) -> P:
        self._set(predictionCol=value)
        return self


def _stable_hash(s: str) -> int:
    """A process-independent string hash (Python's hash() of a str is salted per process)."""
    h = 0
    for ch in s.encode():
        h = (h * 31 + ch) & 0xFFFFFFFF
    return h


def features_per_node(strategy: str, d: int, n_trees: int, classification: bool) -> int:
    """MLlib's featureSubsetStrategy sizes: auto = all for one tree, else sqrt (classification) or onethird
    (regression); sqrt = ceil(sqrt d); log2 = max(1, ceil(log2 d)); onethird = ceil(d / 3); all = d; an integer n =
    min(n, d); a fraction f in (0, 1] = ceil(f d)."""
    s = str(strategy).lower()
    if s == "auto":
        s = "all" if n_trees == 1 else ("sqrt" if classification else "onethird")
    fixed = {"all": d, "sqrt": int(math.ceil(math.sqrt(d))), "log2": max(1, int(math.ceil(math.log2(d)))),
             "onethird": int(math.ceil(d / 3.0))}
    if s in fixed:
        return fixed[s]
    v = _str_or_numerical(s)
    if isinstance(v, int) and v >= 1:
        return min(v, d)
    if isinstance(v, float) and 0.0 < v <= 1.0:
        return int(math.ceil(v * d))
    raise ValueError(f"featureSubsetStrategy given invalid value {strategy}")


class _RandomForestEstimator(_RandomForestClass, _TunedEstimator, _RandomForestCumlParams):
    """The shared estimator: one barrier task per GPU ingests its partition; b2k_rf_fit grows every tree over all
    partitions' rows."""

    def __init__(self, **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        kwargs = dict(self._input_kwargs, **kwargs)
        kwargs.pop("kwargs", None)
        if kwargs.get("num_workers", None) is None:
            kwargs.pop("num_workers", None)
        for bad in ("weightCol", "leafCol"):
            if kwargs.get(bad):
                raise ValueError(f"'{bad}' is not supported by cuML.")
        self._set_params(**kwargs)
        if "n_streams" not in kwargs:
            self._set_cuml_value("n_streams", 1)

    # every map is fitted from one ingest, with its own label pass and histogram passes
    _single_pass_params = frozenset(("maxDepth", "maxBins", "minInstancesPerNode", "minInfoGain", "impurity",
                                     "numTrees", "featureSubsetStrategy", "bootstrap", "seed"))

    def _is_classification(self) -> bool:
        raise NotImplementedError

    def setBootstrap(self: P, value: bool) -> P:
        return self._set_params(bootstrap=value)

    def setFeatureSubsetStrategy(self: P, value: str) -> P:
        return self._set_params(featureSubsetStrategy=value)

    def setImpurity(self: P, value: str) -> P:
        return self._set_params(impurity=value)

    def setMaxBins(self: P, value: int) -> P:
        return self._set_params(maxBins=value)

    def setMaxDepth(self: P, value: int) -> P:
        return self._set_params(maxDepth=value)

    def setMinInstancesPerNode(self: P, value: int) -> P:
        return self._set_params(minInstancesPerNode=value)

    def setMinInfoGain(self: P, value: float) -> P:
        return self._set_params(minInfoGain=value)

    def setNumTrees(self: P, value: int) -> P:
        return self._set_params(numTrees=value)

    def setSeed(self: P, value: int) -> P:
        if value > 0x07FFFFFFF:
            raise ValueError("cuML seed value must be a 32-bit integer.")
        return self._set_params(seed=value)

    def setWeightCol(self, value: str) -> Any:
        raise ValueError("'weightCol' is not supported by cuML.")

    def setLeafCol(self, value: str) -> Any:
        raise ValueError("'leafCol' is not supported by cuML.")

    def _settings(self) -> Dict[str, Any]:
        imp = str(self.getImpurity()).lower()
        allowed = ("gini", "entropy") if self._is_classification() else ("variance",)
        if imp not in allowed:
            raise ValueError(f"impurity given invalid value {self.getImpurity()}")
        return {"n_trees": int(self.getOrDefault("numTrees")), "max_depth": int(self.getMaxDepth()),
                "max_bins": int(self.getMaxBins()), "min_instances": int(self.getMinInstancesPerNode()),
                "min_info_gain": float(self.getMinInfoGain()), "impurity": imp,
                "strategy": str(self.getFeatureSubsetStrategy()), "bootstrap": bool(self.getBootstrap()),
                "seed": int(self.getSeed())}

    def _validate_parameters(self) -> None:
        super()._validate_parameters()
        _check_settings(self._settings())

    def _fit_label_col(self) -> Optional[str]:
        return self.getLabelCol()

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        grid = self._fit_grid or [self._settings()]
        classification = self._is_classification()

        def _rf_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for the per-worker cuML fits and the treelite concatenation of tree.py:343-507; one ingest
            # serves every param map
            ctx = params[param_alias.handle]
            if len(dfs) != 1:
                raise RuntimeError("the worker scaffold hands the fit function ONE device matrix per partition")
            X, y, _ = dfs[0]
            d = int(X.shape[1])
            out: Dict[str, List[Any]] = {"n_cols": [], "dtype": [], "model_json": []}
            if classification:
                out["num_classes"] = []
            for s in grid:
                k = features_per_node(s["strategy"], d, s["n_trees"], classification)
                f = ctx.rf_fit(X, y, n_trees=s["n_trees"], max_depth=s["max_depth"], max_bins=s["max_bins"],
                               min_instances=s["min_instances"], features_per_node=k, bootstrap=s["bootstrap"],
                               impurity=s["impurity"], min_info_gain=s["min_info_gain"], seed=s["seed"])
                out["n_cols"].append(params[param_alias.num_cols])
                out["dtype"].append("float32")
                out["model_json"].append(forest_to_json(f, classification))
                if classification:
                    out["num_classes"].append(int(f["n_values"]))
            return out

        return _rf_fit

    def _out_schema(self) -> Any:
        return "n_cols int, dtype string, model_json string" + (", num_classes int" if self._is_classification() else "")

    def _require_nccl_ucx(self) -> Tuple[bool, bool]:
        return (True, False)

    def _supportsTransformEvaluate(self, evaluator: Any) -> bool:
        from .core import _supports_transform_evaluate

        return _supports_transform_evaluate(self._is_classification(), evaluator)

    def _model_class(self) -> Any:
        raise NotImplementedError

    def _create_pyspark_model(self, result: Row) -> Any:
        r = result.asDict()
        kw = {"n_cols": int(r["n_cols"]), "dtype": str(r["dtype"]), "model_json": r["model_json"]}
        if self._is_classification():
            kw["num_classes"] = int(r["num_classes"])
        return self._model_class()(**kw)


def _check_settings(s: Dict[str, Any]) -> None:
    """The errors b2k_rf_fit would return for the params, raised on the driver before any task starts."""
    if s["max_depth"] < 0:
        raise ValueError(f"maxDepth given invalid value {s['max_depth']}")
    if s["max_depth"] > MAX_DEPTH:
        raise ValueError(f"maxDepth given invalid value {s['max_depth']}: this build supports maxDepth <= {MAX_DEPTH}")
    if not MAX_BINS[0] <= s["max_bins"] <= MAX_BINS[1]:
        raise ValueError(f"maxBins given invalid value {s['max_bins']}")
    if s["n_trees"] < 1:
        raise ValueError(f"numTrees given invalid value {s['n_trees']}")
    if s["min_instances"] < 1:
        raise ValueError(f"minInstancesPerNode given invalid value {s['min_instances']}")
    if not (math.isfinite(s["min_info_gain"]) and s["min_info_gain"] >= 0):
        raise ValueError(f"minInfoGain given invalid value {s['min_info_gain']}")
    features_per_node(s["strategy"], 1, s["n_trees"], True)


# ---- the forest as treelite-shaped JSON, and back to flat arrays ----
def forest_to_json(f: Dict[str, Any], classification: bool) -> str:
    trees = []
    off = f["tree_offsets"]
    for t in range(len(off) - 1):
        nodes = []
        for i in range(int(off[t]), int(off[t + 1])):
            j = i - int(off[t])
            feat = int(f["feature"][i])
            if feat >= 0:
                nodes.append({"node_id": j, "split_feature_id": feat, "default_left": True, "split_type": "numerical",
                              "comparison_op": "<=", "threshold": float(f["threshold"][i]),
                              "left_child": int(f["children"][i][0]), "right_child": int(f["children"][i][1]),
                              "gain": float(f["gain"][i]), "instance_count": int(f["count"][i])})
            else:
                v = f["value"][i]
                nodes.append({"node_id": j, "leaf_value": [float(x) for x in v] if classification else float(v[0]),
                              "instance_count": int(f["count"][i])})
        trees.append({"num_nodes": len(nodes), "nodes": nodes})
    return json.dumps({"trees": trees})


def json_to_forest(model_json: str, n_values: int) -> Dict[str, Any]:
    """Flat arrays (as Context.rf_fit returns them) from model_json; node_id need not follow the array order.  A "<"
    split (a reference-written model) becomes "<=" at the largest float32 below its threshold; any other operator is
    rejected."""
    trees = json.loads(model_json)["trees"]
    feat: List[int] = []
    thr: List[float] = []
    ch: List[Tuple[int, int]] = []
    gain: List[float] = []
    cnt: List[int] = []
    val: List[List[float]] = []
    off = [0]
    for tr in trees:
        nodes = sorted(tr["nodes"], key=lambda nd: int(nd["node_id"]))
        for i, nd in enumerate(nodes):
            if int(nd["node_id"]) != i:
                raise ValueError("model_json: node ids of a tree must be 0..num_nodes-1")
            if "leaf_value" in nd:
                lv = nd["leaf_value"]
                lv = [float(x) for x in lv] if isinstance(lv, list) else [float(lv)]
                if len(lv) != n_values:
                    raise ValueError(f"model_json: a leaf holds {len(lv)} values, expected {n_values}")
                feat.append(-1)
                thr.append(0.0)
                ch.append((-1, -1))
                gain.append(0.0)
                val.append(lv)
            else:
                op = nd.get("comparison_op", "<=")
                t32 = np.float32(nd["threshold"])
                if op == "<":
                    t32 = np.nextafter(t32, np.float32(-np.inf))   # x < t  <=>  x <= the float32 below t
                elif op != "<=":
                    raise ValueError(f"model_json: unsupported comparison_op {op!r} (only '<=' and '<' are read)")
                feat.append(int(nd["split_feature_id"]))
                thr.append(float(t32))
                ch.append((int(nd["left_child"]), int(nd["right_child"])))
                gain.append(float(nd.get("gain", 0.0)))
                val.append([0.0] * n_values)
            cnt.append(int(nd.get("instance_count", 0)))
        off.append(len(feat))
    return {"tree_offsets": np.array(off, dtype=np.int64), "feature": np.array(feat, dtype=np.int32),
            "threshold": np.array(thr, dtype=np.float32), "children": np.array(ch, dtype=np.int32).reshape(-1, 2),
            "gain": np.array(gain, dtype=np.float64), "count": np.array(cnt, dtype=np.int64),
            "value": np.array(val, dtype=np.float64).reshape(-1, n_values)}


class _RandomForestModel(_RandomForestClass, _CumlModelWithPredictionCol, _RandomForestCumlParams):
    """The shared model: model_json (treelite-shaped), n_cols, dtype (and num_classes for classification)."""

    def __init__(self, n_cols: int, dtype: str, model_json: Union[str, List[str]] = "", num_classes: int = -1,
                 treelite_model: Any = None) -> None:
        attrs: Dict[str, Any] = {"model_json": model_json}
        if self._is_classification():
            attrs["num_classes"] = num_classes
        super().__init__(dtype=dtype, n_cols=n_cols, **attrs)
        self._num_classes = num_classes
        self._model_json = model_json
        self._forest: Optional[Dict[str, Any]] = None

    def _is_classification(self) -> bool:
        raise NotImplementedError

    def _flat(self) -> Dict[str, Any]:
        if not isinstance(self._model_json, str):
            raise NotImplementedError("a combined multi-model instance holds several forests; transform one model")
        if self._forest is None:
            self._forest = json_to_forest(self._model_json, self._num_classes if self._is_classification() else 1)
        return self._forest

    def cpu(self) -> Any:
        raise NotImplementedError("cpu() builds a JVM pyspark.ml model; no JVM/pyspark in this build")

    @property
    def trees(self) -> Any:
        raise NotImplementedError("trees are JVM DecisionTree models; no JVM/pyspark in this build")

    @property
    def toDebugString(self) -> str:
        raise NotImplementedError("toDebugString needs the JVM model; no JVM/pyspark in this build")

    def predict(self, value: Any) -> float:
        raise NotImplementedError("predict() of a single vector is not supported; use transform()")

    def predictLeaf(self, value: Any) -> float:
        raise NotImplementedError("predictLeaf() is not supported; use transform()")

    @property
    def getNumTrees(self) -> int:
        """Number of trees in the ensemble."""
        return int(len(self._flat()["tree_offsets"]) - 1)

    @property
    def treeWeights(self) -> List[float]:
        return [1.0] * self.getNumTrees

    @property
    def totalNumNodes(self) -> int:
        return int(self._flat()["tree_offsets"][-1])

    @property
    def featureImportances(self) -> Any:
        """MLlib's rule: each split adds gain * instance count to its feature, each tree's vector is normalised to sum
        to 1, and the trees' sum is normalised (a pyspark DenseVector when available, else a numpy array)."""
        f = self._flat()
        d = int(self.n_cols)
        total = np.zeros(d, dtype=np.float64)
        off = f["tree_offsets"]
        for t in range(len(off) - 1):
            imp = np.zeros(d, dtype=np.float64)
            for i in range(int(off[t]), int(off[t + 1])):
                if f["feature"][i] >= 0:
                    imp[int(f["feature"][i])] += float(f["gain"][i]) * float(f["count"][i])
            s = imp.sum()
            if s > 0:
                total += imp / s
        s = total.sum()
        vals = total / s if s > 0 else total
        try:
            from pyspark.ml.linalg import DenseVector
        except ImportError:
            return vals
        return DenseVector(list(vals))

    _combined_attrs = ("model_json",)

    def _out_schema(self, input_schema: Any = None) -> str:
        return "double"

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        if eval_metric_info is not None:
            return self._eval_func(eval_metric_info)
        forest = self._flat()
        classification = self._is_classification()

        def predict(m: Any, X: Any) -> Tuple[Any, ...]:   # k_rf_predict: (raw, prob, pred), or (None, None, pred)
            raw, prob, pred = m.ctx.rf_predict(X, forest, classification)
            return (raw, prob, pred) if classification else (pred,)

        V = int(forest["value"].shape[1])
        return _DeviceModel, self._grouped_transform(predict, 4 * int(self.n_cols) + 8 * (2 * V + 1)), None

    def _transform_outputs(self) -> List[Tuple[str, str]]:
        pred = (self.getOrDefault("predictionCol"), "double")
        if not self._is_classification():
            return [pred]
        return [(self.getOrDefault("rawPredictionCol"), "array<double>"),
                (self.getOrDefault("probabilityCol"), "array<double>"), pred]

    def _transform(self, dataset: Any) -> Any:
        _no_spark_transform(self, dataset)   # the regressor too: a forest has no pandas_udf transform
        return super()._transform(dataset)

    def _eval_func(self, info: Dict[str, Any]) -> Tuple[Callable, Any, Callable]:
        """(construct, None, evaluate): evaluate(device model, X, y) scores every forest of this (combined) model in
        one device pass (b2k_eval_forest) and returns their accumulators; for a BinaryClassificationEvaluator,
        evaluate(device model, X, y, scores, pos, row0) writes their binary scores (b2k_eval_forest_scores) instead."""
        from .core import _class_accs

        classification = self._is_classification()
        if info["classification"] != classification:
            raise NotImplementedError(f"{type(self).__name__} is evaluated with a "
                                      f"{'MulticlassClassification' if classification else 'Regression'}Evaluator")
        V = self._num_classes if classification else 1
        jsons = self._model_json if isinstance(self._model_json, list) else [self._model_json]
        forests = [json_to_forest(j, V) for j in jsons]
        eps = info["eps"]

        if info["binary"]:
            def _scores(h: Any, X: Any, y: Any, scores: Any, pos: Any, row0: int) -> None:
                h.ctx.binary_scores_forest(X, y, forests, scores, pos, row0)

            _scores.n_models = len(forests)  # type: ignore[attr-defined]
            return _DeviceModel, None, _scores

        def _evaluate(h: Any, X: Any, y: Any) -> List[Dict[str, Any]]:
            return _class_accs(h.ctx.eval_forest(X, y, forests, classification, eps))

        return _DeviceModel, None, _evaluate
