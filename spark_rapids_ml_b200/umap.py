"""UMAP / UMAPModel — the reference's surface (python/src/spark_rapids_ml/umap.py), with cuML UMAP replaced by
b2k_umap_fit / b2k_umap_transform (hand-written sm_90a CUDA, csrc/b2k_umap.cu; semantics in include/b2kmeans.h).

  UMAPClass (params and defaults)                          umap.py:109-141
  _UMAPCumlParams (Spark params, getters and setters)      umap.py:144-675
  UMAP (fit on one GPU: the rows coalesce to one task)     umap.py:678-1065
  UMAPModel (transform one task per GPU, persistence)      umap.py:1068-1551

Differences that are deliberate: fit and transform of a pyspark DataFrame, sparse input, precomputed_knn and metrics
other than euclidean / l2 raise; build_algo "nn_descent" runs the exact search; build_kwds and transform_queue_size are
accepted and unused.  The layout is the epoch-synchronous, deterministic form of DESIGN §17.
"""
from __future__ import annotations

import functools
import json
import os
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import pyarrow as pa

from .core import (FitInputType, _CumlEstimator, _CumlModelWithColumns, _DeviceModel, _save_metadata, _load_metadata,
                   _reset_uid, _set_params_from_metadata, param_alias)
from .params import HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasOutputCol, P, _CumlClass, _CumlParams
from .sparkshim import HAVE_PYSPARK, Param, TypeConverters, keyword_only
from .utils import get_logger

_METRICS = ("euclidean", "l2")


class UMAPClass(_CumlClass):
    @classmethod
    def _param_mapping(cls) -> Dict[str, Optional[str]]:
        return {}

    def _get_cuml_params_default(self) -> Dict[str, Any]:
        return {"n_neighbors": 15, "n_components": 2, "metric": "euclidean", "metric_kwds": None, "n_epochs": None,
                "learning_rate": 1.0, "init": "spectral", "min_dist": 0.1, "spread": 1.0, "set_op_mix_ratio": 1.0,
                "local_connectivity": 1.0, "repulsion_strength": 1.0, "negative_sample_rate": 5,
                "transform_queue_size": 4.0, "a": None, "b": None, "precomputed_knn": None, "random_state": None,
                "verbose": False, "build_algo": "auto", "build_kwds": None}

    def _pyspark_class(self) -> Optional[type]:
        return None


def _p(name: str, doc: str, conv: Any = None) -> Param:
    return Param("parent", name, doc, conv) if conv is not None else Param("parent", name, doc)


class _UMAPCumlParams(_CumlParams, HasFeaturesCol, HasFeaturesCols, HasLabelCol, HasOutputCol):
    """Shared Spark Params of UMAP and UMAPModel (reference: umap.py:144-675)."""

    def __init__(self) -> None:
        super().__init__()
        self._setDefault(n_neighbors=15, n_components=2, metric="euclidean", metric_kwds=None, n_epochs=None,
                         learning_rate=1.0, init="spectral", min_dist=0.1, spread=1.0, set_op_mix_ratio=1.0,
                         local_connectivity=1.0, repulsion_strength=1.0, negative_sample_rate=5,
                         transform_queue_size=4.0, a=None, b=None, random_state=None, build_algo="auto",
                         build_kwds=None, sample_fraction=1.0, outputCol="embedding")

    n_neighbors = _p("n_neighbors", "The size of local neighborhood used for manifold approximation.",
                     TypeConverters.toFloat)
    n_components = _p("n_components", "The dimension of the space to embed into.", TypeConverters.toInt)
    metric = _p("metric", "Distance metric (euclidean or l2).", TypeConverters.toString)
    metric_kwds = _p("metric_kwds", "Additional keyword arguments for the metric function.")
    n_epochs = _p("n_epochs", "The number of training epochs (None: 500 for at most 10000 rows, else 200).",
                  TypeConverters.toInt)
    learning_rate = _p("learning_rate", "The initial learning rate for the embedding optimization.",
                       TypeConverters.toFloat)
    init = _p("init", "How to initialize the low dimensional embedding: 'spectral' or 'random'.",
              TypeConverters.toString)
    min_dist = _p("min_dist", "The effective minimum distance between embedded points.", TypeConverters.toFloat)
    spread = _p("spread", "The effective scale of embedded points.", TypeConverters.toFloat)
    set_op_mix_ratio = _p("set_op_mix_ratio", "Interpolate between fuzzy union (1.0) and intersection (0.0).",
                          TypeConverters.toFloat)
    local_connectivity = _p("local_connectivity", "The local connectivity required.", TypeConverters.toFloat)
    repulsion_strength = _p("repulsion_strength", "Weighting applied to negative samples.", TypeConverters.toFloat)
    negative_sample_rate = _p("negative_sample_rate", "Negative samples per positive sample.", TypeConverters.toInt)
    transform_queue_size = _p("transform_queue_size", "Accepted for compatibility; unused.", TypeConverters.toFloat)
    a = _p("a", "More specific parameter controlling the embedding (None: fitted from min_dist and spread).",
           TypeConverters.toFloat)
    b = _p("b", "More specific parameter controlling the embedding (None: fitted from min_dist and spread).",
           TypeConverters.toFloat)
    random_state = _p("random_state", "Seed of the sample, the initial layout and the negative draws.",
                      TypeConverters.toInt)
    build_algo = _p("build_algo", "k-NN graph construction: 'auto', 'brute_force_knn' or 'nn_descent' (all exact).",
                    TypeConverters.toString)
    build_kwds = _p("build_kwds", "Accepted for compatibility; unused.")
    sample_fraction = _p("sample_fraction", "Fraction of the rows the fit uses (seeded Bernoulli sample).",
                         TypeConverters.toFloat)

    def _g(self, name: str) -> Any:
        return self.getOrDefault(name)

    def getNNeighbors(self) -> float: return self._g("n_neighbors")   # noqa: E704
    def setNNeighbors(self: P, value: float) -> P: return self._set_params(n_neighbors=value)   # noqa: E704
    def getNComponents(self) -> int: return self._g("n_components")   # noqa: E704
    def setNComponents(self: P, value: int) -> P: return self._set_params(n_components=value)   # noqa: E704
    def getMetric(self) -> str: return self._g("metric")   # noqa: E704
    def setMetric(self: P, value: str) -> P: return self._set_params(metric=value)   # noqa: E704
    def getMetricKwds(self) -> Optional[Dict[str, Any]]: return self._g("metric_kwds")   # noqa: E704
    def setMetricKwds(self: P, value: Dict[str, Any]) -> P: return self._set_params(metric_kwds=value)   # noqa: E704
    def getNEpochs(self) -> int: return self._g("n_epochs")   # noqa: E704
    def setNEpochs(self: P, value: int) -> P: return self._set_params(n_epochs=value)   # noqa: E704
    def getLearningRate(self) -> float: return self._g("learning_rate")   # noqa: E704
    def setLearningRate(self: P, value: float) -> P: return self._set_params(learning_rate=value)   # noqa: E704
    def getInit(self) -> str: return self._g("init")   # noqa: E704
    def setInit(self: P, value: str) -> P: return self._set_params(init=value)   # noqa: E704
    def getMinDist(self) -> float: return self._g("min_dist")   # noqa: E704
    def setMinDist(self: P, value: float) -> P: return self._set_params(min_dist=value)   # noqa: E704
    def getSpread(self) -> float: return self._g("spread")   # noqa: E704
    def setSpread(self: P, value: float) -> P: return self._set_params(spread=value)   # noqa: E704
    def getSetOpMixRatio(self) -> float: return self._g("set_op_mix_ratio")   # noqa: E704
    def setSetOpMixRatio(self: P, value: float) -> P: return self._set_params(set_op_mix_ratio=value)   # noqa: E704
    def getLocalConnectivity(self) -> float: return self._g("local_connectivity")   # noqa: E704
    def setLocalConnectivity(self: P, value: float) -> P: return self._set_params(local_connectivity=value)   # noqa: E704,E501
    def getRepulsionStrength(self) -> float: return self._g("repulsion_strength")   # noqa: E704
    def setRepulsionStrength(self: P, value: float) -> P: return self._set_params(repulsion_strength=value)   # noqa: E704,E501
    def getNegativeSampleRate(self) -> int: return self._g("negative_sample_rate")   # noqa: E704
    def setNegativeSampleRate(self: P, value: int) -> P: return self._set_params(negative_sample_rate=value)   # noqa: E704,E501
    def getTransformQueueSize(self) -> float: return self._g("transform_queue_size")   # noqa: E704
    def setTransformQueueSize(self: P, value: float) -> P: return self._set_params(transform_queue_size=value)   # noqa: E704,E501
    def getA(self) -> float: return self._g("a")   # noqa: E704
    def setA(self: P, value: float) -> P: return self._set_params(a=value)   # noqa: E704
    def getB(self) -> float: return self._g("b")   # noqa: E704
    def setB(self: P, value: float) -> P: return self._set_params(b=value)   # noqa: E704
    def getRandomState(self) -> int: return self._g("random_state")   # noqa: E704
    def setRandomState(self: P, value: int) -> P: return self._set_params(random_state=value)   # noqa: E704
    def getBuildAlgo(self) -> str: return self._g("build_algo")   # noqa: E704
    def setBuildAlgo(self: P, value: str) -> P: return self._set_params(build_algo=value)   # noqa: E704
    def getBuildKwds(self) -> Optional[Dict[str, Any]]: return self._g("build_kwds")   # noqa: E704
    def setBuildKwds(self: P, value: Dict[str, Any]) -> P: return self._set_params(build_kwds=value)   # noqa: E704
    def getSampleFraction(self) -> float: return self._g("sample_fraction")   # noqa: E704
    def setSampleFraction(self: P, value: float) -> P: return self._set_params(sample_fraction=value)   # noqa: E704

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

    def getOutputCol(self) -> str:
        return self.getOrDefault("outputCol")

    def setOutputCol(self: P, value: str) -> P:
        return self._set_params(outputCol=value)


def find_ab_params(spread: float = 1.0, min_dist: float = 0.1) -> Tuple[float, float]:
    """a, b of 1 / (1 + a x^(2b)) fitted by least squares (Gauss-Newton, fp64) to the target curve: 1 below min_dist,
    exp(-(x - min_dist) / spread) above, at 300 points on [0, 3 spread]."""
    x = np.linspace(0, spread * 3, 300)
    y = np.where(x < min_dist, 1.0, np.exp(-(x - min_dist) / spread))
    a, b = 1.0, 1.0
    lx = np.where(x > 0, np.log(np.where(x > 0, x, 1.0)), 0.0)
    for _ in range(200):
        xb = np.where(x > 0, x ** (2 * b), 0.0)
        f = 1.0 / (1.0 + a * xb)
        J = np.stack([-xb * f * f, -a * xb * 2 * lx * f * f], 1)
        step = np.linalg.lstsq(J, y - f, rcond=None)[0]
        a, b = a + step[0], b + step[1]
        if np.abs(step).max() < 1e-14:
            break
    return float(a), float(b)


def bernoulli_sample(n: int, fraction: float, seed: int) -> np.ndarray:
    """Rows kept by the fit's sample: row r is kept when u_r < fraction, u from numpy.random.default_rng(seed)."""
    if fraction >= 1.0:
        return np.arange(n)
    return np.nonzero(np.random.default_rng(seed).random(n) < fraction)[0]


def _no_pyspark(dataset: Any, what: str) -> None:
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError(f"UMAP {what} of a pyspark DataFrame is not supported yet; use a local frame")


def _check_supported(p: Any) -> None:
    metric = p.getOrDefault("metric")
    if metric not in _METRICS:
        raise ValueError(f"metric {metric!r} is not supported: use 'euclidean' or 'l2'")
    if p.cuml_params.get("precomputed_knn") is not None:
        raise ValueError("precomputed_knn is not supported")
    if p.getOrDefault("init") not in ("spectral", "random"):
        raise ValueError(f"init must be 'spectral' or 'random', got {p.getOrDefault('init')!r}")
    if p.getOrDefault("build_algo") not in ("auto", "brute_force_knn", "nn_descent"):
        raise ValueError(f"build_algo {p.getOrDefault('build_algo')!r} is not supported")
    nc = p.getOrDefault("n_components")
    if not 1 <= int(nc) <= 100:
        raise ValueError(f"n_components must be in [1, 100], got {nc}")
    sf = float(p.getOrDefault("sample_fraction"))
    if not 0.0 < sf <= 1.0:
        raise ValueError(f"sample_fraction must be in (0, 1], got {sf}")


def _device_params(cp: Dict[str, Any], k: int, n_epochs: int, init: str, seed: int) -> Any:
    from . import _native

    a, b = cp.get("a"), cp.get("b")
    if a is None or b is None:
        a, b = find_ab_params(float(cp["spread"]), float(cp["min_dist"]))
    return _native.umap_params(n_neighbors=k, n_components=int(cp["n_components"]), n_epochs=n_epochs, init=init,
                               negative_sample_rate=int(cp["negative_sample_rate"]),
                               local_connectivity=float(cp["local_connectivity"]),
                               set_op_mix_ratio=float(cp["set_op_mix_ratio"]),
                               learning_rate=float(cp["learning_rate"]),
                               repulsion_strength=float(cp["repulsion_strength"]), a=float(a), b=float(b), seed=seed)


class UMAP(UMAPClass, _CumlEstimator, _UMAPCumlParams):
    """UMAP on H100 (reference: umap.py:678-1065).  fit() coalesces the rows to one task on one GPU, whatever
    num_workers is, as the reference does; UMAPModel.transform runs one task per GPU over the frame's partitions.

    >>> from spark_rapids_ml_b200.umap import UMAP
    >>> model = UMAP(n_neighbors=10, random_state=1).setFeaturesCol("features").fit(df)
    >>> model.transform(df)   # appends "embedding" (array<float>)
    """

    @keyword_only
    def __init__(self, *, n_neighbors: Optional[float] = 15, n_components: Optional[int] = 2,
                 metric: str = "euclidean", metric_kwds: Optional[Dict[str, Any]] = None,
                 n_epochs: Optional[int] = None, learning_rate: Optional[float] = 1.0,
                 init: Optional[str] = "spectral", min_dist: Optional[float] = 0.1, spread: Optional[float] = 1.0,
                 set_op_mix_ratio: Optional[float] = 1.0, local_connectivity: Optional[float] = 1.0,
                 repulsion_strength: Optional[float] = 1.0, negative_sample_rate: Optional[int] = 5,
                 transform_queue_size: Optional[float] = 4.0, a: Optional[float] = None, b: Optional[float] = None,
                 precomputed_knn: Optional[List[List[float]]] = None, random_state: Optional[int] = None,
                 build_algo: Optional[str] = "auto", build_kwds: Optional[Dict[str, Any]] = None,
                 sample_fraction: Optional[float] = 1.0, featuresCol: Optional[Union[str, List[str]]] = None,
                 labelCol: Optional[str] = None, outputCol: Optional[str] = None, num_workers: Optional[int] = None,
                 enable_sparse_data_optim: Optional[bool] = None, verbose: Union[int, bool] = False,
                 **kwargs: Any) -> None:
        super().__init__()
        self._handle_param_spark_confs()
        self._input_kwargs.pop("kwargs", None)
        self._input_kwargs.update(kwargs)
        if not self._input_kwargs.get("float32_inputs", True):
            get_logger(self.__class__).warning("This estimator does not support double precision inputs. Setting "
                                               "float32_inputs to False will be ignored.")
            self._input_kwargs.pop("float32_inputs")
        if self._input_kwargs.pop("enable_sparse_data_optim", None):
            raise ValueError("sparse input is not supported by UMAP")
        if self._input_kwargs.get("precomputed_knn") is not None:
            raise ValueError("precomputed_knn is not supported")
        self._input_kwargs.pop("precomputed_knn", None)
        for name in ("featuresCol", "labelCol", "outputCol", "num_workers"):
            if self._input_kwargs.get(name, None) is None:
                self._input_kwargs.pop(name, None)
        self._set_params(**self._input_kwargs)

    def _fit_label_col(self) -> Optional[str]:
        return self.getOrDefault("labelCol") if self.isDefined(self.labelCol) and self.isSet(self.labelCol) else None

    @property
    def num_workers(self) -> int:
        return 1   # the reference coalesces the fit's rows to one partition (umap.py:934-941)

    @num_workers.setter
    def num_workers(self, value: int) -> None:
        self._num_workers = value

    def _fit(self, dataset: Any) -> "UMAPModel":
        _no_pyspark(dataset, "fit")
        _check_supported(self)
        if self.getOrDefault("build_algo") == "nn_descent":
            get_logger(self.__class__).info("build_algo 'nn_descent': the graph is built by the exact k-NN search")
        est = self
        if self.cuml_params.get("random_state") is None:   # drawn once; the model records it
            est = self.copy()
            est._cuml_params["random_state"] = int(np.random.SeedSequence().generate_state(1, np.uint32)[0])
        return _CumlEstimator._fit(est, dataset)

    def _out_schema(self) -> Any:
        return "embedding_ array<array<float>>, raw_data_ array<array<float>>, n_cols int, dtype string"

    def _get_cuml_fit_func(self, dataset: Any, extra_params: Optional[List[Dict[str, Any]]] = None
                           ) -> Callable[[FitInputType, Dict[str, Any]], Dict[str, Any]]:
        logger = get_logger(self.__class__)

        def _cuml_fit(dfs: FitInputType, params: Dict[str, Any]) -> Dict[str, Any]:
            # stands in for cuML UMAP(**cuml_init).fit(features, y) on the coalesced rows (umap.py:1009-1065)
            import torch

            ctx = params[param_alias.handle]
            cp = params[param_alias.cuml_init]
            seed = int(cp["random_state"])
            X, y, _ = dfs[0]
            keep = bernoulli_sample(int(X.shape[0]), float(cp.get("sample_fraction", 1.0)), seed)
            if keep.size != X.shape[0]:
                X = X.index_select(0, torch.from_numpy(keep).to(X.device)).contiguous()
                y = y.index_select(0, torch.from_numpy(keep).to(X.device)) if y is not None else None
            n = int(X.shape[0])
            k = int(cp["n_neighbors"])
            if k > n:
                logger.warning(f"n_neighbors ({k}) is larger than the number of rows ({n}): using {n}")
                k = n
            n_epochs = cp.get("n_epochs")
            n_epochs = (500 if n <= 10000 else 200) if n_epochs is None else int(n_epochs)
            labels = None
            if y is not None:
                yh = y.cpu().numpy()
                codes = np.full(n, -1, np.int32)
                known = yh != -1
                codes[known] = np.unique(yh[known], return_inverse=True)[1].astype(np.int32)
                labels = torch.from_numpy(codes).to(X.device)
            emb, info = ctx.umap_fit(X, _device_params(cp, k, n_epochs, cp["init"], seed), labels=labels)
            if cp["init"] == "spectral" and info["init_used"] == 0:
                logger.info("the k-NN graph has more than one connected component: random initial layout")
            return {"embedding_": [emb.cpu().numpy().tolist()], "raw_data_": [X.cpu().numpy().tolist()],
                    "n_cols": params[param_alias.num_cols], "dtype": "float32"}

        return _cuml_fit

    def _create_pyspark_model(self, result: Any) -> "UMAPModel":
        r = result.asDict()
        return UMAPModel(embedding_=[list(e) for e in r["embedding_"]], raw_data_=[list(x) for x in r["raw_data_"]],
                         n_cols=int(r["n_cols"]), dtype=str(r["dtype"]))


class UMAPModel(UMAPClass, _CumlModelWithColumns, _UMAPCumlParams):
    """reference: umap.py:1068-1551.  transform() appends outputCol (array<float>): each row embedded against the
    model's training rows and embedding, independently of every other row."""

    def __init__(self, embedding_: Any, raw_data_: Any, n_cols: int, dtype: str) -> None:
        super().__init__(n_cols=n_cols, dtype=dtype)
        self.embedding_ = np.asarray(embedding_, dtype=np.float32)
        self.raw_data_ = np.asarray(raw_data_, dtype=np.float32)

    @property
    def embedding(self) -> List[List[float]]:
        return self.embedding_.tolist()

    @property
    def rawData(self) -> List[List[float]]:
        return self.raw_data_.tolist()

    def _output_col_name(self) -> str:
        return self.getOrDefault("outputCol")

    def _out_schema(self, input_schema: Any = None) -> str:
        return "array<float>"

    def _transform(self, dataset: Any) -> Any:
        _no_pyspark(dataset, "transform")
        _check_supported(self)
        return super()._transform(dataset)

    def _get_cuml_transform_func(self, dataset: Any, eval_metric_info: Any = None
                                 ) -> Tuple[Callable, Callable, Optional[Callable]]:
        emb, raw = self.embedding_, self.raw_data_
        cp = dict(self.cuml_params)
        n_cols = int(self.n_cols)
        n_train = int(raw.shape[0])
        k = min(int(cp["n_neighbors"]), n_train)
        n_epochs = cp.get("n_epochs")
        n_epochs = (100 if n_train <= 10000 else 30) if n_epochs is None else int(n_epochs) // 3
        params = _device_params(cp, k, n_epochs, "random", int(cp.get("random_state") or 0))

        def predict(m: Any, Q: Any) -> Tuple[Any]:
            return (m.ctx.umap_transform(m.arrays["X"], m.arrays["E"], Q, params),)

        construct = functools.partial(_DeviceModel, X=raw, E=emb)
        return construct, self._grouped_transform(predict, 4 * (n_cols + int(emb.shape[1]))), None

    # -- persistence in the reference's layout (umap.py:1553-1640): metadata, data/metadata.json and two parquet files
    def write(self) -> Any:
        return _UMAPModelWriter(self)

    @classmethod
    def read(cls) -> Any:
        return _UMAPModelReader()


def _table(a: np.ndarray) -> pa.Table:
    return pa.table({"row_id": pa.array(np.arange(a.shape[0], dtype=np.int64)),
                     "data": pa.array(list(a), type=pa.list_(pa.float32()))})


class _UMAPModelWriter:
    def __init__(self, inst: UMAPModel) -> None:
        self.inst = inst
        self._overwrite = False

    def overwrite(self) -> "_UMAPModelWriter":
        self._overwrite = True
        return self

    def save(self, path: str) -> None:
        import pyarrow.parquet as pq

        _save_metadata(self.inst, path, self._overwrite)
        data = os.path.join(path, "data")
        os.makedirs(data, exist_ok=True)
        pq.write_table(_table(self.inst.embedding_), os.path.join(data, "embedding_.parquet"))
        pq.write_table(_table(self.inst.raw_data_), os.path.join(data, "raw_data_.parquet"))
        with open(os.path.join(data, "metadata.json"), "w") as f:
            json.dump({"n_cols": self.inst.n_cols, "dtype": self.inst.dtype}, f)


class _UMAPModelReader:
    def load(self, path: str) -> UMAPModel:
        import pyarrow.parquet as pq

        data = os.path.join(path, "data")
        with open(os.path.join(data, "metadata.json")) as f:
            md = json.load(f)

        def read(name: str) -> np.ndarray:
            t = pq.read_table(os.path.join(data, name)).sort_by("row_id")
            return np.array(t.column("data").to_pylist(), dtype=np.float32)

        model = UMAPModel(embedding_=read("embedding_.parquet"), raw_data_=read("raw_data_.parquet"),
                          n_cols=int(md["n_cols"]), dtype=str(md["dtype"]))
        meta = _load_metadata(path)
        _reset_uid(model, meta["uid"])
        _set_params_from_metadata(model, meta)
        return model
