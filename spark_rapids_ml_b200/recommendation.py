"""ALS / ALSModel: Spark's pyspark.ml.recommendation.ALS (alternating least squares collaborative filtering) on H100.

The reference has no recommender; this follows Spark's estimator, its rules pinned in include/b2kmeans.h
(b2k_als_fit / b2k_als_predict / b2k_als_recommend; DESIGN §25).  Fit, transform and the recommendFor* calls run on
local frames; a pyspark DataFrame raises.
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa

from .core import _load_metadata, _reset_uid, _row_groups, _save_metadata, _set_params_from_metadata
from .sparkshim import HAVE_PYSPARK, Param, Params, TypeConverters, keyword_only

_ALS_PARAMS = [
    # (name, default, converter, doc)
    ("rank", 10, TypeConverters.toInt, "rank of the factorization"),
    ("maxIter", 10, TypeConverters.toInt, "max number of iterations (>= 0)"),
    ("regParam", 0.1, TypeConverters.toFloat, "regularization parameter (>= 0)"),
    ("implicitPrefs", False, TypeConverters.toBoolean if hasattr(TypeConverters, "toBoolean") else bool,
     "whether to use implicit preference"),
    ("alpha", 1.0, TypeConverters.toFloat, "alpha for implicit preference"),
    ("userCol", "user", TypeConverters.toString, "column name for user ids; ids must be within the integer value range"),
    ("itemCol", "item", TypeConverters.toString, "column name for item ids; ids must be within the integer value range"),
    ("ratingCol", "rating", TypeConverters.toString, "column name for ratings"),
    ("predictionCol", "prediction", TypeConverters.toString, "prediction column name"),
    ("coldStartStrategy", "nan", TypeConverters.toString,
     "strategy for dealing with unknown or new users/items at prediction time: nan or drop"),
    ("seed", None, TypeConverters.toInt, "random seed"),
    # accepted and recorded with Spark's defaults; they have no effect here
    ("nonnegative", False, TypeConverters.toBoolean if hasattr(TypeConverters, "toBoolean") else bool,
     "whether to use nonnegative constraint for least squares"),
    ("numUserBlocks", 10, TypeConverters.toInt, "number of user blocks (no effect)"),
    ("numItemBlocks", 10, TypeConverters.toInt, "number of item blocks (no effect)"),
    ("checkpointInterval", 10, TypeConverters.toInt, "checkpoint interval (no effect)"),
    ("intermediateStorageLevel", "MEMORY_AND_DISK", TypeConverters.toString, "storage level (no effect)"),
    ("finalStorageLevel", "MEMORY_AND_DISK", TypeConverters.toString, "storage level (no effect)"),
    ("blockSize", 4096, TypeConverters.toInt, "block size for stacking input data (no effect)"),
]
_MODEL_PARAMS = ("userCol", "itemCol", "predictionCol", "coldStartStrategy", "blockSize")


def _refuse_pyspark(dataset: Any, who: str) -> None:
    if HAVE_PYSPARK:
        from . import spark_binding

        if spark_binding.is_spark_dataframe(dataset):
            raise NotImplementedError(f"{who} of a pyspark DataFrame is not supported yet; use a local frame")


def _id_values(table: pa.Table, col: str) -> np.ndarray:
    """A user or item column as float64, checked by Spark's rule: numeric, integral, inside int32, no null."""
    if col not in table.column_names:
        raise ValueError(f"column {col} does not exist in the dataset")
    c = table.column(col)
    if not (pa.types.is_integer(c.type) or pa.types.is_floating(c.type) or pa.types.is_decimal(c.type)):
        raise TypeError(f"Column {col} must be of type numeric but was actually of type {c.type}.")
    if c.null_count:
        raise ValueError(f"ALS only supports values in Integer range and without fractional part for column {col}. "
                         "Value null was either out of Integer range or contained a fractional part that could not be "
                         "converted.")
    v = np.asarray(c.to_numpy(zero_copy_only=False), dtype=np.float64)
    bad = ~(np.isfinite(v) & (v >= -2.0 ** 31) & (v <= 2.0 ** 31 - 1) & (v == np.floor(v)))
    if bad.any():
        x = float(v[int(np.argmax(bad))])
        s = "NaN" if x != x else (f"{x:.1f}" if x == np.floor(x) and abs(x) < 1e18 else repr(x))
        raise ValueError(f"ALS only supports values in Integer range and without fractional part for column {col}. "
                         f"Value {s} was either out of Integer range or contained a fractional part that could not be "
                         "converted.")
    return v


class _ALSParams(Params):
    _param_names: Tuple[str, ...] = tuple(n for n, *_ in _ALS_PARAMS)

    def __init__(self) -> None:
        super().__init__()
        mine = [p for p in _ALS_PARAMS if p[0] in self._param_names]
        for name, default, conv, doc in mine:
            setattr(self, name, Param(self, name, doc, typeConverter=conv))
        self._setDefault(**{n: d for n, d, _, _ in mine if d is not None})
        if "seed" in self._param_names:   # the KMeans rule: a 32-bit signed seed from the class name
            self._setDefault(seed=hash(type(self).__name__) & 0x07FFFFFFF)
        self._cuml_params: Dict[str, Any] = {}
        self._num_workers = None
        self._float32_inputs = True

    def _p(self, name: str) -> Any:
        return self.getOrDefault(name)

    def getRank(self) -> int:
        return int(self._p("rank"))

    def getMaxIter(self) -> int:
        return int(self._p("maxIter"))

    def getRegParam(self) -> float:
        return float(self._p("regParam"))

    def getImplicitPrefs(self) -> bool:
        return bool(self._p("implicitPrefs"))

    def getAlpha(self) -> float:
        return float(self._p("alpha"))

    def getUserCol(self) -> str:
        return self._p("userCol")

    def getItemCol(self) -> str:
        return self._p("itemCol")

    def getRatingCol(self) -> str:
        return self._p("ratingCol")

    def getPredictionCol(self) -> str:
        return self._p("predictionCol")

    def getColdStartStrategy(self) -> str:
        return self._p("coldStartStrategy")

    def getSeed(self) -> int:
        return int(self._p("seed"))

    def getNonnegative(self) -> bool:
        return bool(self._p("nonnegative"))

    def getNumUserBlocks(self) -> int:
        return int(self._p("numUserBlocks"))

    def getNumItemBlocks(self) -> int:
        return int(self._p("numItemBlocks"))

    def getCheckpointInterval(self) -> int:
        return int(self._p("checkpointInterval"))

    def getIntermediateStorageLevel(self) -> str:
        return self._p("intermediateStorageLevel")

    def getFinalStorageLevel(self) -> str:
        return self._p("finalStorageLevel")

    def getBlockSize(self) -> int:
        return int(self._p("blockSize"))

    def _set_checked(self, **kw: Any) -> Any:
        for k, v in kw.items():
            if v is None:
                continue
            if k == "coldStartStrategy" and str(v).lower() not in ("nan", "drop"):
                raise ValueError(f"coldStartStrategy must be one of nan, drop, got {v!r}")
            if k in ("rank", "numUserBlocks", "numItemBlocks", "blockSize") and int(v) < 1:
                raise ValueError(f"{k} given invalid value {v}")
            if k in ("maxIter",) and int(v) < 0:
                raise ValueError(f"maxIter given invalid value {v}")
            if k in ("regParam", "alpha") and not float(v) >= 0:
                raise ValueError(f"{k} given invalid value {v}")
            if k == "coldStartStrategy":
                v = str(v).lower()
            self._set(**{k: v})
        return self


def _setter(name: str) -> Any:
    def f(self: Any, value: Any) -> Any:
        return self._set_checked(**{name: value})
    f.__name__ = "set" + name[0].upper() + name[1:]
    return f


class ALS(_ALSParams):
    """Alternating least squares matrix factorization on H100, Spark's pyspark.ml.recommendation.ALS: explicit or
    implicit feedback, per half-step one fp64 normal-equation pass over each destination's ratings and one batched
    Cholesky solve (b2k_als.cu).  Params with Spark's names and defaults: rank (10), maxIter (10), regParam (0.1),
    implicitPrefs (False), alpha (1.0), userCol ("user"), itemCol ("item"), ratingCol ("rating"; "" = every rating 1.0),
    predictionCol ("prediction"), coldStartStrategy ("nan" | "drop"), seed; numUserBlocks, numItemBlocks,
    checkpointInterval, intermediateStorageLevel, finalStorageLevel and blockSize are accepted and recorded and have no
    effect.  The start factors come from the library's seeded generator, not Spark's XORShiftRandom, so they differ from
    Spark's for the same seed.  nonnegative = True, a pyspark DataFrame and CrossValidator / fitMultiple raise."""

    @keyword_only
    def __init__(self, *, rank: int = 10, maxIter: int = 10, regParam: float = 0.1, numUserBlocks: int = 10,
                 numItemBlocks: int = 10, implicitPrefs: bool = False, alpha: float = 1.0, userCol: str = "user",
                 itemCol: str = "item", seed: Optional[int] = None, ratingCol: str = "rating",
                 nonnegative: bool = False, checkpointInterval: int = 10,
                 intermediateStorageLevel: str = "MEMORY_AND_DISK", finalStorageLevel: str = "MEMORY_AND_DISK",
                 coldStartStrategy: str = "nan", blockSize: int = 4096, predictionCol: str = "prediction") -> None:
        super().__init__()
        self._set_checked(**self._input_kwargs)

    def setParams(self, **kw: Any) -> "ALS":
        return self._set_checked(**kw)

    for _n, *_ in _ALS_PARAMS:
        locals()["set" + _n[0].upper() + _n[1:]] = _setter(_n)
    del _n

    def fitMultiple(self, dataset: Any, paramMaps: Any) -> Any:
        raise NotImplementedError("ALS.fitMultiple is not supported: CrossValidator does not tune ALS in this build")

    def _supportsTransformEvaluate(self, evaluator: Any) -> bool:
        return False

    def fit(self, dataset: Any, params: Optional[Dict[Any, Any]] = None) -> "ALSModel":
        if params:
            return self.copy(params).fit(dataset)
        _refuse_pyspark(dataset, "ALS.fit")
        if self.getNonnegative():
            raise NotImplementedError("ALS with nonnegative = True (NNLS) is not supported")
        import torch

        from . import _native

        table = dataset._table()
        u = _id_values(table, self.getUserCol())
        i = _id_values(table, self.getItemCol())
        rc = self.getRatingCol()
        r = None
        if rc:
            if rc not in table.column_names:
                raise ValueError(f"column {rc} does not exist in the dataset")
            c = table.column(rc)
            if c.null_count:
                raise ValueError(f"ALS only supports finite ratings in column {rc}; got null")
            r = np.asarray(c.to_numpy(zero_copy_only=False), dtype=np.float32)
            if not np.isfinite(r).all():
                raise ValueError(f"ALS only supports finite ratings in column {rc}; got "
                                 f"{r[int(np.argmax(~np.isfinite(r)))]}")
        if len(u) == 0:
            raise ValueError("ALS: the dataset has no ratings")
        dev = torch.device("cuda", torch.cuda.current_device())
        with _native.Context(dev.index) as ctx:
            out = ctx.als_fit(torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev),
                              None if r is None else torch.from_numpy(r).to(dev), rank=self.getRank(),
                              max_iter=self.getMaxIter(), reg_param=self.getRegParam(),
                              implicit_prefs=self.getImplicitPrefs(), alpha=self.getAlpha(), seed=self.getSeed())
            res = {k: v.cpu().numpy() for k, v in out.items()}
        model = ALSModel(self.getRank(), res["user_ids"], res["user_factors"], res["item_ids"], res["item_factors"])
        for name in _MODEL_PARAMS:
            if self.isSet(name):
                model._set(**{name: self.getOrDefault(name)})
        return model

    def write(self) -> Any:
        from .core import _Writer

        return _Writer(self, None)

    def save(self, path: str, overwrite: bool = False) -> None:
        w = self.write()
        (w.overwrite() if overwrite else w).save(path)

    @classmethod
    def load(cls, path: str) -> "ALS":
        from .core import _Reader

        return _Reader(cls, False).load(path)


def _factors_frame(session: Any, ids: np.ndarray, F: np.ndarray) -> Any:
    rank = F.shape[1]
    offsets = pa.array(np.arange(0, (len(ids) + 1) * rank, rank, dtype=np.int32))
    feats = pa.ListArray.from_arrays(offsets, pa.array(np.ascontiguousarray(F, dtype=np.float32).reshape(-1)))
    return session.createDataFrame(pa.Table.from_arrays([pa.array(ids.astype(np.int32)), feats],
                                                        names=["id", "features"]))


class ALSModel(_ALSParams):
    """A fitted ALS model: rank, userFactors / itemFactors (columns id int, features array<float>, sorted by id),
    transform (a prediction column by the device predict pass; coldStartStrategy "nan" gives NaN for an unknown user or
    item, "drop" removes those rows), recommendForAllUsers / recommendForAllItems / recommendForUserSubset /
    recommendForItemSubset (Spark's schema; scores bitwise equal to the predictions), and Spark's ALSModel persistence
    layout (metadata with rank, userFactors/ and itemFactors/ parquet)."""

    _param_names = _MODEL_PARAMS

    def __init__(self, rank: int, user_ids: Any, user_factors: Any, item_ids: Any, item_factors: Any) -> None:
        super().__init__()
        self._rank = int(rank)
        self._uid_ = np.asarray(user_ids, dtype=np.int32)
        self._uf = np.ascontiguousarray(user_factors, dtype=np.float32).reshape(len(self._uid_), self._rank)
        self._iid_ = np.asarray(item_ids, dtype=np.int32)
        self._if = np.ascontiguousarray(item_factors, dtype=np.float32).reshape(len(self._iid_), self._rank)

    for _n in _MODEL_PARAMS:
        locals()["set" + _n[0].upper() + _n[1:]] = _setter(_n)
    del _n

    @property
    def rank(self) -> int:
        return self._rank

    def _session(self) -> Any:
        from .sparkshim import get_session

        return get_session()

    @property
    def userFactors(self) -> Any:
        return _factors_frame(self._session(), self._uid_, self._uf)

    @property
    def itemFactors(self) -> Any:
        return _factors_frame(self._session(), self._iid_, self._if)

    def _device(self) -> Tuple[Any, Any]:
        import torch

        from . import _native

        dev = torch.device("cuda", torch.cuda.current_device())
        ctx = _native.Context(dev.index)
        t = {k: torch.from_numpy(np.array(v)).to(dev) for k, v in (("user_ids", self._uid_), ("user_factors", self._uf),
                                                                    ("item_ids", self._iid_), ("item_factors", self._if))}
        return ctx, t

    def transform(self, dataset: Any, params: Optional[Dict[Any, Any]] = None) -> Any:
        if params:
            return self.copy(params).transform(dataset)
        _refuse_pyspark(dataset, "ALSModel.transform")
        import pyarrow.compute as pc
        import torch

        from .sparkshim.sql import _batches_to_pdf_iter

        ucol, icol = self.getUserCol(), self.getItemCol()
        ctx, dm = self._device()
        dev = dm["user_ids"].device
        cols: List[List[pa.Array]] = []
        try:
            for part in dataset._parts:
                sel = [b.select([ucol, icol]) for b in part]
                frames = _batches_to_pdf_iter(sel, dataset.arrow_backed_pandas)
                arrs: List[pa.Array] = []
                # the grouped device-predict path: consecutive batches go to the device as one prediction pass
                for group in _row_groups(frames, 16):
                    uv = [_id_values(pa.Table.from_pandas(f, preserve_index=False), ucol) for f in group]
                    iv = [_id_values(pa.Table.from_pandas(f, preserve_index=False), icol) for f in group]
                    n_all = sum(len(x) for x in uv)
                    if n_all == 0:
                        arrs.extend(pa.array(np.zeros(0, dtype=np.float32)) for _ in group)
                        continue
                    p = ctx.als_predict(torch.from_numpy(np.concatenate(uv)).to(dev),
                                        torch.from_numpy(np.concatenate(iv)).to(dev), dm["user_ids"],
                                        dm["user_factors"], dm["item_ids"], dm["item_factors"]).cpu().numpy()
                    o = 0
                    for x in uv:
                        arrs.append(pa.array(p[o:o + len(x)], type=pa.float32()))
                        o += len(x)
                cols.append(arrs)
        finally:
            ctx.close()
        out = dataset.with_appended_column(self.getPredictionCol(), cols)
        if self.getColdStartStrategy() == "drop":
            parts = [[b.filter(pc.invert(pc.is_nan(b.column(self.getPredictionCol())))) for b in p] for p in out._parts]
            out = out._derive(parts)
        return out

    def _recommend(self, q_ids: np.ndarray, Q: np.ndarray, t_ids: np.ndarray, T: np.ndarray, n: int, qcol: str,
                   tcol: str) -> Any:
        import torch

        from . import _native

        n = int(n)
        if not 1 <= n <= _native.ALS_MAX_N:
            raise ValueError(f"the number of recommendations must be in [1, {_native.ALS_MAX_N}], got {n}")
        k = min(n, len(t_ids))
        idx = np.zeros((len(q_ids), k), dtype=np.int64)
        sc = np.zeros((len(q_ids), k), dtype=np.float32)
        if len(q_ids) and k:
            dev = torch.device("cuda", torch.cuda.current_device())
            with _native.Context(dev.index) as ctx:
                di, ds = ctx.als_recommend(torch.from_numpy(np.ascontiguousarray(Q)).to(dev),
                                           torch.from_numpy(T).to(dev), n)
                idx, sc = di.cpu().numpy()[:, :k].astype(np.int64), ds.cpu().numpy()[:, :k]
        struct = pa.StructArray.from_arrays([pa.array(t_ids[idx.reshape(-1)].astype(np.int32)),
                                             pa.array(sc.reshape(-1), type=pa.float32())], names=[tcol, "rating"])
        recs = pa.ListArray.from_arrays(pa.array(np.arange(0, (len(q_ids) + 1) * k, k, dtype=np.int32)), struct)
        return self._session().createDataFrame(pa.Table.from_arrays([pa.array(q_ids.astype(np.int32)), recs],
                                                                    names=[qcol, "recommendations"]))

    def recommendForAllUsers(self, numItems: int) -> Any:
        return self._recommend(self._uid_, self._uf, self._iid_, self._if, numItems, self.getUserCol(),
                               self.getItemCol())

    def recommendForAllItems(self, numUsers: int) -> Any:
        return self._recommend(self._iid_, self._if, self._uid_, self._uf, numUsers, self.getItemCol(),
                               self.getUserCol())

    def _subset(self, dataset: Any, col: str, ids: np.ndarray) -> np.ndarray:
        _refuse_pyspark(dataset, "ALSModel.recommendFor*Subset")
        v = np.unique(_id_values(dataset._table(), col).astype(np.int64))
        pos = np.searchsorted(ids, v)
        known = (pos < len(ids)) & (ids[np.minimum(pos, len(ids) - 1)] == v)
        return pos[known]

    def recommendForUserSubset(self, dataset: Any, numItems: int) -> Any:
        rows = self._subset(dataset, self.getUserCol(), self._uid_)
        return self._recommend(self._uid_[rows], self._uf[rows], self._iid_, self._if, numItems, self.getUserCol(),
                               self.getItemCol())

    def recommendForItemSubset(self, dataset: Any, numUsers: int) -> Any:
        rows = self._subset(dataset, self.getItemCol(), self._iid_)
        return self._recommend(self._iid_[rows], self._if[rows], self._uid_, self._uf, numUsers, self.getItemCol(),
                               self.getUserCol())

    # -- persistence: Spark's ALSModel layout --
    def write(self) -> Any:
        model = self

        class _W:
            _overwrite = False

            def overwrite(self) -> Any:
                self._overwrite = True
                return self

            def save(self, path: str) -> None:
                import pyarrow.parquet as pq

                _save_metadata(model, path, self._overwrite, {"rank": model._rank})
                for name, ids, F in (("userFactors", model._uid_, model._uf), ("itemFactors", model._iid_, model._if)):
                    d = os.path.join(path, name)
                    os.makedirs(d, exist_ok=True)
                    rank = F.shape[1]
                    feats = pa.ListArray.from_arrays(pa.array(np.arange(0, (len(ids) + 1) * rank, rank, dtype=np.int32)),
                                                     pa.array(F.reshape(-1), type=pa.float32()))
                    pq.write_table(pa.Table.from_arrays([pa.array(ids, type=pa.int32()), feats], names=["id", "features"]),
                                   os.path.join(d, "part-00000.parquet"))
                    open(os.path.join(d, "_SUCCESS"), "w").close()

        return _W()

    def save(self, path: str, overwrite: bool = False) -> None:
        w = self.write()
        (w.overwrite() if overwrite else w).save(path)

    @classmethod
    def load(cls, path: str) -> "ALSModel":
        import pyarrow.parquet as pq

        meta = _load_metadata(path)
        tabs = []
        for name in ("userFactors", "itemFactors"):
            t = pq.read_table(os.path.join(path, name)).sort_by("id")
            ids = np.asarray(t.column("id").to_numpy(), dtype=np.int32)
            F = np.asarray(t.column("features").combine_chunks().flatten().to_numpy(), dtype=np.float32)
            tabs.append((ids, F))
        rank = int(meta["rank"])
        inst = cls(rank, tabs[0][0], tabs[0][1], tabs[1][0], tabs[1][1])
        _reset_uid(inst, meta["uid"])
        _set_params_from_metadata(inst, meta)
        return inst


__all__ = ["ALS", "ALSModel"]
