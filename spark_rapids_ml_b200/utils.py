"""Worker utilities on the KMeans path (reference: python/src/spark_rapids_ml/utils.py:138-170 GPU id from task
resources, :358-400 _concat_and_free, :403-522 reserved-buffer ingest, :555-576 logger) — re-designed around the
device-resident ingest of libb2kmeans (no host-side stacking, no second host copy)."""
from __future__ import annotations

import logging
import sys
from typing import Any, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import pandas as pd
import pyarrow as pa

_ArrayOrder = str  # "C" | "F"


def get_logger(cls_or_callable: Any, level: str = "INFO") -> logging.Logger:
    """reference: utils.py:555-576 — one stderr logger per class name."""
    name = cls_or_callable if isinstance(cls_or_callable, str) else getattr(cls_or_callable, "__name__", str(cls_or_callable))
    logger = logging.getLogger(f"spark_rapids_ml_b200.{name}")
    logger.setLevel(level)
    if not logger.handlers:
        h = logging.StreamHandler(sys.stderr)
        h.setFormatter(logging.Formatter("%(asctime)s - %(name)s - %(levelname)s - %(message)s"))
        logger.addHandler(h)
    return logger


def _get_gpu_id(task_context: Any) -> int:
    """reference: utils.py:138-170 — GPU address from the barrier task's resources, else CUDA_VISIBLE_DEVICES[0]."""
    import os

    res = task_context.resources() if task_context is not None else {}
    if "gpu" in res and res["gpu"].addresses:
        return int(res["gpu"].addresses[0].strip())
    vis = os.environ.get("CUDA_VISIBLE_DEVICES")
    if vis:
        return 0  # first visible device
    raise RuntimeError("Couldn't get gpu id, please check the GPU resource configuration")


def _is_local(session: Any) -> bool:
    return True  # the shim session is always local mode; real Spark: sc._jsc.sc().isLocal() (utils.py:128-135)


class PartitionDescriptor:
    """reference: utils.py:300-355 — (m, n, rank, parts_rank_size) built from every rank's part sizes."""

    def __init__(self, m: int, n: int, rank: int, parts_rank_size: List[Tuple[int, int]]):
        self.m, self.n, self.rank, self.parts_rank_size = m, n, rank, parts_rank_size

    @classmethod
    def build(cls, partition_rows: List[int], total_cols: int) -> "PartitionDescriptor":
        import json

        from .sparkshim import BarrierTaskContext

        context = BarrierTaskContext.get()
        rank = context.partitionId()
        msgs = context.allGather(json.dumps((rank, partition_rows)))
        parts: List[Tuple[int, int]] = []
        total = 0
        for m_ in msgs:
            r, rows = json.loads(m_)
            for sz in rows:
                parts.append((r, sz))
                total += sz
        return cls(total, total_cols, rank, parts)


# ------------------------------------------------------------------------------------------------
# Arrow-buffer access for the ingest fast path
# ------------------------------------------------------------------------------------------------
def arrow_list_column_buffers(col: pd.Series, d: Optional[int] = None) -> Optional[Tuple[np.ndarray, np.ndarray, int]]:
    """If `col` is an Arrow-backed list<T> column, return (flat values ndarray view, int32 offsets, n_rows)
    WITHOUT copying; else None (object column of ndarrays -> the caller stacks on the host like the reference).
    `d`: the expected row width; a fixed_size_list of another width is an error (list<T> rows are validated against
    their offsets by the library)."""
    dt = col.dtype
    if not isinstance(dt, pd.ArrowDtype):
        return None
    arr = col.array._pa_array if hasattr(col.array, "_pa_array") else pa.chunked_array(col.array)
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.chunk(0) if arr.num_chunks == 1 else arr.combine_chunks()   # single chunk: stay zero-copy
    t = arr.type
    if arr.null_count:
        raise ValueError("null feature rows are not supported")
    if pa.types.is_fixed_size_list(t):
        width = t.list_size
        if d is not None and width != d:
            raise ValueError(f"feature rows are {width} wide, expected {d}")
        vals = arr.flatten().to_numpy(zero_copy_only=True)
        return vals, None, len(arr) if width else 0
    if pa.types.is_list(t):
        offsets = arr.offsets.to_numpy(zero_copy_only=True)
        vals = arr.values.to_numpy(zero_copy_only=True)  # full child buffer; offsets[0] locates the first row
        return vals, offsets, len(arr)
    return None


VECTOR_FIELDS = ("type", "size", "indices", "values")


def is_vector_struct(t: pa.DataType) -> bool:
    """Whether an Arrow type is Spark's VectorUDT SQL layout: struct<type: tinyint, size: int, indices: array<int>,
    values: array<double>> (type 0 a sparse row, 1 a dense row whose size and indices are null)."""
    return pa.types.is_struct(t) and tuple(t.field(i).name for i in range(t.num_fields)) == VECTOR_FIELDS


def _arrow_array(col: Any) -> pa.Array:
    arr = col.array._pa_array if hasattr(col.array, "_pa_array") else pa.chunked_array(col.array)
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.chunk(0) if arr.num_chunks == 1 else arr.combine_chunks()   # single chunk: stay zero-copy
    return arr


def arrow_vector_column_buffers(col: Any) -> Tuple[np.ndarray, ...]:
    """The child buffers of an Arrow-backed vector struct column, without copying the index and value buffers:
    (type int8 [n], size int32 [n], index offsets int32 [n + 1], indices int32, value offsets int32 [n + 1], values)."""
    arr = _arrow_array(col)
    if not is_vector_struct(arr.type):
        raise ValueError(f"expected a vector struct column, got {arr.type}")
    if arr.null_count:
        raise ValueError("null feature rows are not supported")
    t, size, idx, val = arr.flatten()   # flatten applies the struct's offset (zero-copy slices)
    if t.null_count:
        raise ValueError("a vector row has a null type")
    return (t.to_numpy(zero_copy_only=False).astype(np.int8, copy=False),
            size.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int32, copy=False),
            idx.offsets.to_numpy(zero_copy_only=True), idx.values.to_numpy(zero_copy_only=True),
            val.offsets.to_numpy(zero_copy_only=True), val.values.to_numpy(zero_copy_only=True))


def densify_vector_column(arr: pa.Array, d: int) -> pa.Array:
    """A vector struct array as a list<float> column of width d (the dense path's input)."""
    if arr.null_count:
        raise ValueError("null feature rows are not supported")
    t, size, idx, val = arr.flatten()
    types = t.to_numpy(zero_copy_only=False)
    n = len(arr)
    out = np.zeros((n, d), dtype=np.float32)
    vo, vv = val.offsets.to_numpy(), val.values.to_numpy(zero_copy_only=False)
    io, iv = idx.offsets.to_numpy(), idx.values.to_numpy(zero_copy_only=False)
    sizes = size.fill_null(d).to_numpy(zero_copy_only=False)
    lens = np.diff(vo)
    if np.any((types == 0) & (sizes != d)) or np.any((types == 1) & (lens != d)):
        raise ValueError(f"feature vectors have different sizes: expected {d}")
    rows = np.repeat(np.arange(n), lens)
    vals = vv[vo[0]:vo[-1]]
    pos = np.arange(vals.size) - np.repeat(vo[:-1] - vo[0], lens)   # position within the row
    cols = np.where(np.repeat(types == 1, lens), pos, 0)
    sp = np.repeat(types == 0, lens)
    if sp.any():
        if np.any(np.diff(io)[types == 0] != lens[types == 0]):
            raise ValueError("a sparse vector holds different numbers of indices and values")
        ip = np.repeat(io[:-1], lens) + pos
        cols = np.where(sp, iv[np.where(sp, ip, 0)] if iv.size else 0, cols)
    if np.any((cols < 0) | (cols >= d)):
        raise ValueError(f"a vector index is out of bounds for vectors of size {d}")
    out[rows, cols] = vals
    offsets = pa.array(np.arange(n + 1, dtype=np.int32) * np.int32(d))
    return pa.ListArray.from_arrays(offsets, pa.array(out.reshape(-1)))


class DeviceCsrAppender:
    """Growing device CSR (indptr int64 [n + 1], indices int32 [nnz], values float32 [nnz]) fed batch by batch from a
    vector struct column through b2k_ingest_csr_append; grown geometrically, on the device."""

    def __init__(self, ctx: Any, d: int, first_rows: int = 1 << 16, first_nnz: int = 1 << 20):
        import torch

        self._torch = torch
        self.ctx, self.d = ctx, d
        self.n = self.nnz = 0
        self.indptr = torch.zeros(max(1, first_rows) + 1, dtype=torch.int64, device=ctx.device)
        self.indices = torch.empty(max(1, first_nnz), dtype=torch.int32, device=ctx.device)
        self.values = torch.empty(max(1, first_nnz), dtype=torch.float32, device=ctx.device)

    def _grow(self, name: str, need: int) -> None:
        old = getattr(self, name)
        if need <= old.shape[0]:
            return
        new = self._torch.empty(max(need, 2 * old.shape[0]), dtype=old.dtype, device=old.device)
        new[: old.shape[0]] = old
        setattr(self, name, new)

    def append_column(self, col: Any) -> int:
        """One batch's vector struct column (Arrow-backed pandas Series) -> rows of the CSR; returns its row count."""
        bufs = arrow_vector_column_buffers(col)
        n_b = int(bufs[0].shape[0])
        if n_b == 0:
            return 0
        nnz_b = int(bufs[4][-1]) - int(bufs[4][0])
        self._grow("indptr", self.n + n_b + 1)
        self._grow("indices", self.nnz + nnz_b)
        self._grow("values", self.nnz + nnz_b)
        self.ctx.ingest_csr(self.indptr, self.indices, self.values, self.d, self.n, self.nnz, *bufs)
        self.n += n_b
        self.nnz += nnz_b
        return n_b

    @property
    def rows(self) -> int:
        return self.n

    def finish(self) -> Tuple[Any, Any, Any]:
        return self.indptr[: self.n + 1], self.indices[: self.nnz], self.values[: self.nnz]


class DeviceRowAppender:
    """Growing device matrix [n, d] f32 fed batch by batch through b2k_ingest_append (replaces core.py:907-941
    + clustering.py:388-393).  Capacity grows geometrically by segments; segments are concatenated on the device
    once at the end (HBM copy, not a host copy)."""

    def __init__(self, ctx: Any, d: int, first_capacity: int = 1 << 20):
        import torch

        self._torch = torch
        self.ctx, self.d = ctx, d
        self.segments: List[Any] = []
        self.fill: List[int] = []
        self.next_cap = max(1024, first_capacity)

    def _room(self, n_b: int) -> Tuple[Any, int]:
        t = self._torch
        if not self.segments or self.fill[-1] + n_b > self.segments[-1].shape[0]:
            cap = max(self.next_cap, n_b)
            self.segments.append(t.empty((cap, self.d), dtype=t.float32, device=self.ctx.device))
            self.fill.append(0)
            self.next_cap = cap * 2
        return self.segments[-1], self.fill[-1]

    def append_values(self, values: np.ndarray, offsets: Optional[np.ndarray], n_b: int) -> None:
        seg, r0 = self._room(n_b)
        self.ctx.ingest_rows(seg, r0, values, self.d, offsets=offsets, n_rows=n_b)
        self.fill[-1] += n_b

    def append_columns(self, cols: Sequence[np.ndarray]) -> None:
        n_b = int(cols[0].shape[0])
        seg, r0 = self._room(n_b)
        self.ctx.ingest_columns(seg, r0, cols)
        self.fill[-1] += n_b

    @property
    def rows(self) -> int:
        return sum(self.fill)

    def finish(self) -> Any:
        t = self._torch
        if not self.segments:
            return t.empty((0, self.d), dtype=t.float32, device=self.ctx.device)
        if len(self.segments) == 1:
            return self.segments[0][: self.fill[0]]
        out = t.cat([s[:f] for s, f in zip(self.segments, self.fill)], dim=0)
        self.segments, self.fill = [], []
        return out
