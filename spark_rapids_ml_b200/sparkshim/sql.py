"""Local stand-in for the slice of the Spark SQL API the KMeans path drives (used only without pyspark).

A LocalDataFrame is a list of partitions, each a list of pyarrow RecordBatches of at most
spark.sql.execution.arrow.maxRecordsPerBatch rows — what a Spark Python worker receives over the Arrow IPC
socket.  mapInPandas hands the UDF an Iterator[pd.DataFrame] per partition exactly as Spark does; in barrier
mode each partition runs in its own spawned process (one process <-> one GPU, core.py:1005-1009) with a
BarrierTaskContext backed by a TCPStore.
"""
from __future__ import annotations

import os
import traceback
from typing import Any, Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import pandas as pd
import pyarrow as pa

from .barrier import BarrierTaskContext, free_port, make_store


class Row(dict):
    """pyspark.sql.Row subset: attribute + key access, asDict()."""

    def __getattr__(self, k: str) -> Any:
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def asDict(self) -> Dict[str, Any]:
        return dict(self)


class LocalSession:
    _active: Optional["LocalSession"] = None

    def __init__(self, conf: Optional[Dict[str, str]] = None, default_parallelism: Optional[int] = None):
        self.conf_map: Dict[str, str] = {"spark.sql.execution.arrow.maxRecordsPerBatch": "10000"}
        if conf:
            self.conf_map.update({k: str(v) for k, v in conf.items()})
        self.defaultParallelism = default_parallelism or max(1, os.cpu_count() or 1)
        LocalSession._active = self

    class _Conf:
        def __init__(self, m: Dict[str, str]):
            self._m = m

        def get(self, k: str, default: Optional[str] = None) -> Optional[str]:
            return self._m.get(k, default)

        def set(self, k: str, v: Any) -> None:
            self._m[k] = str(v)

        def unset(self, k: str) -> None:
            self._m.pop(k, None)

    @property
    def conf(self) -> "LocalSession._Conf":
        return LocalSession._Conf(self.conf_map)

    @property
    def max_records_per_batch(self) -> int:
        return int(self.conf_map.get("spark.sql.execution.arrow.maxRecordsPerBatch", "10000"))

    # -- constructors --
    def createDataFrame(self, data: Any, schema: Optional[Sequence[str]] = None, num_partitions: int = 1) -> "LocalDataFrame":
        if isinstance(data, pd.DataFrame):
            table = pa.Table.from_pandas(data, preserve_index=False)
        elif isinstance(data, pa.Table):
            table = data
        else:
            rows = list(data)
            types: List[Optional[pa.DataType]]
            if isinstance(schema, str):   # Spark DDL: "c1 int, c2 int" / "features array<float>, label float"
                names, types = _parse_ddl(schema)
            else:
                names = list(schema) if schema is not None else [f"_{i + 1}" for i in range(len(rows[0]))]
                types = [None] * len(names)
            cols = list(zip(*rows)) if rows else [[] for _ in names]
            arrays = []
            for c, t in zip(cols, types):
                c = list(c)
                if len(c) and hasattr(c[0], "toArray"):  # pyspark.ml.linalg vectors, if someone passes them
                    c = [v.toArray().tolist() for v in c]
                arrays.append(pa.array(c, type=t) if t is not None else pa.array(c))
            table = pa.Table.from_arrays(arrays, names=names)
        return LocalDataFrame(self, _split_table(table, num_partitions, self.max_records_per_batch), table.schema)

    def from_numpy(self, X: np.ndarray, col: str = "features", num_partitions: int = 1,
                   extra: Optional[Dict[str, np.ndarray]] = None) -> "LocalDataFrame":
        """[n,d] array -> one array<float|double> column (zero-copy list view of the buffer)."""
        X = np.ascontiguousarray(X)
        n, d = X.shape
        offsets = pa.array(np.arange(0, (n + 1) * d, d, dtype=np.int32))
        arr = pa.ListArray.from_arrays(offsets, pa.array(X.reshape(-1)))
        names, arrays = [col], [arr]
        for k, v in (extra or {}).items():
            names.append(k)
            arrays.append(pa.array(v))
        return LocalDataFrame(self, _split_table(pa.Table.from_arrays(arrays, names=names), num_partitions,
                                                 self.max_records_per_batch))


_DDL_TYPES = {"byte": pa.int8(), "tinyint": pa.int8(), "short": pa.int16(), "smallint": pa.int16(), "int": pa.int32(),
              "integer": pa.int32(), "long": pa.int64(), "bigint": pa.int64(), "float": pa.float32(), "real": pa.float32(),
              "double": pa.float64(), "string": pa.string(), "boolean": pa.bool_()}


def _parse_ddl(schema: str) -> Tuple[List[str], List[Optional[pa.DataType]]]:
    """The subset of Spark's DDL schema strings the KMeans tests use: `name type` pairs, scalar types and array<scalar>."""
    names: List[str] = []
    types: List[Optional[pa.DataType]] = []
    depth, start, fields = 0, 0, []
    for i, ch in enumerate(schema):   # split on commas outside <...>
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "," and depth == 0:
            fields.append(schema[start:i])
            start = i + 1
    fields.append(schema[start:])
    for f in fields:
        name, _, tname = f.strip().partition(" ")
        tname = tname.strip().lower()
        if tname.startswith("array<") and tname.endswith(">"):
            inner = _DDL_TYPES.get(tname[6:-1].strip())
            if inner is None:
                raise ValueError(f"unsupported element type in schema field '{f.strip()}'")
            t: Optional[pa.DataType] = pa.list_(inner)
        else:
            t = _DDL_TYPES.get(tname)
            if t is None:
                raise ValueError(f"unsupported type in schema field '{f.strip()}'")
        names.append(name)
        types.append(t)
    return names, types


def get_session() -> LocalSession:
    return LocalSession._active or LocalSession()


def _split_table(table: pa.Table, num_partitions: int, max_records: int) -> List[List[pa.RecordBatch]]:
    n = table.num_rows
    parts: List[List[pa.RecordBatch]] = []
    bounds = np.linspace(0, n, num_partitions + 1).astype(np.int64)
    for p in range(num_partitions):
        sub = table.slice(int(bounds[p]), int(bounds[p + 1] - bounds[p])).combine_chunks()
        parts.append(sub.to_batches(max_chunksize=max_records) if sub.num_rows else [])
    return parts


def _spark_type(t: pa.DataType) -> str:
    if pa.types.is_list(t) or pa.types.is_large_list(t) or pa.types.is_fixed_size_list(t):
        return f"array<{_spark_type(t.value_type)}>"
    return {pa.float32(): "float", pa.float64(): "double", pa.int8(): "tinyint", pa.int16(): "smallint",
            pa.int32(): "int", pa.int64(): "bigint", pa.string(): "string", pa.bool_(): "boolean"}.get(t, str(t))


def _batches_to_pdf_iter(batches: List[pa.RecordBatch], arrow_backed: bool) -> Iterator[pd.DataFrame]:
    cols_idx: Optional[pd.Index] = None
    for b in batches:
        if arrow_backed:
            # zero-copy: every column keeps its Arrow buffers (ArrowDtype).  The frame is assembled from the arrays with
            # ONE column Index shared by all batches of the partition: RecordBatch.to_pandas(types_mapper=...) spends
            # ~0.5 ms per batch on index / metadata handling, a dict-built frame ~0.2 ms, this ~0.05 ms
            if cols_idx is None or list(cols_idx) != b.schema.names:
                cols_idx = pd.Index(b.schema.names)
            arrs = [pd.arrays.ArrowExtensionArray(pa.chunked_array([b.column(i)])) for i in range(b.num_columns)]
            try:
                yield pd.DataFrame._from_arrays(arrs, columns=cols_idx, index=pd.RangeIndex(b.num_rows),
                                                verify_integrity=False)
            except (AttributeError, TypeError):   # private constructor moved: the public one
                yield pd.DataFrame(dict(zip(b.schema.names, arrs)), copy=False)
        else:
            yield b.to_pandas()                              # Spark's classic conversion: object column of ndarrays


def run_barrier_task(rank: int, world: int, port: int, payload_path: str, result_path: str) -> None:
    """Body of one barrier task process (entry: python -m spark_rapids_ml_b200.sparkshim._task)."""
    import cloudpickle

    try:
        with open(payload_path, "rb") as f:
            fn, batches, arrow_backed, conf = cloudpickle.load(f)
        LocalSession(conf)
        store = make_store(rank, world, port) if world > 1 else None
        BarrierTaskContext._install(BarrierTaskContext(rank, world, store))
        out = [pdf for pdf in fn(_batches_to_pdf_iter(batches, arrow_backed))]
        res = ("ok", out)
    except BaseException as e:  # noqa: BLE001 - report everything to the driver, Spark-style
        res = ("err", f"{type(e).__name__}: {e}\n{traceback.format_exc()}")
    with open(result_path, "wb") as f:
        cloudpickle.dump(res, f)


class LocalDataFrame:
    def __init__(self, session: LocalSession, partitions: List[List[pa.RecordBatch]], schema: Optional[pa.Schema] = None):
        self.sparkSession = session
        self._parts = partitions
        self._schema = schema
        if self._schema is None:
            for p in partitions:
                if p:
                    self._schema = p[0].schema
                    break
        # pandas conversion mode for mapInPandas: Arrow-backed columns (fast ingest path) or Spark-classic objects
        self.arrow_backed_pandas = True

    # -- metadata --
    @property
    def columns(self) -> List[str]:
        return list(self._schema.names) if self._schema is not None else []

    @property
    def dtypes(self) -> List[Tuple[str, str]]:
        return [(f.name, _spark_type(f.type)) for f in self._schema]

    @property
    def schema(self) -> pa.Schema:
        return self._schema

    def getNumPartitions(self) -> int:
        return len(self._parts)

    def count(self) -> int:
        return sum(b.num_rows for p in self._parts for b in p)

    def _table(self) -> pa.Table:
        batches = [b for p in self._parts for b in p]
        return pa.Table.from_batches(batches, schema=self._schema) if batches else self._schema.empty_table()

    def toPandas(self) -> pd.DataFrame:
        return self._table().to_pandas()

    def collect(self) -> List[Row]:
        t = self._table().to_pylist()
        return [Row(r) for r in t]

    def first(self) -> Optional[Row]:
        for p in self._parts:
            for b in p:
                if b.num_rows:
                    return Row(b.slice(0, 1).to_pylist()[0])
        return None

    head = first

    # -- transformations --
    def _derive(self, parts: List[List[pa.RecordBatch]], schema: Optional[pa.Schema] = None) -> "LocalDataFrame":
        df = LocalDataFrame(self.sparkSession, parts, schema)
        df.arrow_backed_pandas = self.arrow_backed_pandas
        return df

    def select(self, *cols: str) -> "LocalDataFrame":
        names = list(cols[0]) if len(cols) == 1 and isinstance(cols[0], (list, tuple)) else list(cols)
        parts = [[b.select(names) for b in p] for p in self._parts]
        return self._derive(parts, pa.schema([self._schema.field(n) for n in names]))

    def withColumnRenamed(self, old: str, new: str) -> "LocalDataFrame":
        names = [new if n == old else n for n in self.columns]
        parts = [[b.rename_columns(names) for b in p] for p in self._parts]
        return self._derive(parts)

    def cast_column(self, name: str, arrow_type: pa.DataType) -> "LocalDataFrame":
        """col(name).cast(type) for list/scalar numeric columns (what core.py:489-495,543-557 build)."""
        idx = self._schema.get_field_index(name)
        parts = []
        for p in self._parts:
            nb = []
            for b in p:
                arrs = list(b.columns)
                arrs[idx] = arrs[idx].cast(arrow_type)
                nb.append(pa.RecordBatch.from_arrays(arrs, names=b.schema.names))
            parts.append(nb)
        fields = list(self._schema)
        fields[idx] = pa.field(name, arrow_type)
        return self._derive(parts, pa.schema(fields))

    def repartition(self, n: int) -> "LocalDataFrame":
        return self._derive(_split_table(self._table(), n, self.sparkSession.max_records_per_batch), self._schema)

    def union(self, other: "LocalDataFrame") -> "LocalDataFrame":
        """DataFrame.union: the rows of both, matched by column position (names from this frame), partitions of this frame
        first.  The column counts and types must agree."""
        a, b = self._schema, other._schema
        if len(a) != len(b):
            raise ValueError(f"union needs the same number of columns: {len(a)} vs {len(b)}")
        for fa, fb in zip(a, b):
            if fa.type != fb.type:
                raise ValueError(f"union: column '{fa.name}' is {fa.type}, the other frame's '{fb.name}' is {fb.type}")
        theirs = [[pa.RecordBatch.from_arrays(bt.columns, schema=a) for bt in p] for p in other._parts]
        return self._derive(self._parts + theirs, a)

    def with_constant_column(self, name: str, value: int) -> "LocalDataFrame":
        """withColumn(name, lit(value)) for an integer literal (Spark types it int)."""
        parts = [[b.append_column(name, pa.array(np.full(b.num_rows, value, dtype=np.int32))) for b in p]
                 for p in self._parts]
        return self._derive(parts, self._schema.append(pa.field(name, pa.int32())))

    def with_monotonically_increasing_id(self, name: str) -> "LocalDataFrame":
        """select(monotonically_increasing_id().alias(name), "*"): Spark's id, partition_id << 33 | row in partition."""
        parts = []
        for pid, p in enumerate(self._parts):
            nb, row = [], 0
            for b in p:
                ids = (np.int64(pid) << np.int64(33)) + np.arange(row, row + b.num_rows, dtype=np.int64)
                nb.append(pa.RecordBatch.from_arrays([pa.array(ids)] + list(b.columns),
                                                     names=[name] + b.schema.names))
                row += b.num_rows
            parts.append(nb)
        return self._derive(parts, pa.schema([pa.field(name, pa.int64())] + list(self._schema)))

    def with_appended_column(self, name: str, per_partition_arrays: List[List[pa.Array]]) -> "LocalDataFrame":
        parts = []
        for p, arrs in zip(self._parts, per_partition_arrays):
            parts.append([b.append_column(name, a) for b, a in zip(p, arrs)])
        return self._derive(parts)

    # -- actions with UDFs --
    def mapInPandas(self, fn: Callable[[Iterator[pd.DataFrame]], Iterator[pd.DataFrame]], schema: Any = None,
                    barrier: bool = False) -> "LocalDataFrame":
        """Evaluate fn per partition. barrier=True: one spawned process per partition, all running concurrently
        (Spark barrier stage); with a single partition the task runs in-process."""
        nparts = len(self._parts)
        results: List[List[pd.DataFrame]] = []
        if not barrier or nparts == 1:
            for pid, p in enumerate(self._parts):
                if barrier:
                    BarrierTaskContext._install(BarrierTaskContext(pid, nparts, None))
                try:
                    results.append([pdf for pdf in fn(_batches_to_pdf_iter(p, self.arrow_backed_pandas))])
                finally:
                    if barrier:
                        BarrierTaskContext._install(None)
        else:
            import subprocess
            import sys
            import tempfile

            import cloudpickle

            port = free_port()
            tmp = tempfile.mkdtemp(prefix="b2k_barrier_")
            procs = []
            root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
            env = dict(os.environ)
            env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
            for pid, p in enumerate(self._parts):
                pay, res = os.path.join(tmp, f"task{pid}.in"), os.path.join(tmp, f"task{pid}.out")
                with open(pay, "wb") as f:
                    cloudpickle.dump((fn, p, self.arrow_backed_pandas, dict(self.sparkSession.conf_map)), f)
                procs.append((subprocess.Popen([sys.executable, "-m", "spark_rapids_ml_b200.sparkshim._task",
                                                str(pid), str(nparts), str(port), pay, res], env=env), res))
            # Spark fails the whole barrier stage as soon as one task fails: poll all tasks and kill the survivors, which
            # may be blocked in a collective waiting for the dead peer (reference: core.py:975-981, cuml_context.py:163-167)
            import time as _time

            deadline = _time.monotonic() + 1800
            failed = False
            while True:
                codes = [pr.poll() for pr, _ in procs]
                if any(c is not None and c != 0 for c in codes):
                    failed = True
                if all(c is not None for c in codes):
                    break
                # a task that wrote an error result is as good as dead even if it is still tearing down
                if not failed:
                    for _, res in procs:
                        if os.path.exists(res):
                            try:
                                with open(res, "rb") as f:
                                    if cloudpickle.load(f)[0] != "ok":
                                        failed = True
                            except Exception:
                                pass   # still being written
                if failed or _time.monotonic() > deadline:
                    grace = _time.monotonic() + 5.0
                    while _time.monotonic() < grace and any(pr.poll() is None for pr, _ in procs):
                        _time.sleep(0.05)
                    for pr, _ in procs:
                        if pr.poll() is None:
                            pr.kill()
                    for pr, _ in procs:
                        pr.wait()
                    break
                _time.sleep(0.02)
            errors = []
            for pid, (pr, res) in enumerate(procs):
                status, val = "err", f"barrier task {pid} was killed with the failed stage or died without a result (exit code {pr.returncode})"
                if os.path.exists(res):
                    try:
                        with open(res, "rb") as f:
                            status, val = cloudpickle.load(f)
                    except Exception:
                        pass
                if status == "ok":
                    results.append(val)
                else:
                    errors.append(f"[task {pid}] {val}")
                    results.append([])
            import shutil

            shutil.rmtree(tmp, ignore_errors=True)
            if errors:  # Spark fails the whole barrier stage
                raise RuntimeError("barrier stage failed:\n" + "\n".join(errors))
        parts = []
        for r in results:
            parts.append([pa.RecordBatch.from_pandas(pdf, preserve_index=False) for pdf in r if len(pdf)])
        return LocalDataFrame(self.sparkSession, parts)
