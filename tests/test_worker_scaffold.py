"""The N>1 host path on CPU: the barrier-task scaffolding (one process per partition, BarrierTaskContext
allGather/barrier over a TCPStore, rank-0-only result, loud failure of the whole stage) exercised with a FAKE
backend — the counterpart of the reference's CumlDummy/SparkRapidsMLDummy scaffolding test
(python/tests/test_common_estimator.py:46-318, 486-583) — plus a world_size-2 gloo check of the row-sharded
partial-sum + allreduce arithmetic the GPU ranks perform."""
import numpy as np
import pandas as pd
import pytest

from spark_rapids_ml_b200.sparkshim import BarrierTaskContext, LocalSession


def _rows(n, d, seed=0):
    return np.random.default_rng(seed).normal(size=(n, d)).astype(np.float32)


def test_barrier_stage_two_processes_rank0_yields():
    s = LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "7"})
    X = _rows(50, 3)
    df = s.from_numpy(X, num_partitions=2)

    def udf(it):
        ctx = BarrierTaskContext.get()
        rank = ctx.partitionId()
        sizes = [len(p) for p in it]
        assert max(sizes) <= 7                       # Arrow batches honour maxRecordsPerBatch
        msgs = ctx.allGather(f"{rank}:{sum(sizes)}")  # NCCL-uid style rendezvous
        ctx.barrier()
        if rank == 0:
            yield pd.DataFrame({"ranks": [",".join(sorted(msgs))], "batches": [len(sizes)]})

    out = df.mapInPandas(udf, barrier=True).toPandas()
    assert out["ranks"][0] == "0:25,1:25" and len(out) == 1


def test_barrier_stage_failure_is_loud():
    s = LocalSession()
    df = s.from_numpy(_rows(10, 2), num_partitions=2)

    def udf(it):
        ctx = BarrierTaskContext.get()
        list(it)
        if ctx.partitionId() == 1:
            raise RuntimeError("A python worker received no data.  Please increase amount of data or use fewer workers.")
        yield pd.DataFrame({"ok": [1]})

    with pytest.raises(RuntimeError, match="barrier stage failed"):
        df.mapInPandas(udf, barrier=True)


def test_barrier_stage_failure_kills_blocked_peers_quickly():
    """A task that fails while its peer is blocked in a rendezvous (the NCCL-collective situation) must fail the whole
    stage within seconds: the driver kills the survivors instead of waiting out their time-outs
    (reference behaviour: core.py:975-981, cuml_context.py:163-167)."""
    import time

    s = LocalSession()
    df = s.from_numpy(_rows(10, 2), num_partitions=2)

    def udf(it):
        ctx = BarrierTaskContext.get()
        list(it)
        if ctx.partitionId() == 1:
            raise RuntimeError("rank 1 fails before the rendezvous")
        ctx.allGather("rank 0 waits for a peer that never arrives")   # blocks (TCPStore time-out: 300 s)
        yield pd.DataFrame({"ok": [1]})

    t0 = time.monotonic()
    with pytest.raises(RuntimeError, match="barrier stage failed"):
        df.mapInPandas(udf, barrier=True)
    assert time.monotonic() - t0 < 60


def test_pandas_conversion_modes_and_arrow_fast_path():
    """Arrow-backed columns expose the list child buffer zero-copy; the classic object-column conversion takes the
    stacking path — both must describe the same [n_b, d] values."""
    from spark_rapids_ml_b200.core import alias
    from spark_rapids_ml_b200.utils import arrow_list_column_buffers

    s = LocalSession()
    X = _rows(9, 4, seed=3)
    df = s.from_numpy(X, col=alias.data)
    batch = df._parts[0][0]
    fast = batch.to_pandas(types_mapper=pd.ArrowDtype)
    vals, offsets, n = arrow_list_column_buffers(fast[alias.data])
    assert n == 9 and np.shares_memory(vals, batch.column(0).values.to_numpy(zero_copy_only=True))
    np.testing.assert_array_equal(vals[offsets[0]:offsets[-1]].reshape(9, 4), X)
    classic = batch.to_pandas()
    assert arrow_list_column_buffers(classic[alias.data]) is None
    np.testing.assert_array_equal(np.array(list(classic[alias.data])), X)


def _gloo_worker(rank, world, port, q):
    import os

    import torch
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import kmeans_oracle as ko

    X, _ = ko.make_blobs(4000, 8, 5, seed=2)
    C0 = X[:5].copy()
    part = np.array_split(X, world)[rank]
    C = C0.copy()
    for _ in range(6):  # what every GPU rank does per iteration: local partial sums, ONE fused allreduce, finalize
        lab, md, _ = ko.assign(part, C)
        S, w = ko.partial_sums(part, lab, 5)
        buf = torch.from_numpy(np.concatenate([S.reshape(-1), w, [md.sum()]]))
        dist.all_reduce(buf)
        S = buf[:40].numpy().reshape(5, 8)
        w = buf[40:45].numpy()
        Cn = C.astype(np.float64)
        Cn[w > 0] = S[w > 0] / w[w > 0][:, None]
        C = Cn.astype(np.float32)
    q.put((rank, C))
    dist.destroy_process_group()


def test_world_size_2_gloo_row_sharding_matches_single_rank():
    import torch.multiprocessing as mp

    from oracle import kmeans_oracle as ko
    from spark_rapids_ml_b200.sparkshim.barrier import free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    X, _ = ko.make_blobs(4000, 8, 5, seed=2)
    ref = ko.lloyd([X], X[:5].copy(), 6, -1.0)
    np.testing.assert_array_equal(got[0], got[1])            # replicas stay identical without a broadcast
    np.testing.assert_array_equal(got[0], ref["centers"])    # and equal the single-rank oracle exactly


def test_grouped_transform_sees_batches_in_row_and_byte_capped_groups_in_order():
    """core._iter_transform: a model's grouped transform function sees consecutive batches in groups bounded by rows
    and bytes; results come back one per batch, in order."""
    import pandas as pd
    from spark_rapids_ml_b200 import core

    frames = [pd.DataFrame({"a": range(i * 10, i * 10 + n)}) for i, n in enumerate([3, 0, 5, 2, 7, 1])]
    calls = []

    def many(model, fs):
        calls.append(("many", [len(f) for f in fs]))
        return [pd.Series(f["a"].to_numpy() + model) for f in fs]

    want = [list(f["a"] + 100) for f in frames]
    many.row_bytes = 8
    old = core.TRANSFORM_GROUP_ROWS, core.TRANSFORM_GROUP_BYTES
    try:
        core.TRANSFORM_GROUP_ROWS, core.TRANSFORM_GROUP_BYTES = 8, 1 << 30
        assert [list(r) for r in core._iter_transform(many, 100, iter(frames))] == want
        assert calls == [("many", [3, 0, 5]), ("many", [2, 7]), ("many", [1])]
        del calls[:]
        core.TRANSFORM_GROUP_ROWS, core.TRANSFORM_GROUP_BYTES = 1 << 20, 8 * 4      # the byte cap: 4 rows per group
        assert [list(r) for r in core._iter_transform(many, 100, iter(frames))] == want
        assert calls == [("many", [3, 0, 5]), ("many", [2, 7]), ("many", [1])]
    finally:
        core.TRANSFORM_GROUP_ROWS, core.TRANSFORM_GROUP_BYTES = old
