"""The ingest path every estimator's rows take (Arrow batch -> DeviceRowAppender / DeviceCsrAppender ->
b2k_ingest_append / b2k_ingest_csr_append -> k_convert_rows, k_transpose_cols, k_csr_ingest through two pinned and
device staging slots) against the host conversion, bit for bit.

The rule is the same everywhere: the device matrix equals np.asarray(src).astype(np.float32), NaN positions compared
by isnan (the device's cvt writes the canonical NaN, the host keeps the payload) and every other entry by its float32
bits.  The kernels convert with plain (float)v casts, round to nearest even, and the library is built without fast-math
or flush-to-zero, so this holds exactly, fp32 subnormals and int64 rounding included.

The batch sizes that turn the staging slots over are derived from the library's staging constants below."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STAGE_BYTES = 64 << 20          # one staging slot (pinned and device), csrc/b2k_ingest.cu
ERR_UNSUPPORTED = 4             # B2K_ERR_UNSUPPORTED
DTYPES = [np.float32, np.float64, np.int8, np.int16, np.int32, np.int64]
F32 = np.finfo(np.float32)
SENTINEL = np.float32(-7.25)


def slot_elems(es):
    """Elements of an es-byte type one slot takes in the row layout (a multiple of 4)."""
    per = STAGE_BYTES // es
    return per - per % 4


def col_chunk(d, es):
    """Rows of d es-byte columns one slot takes in the column layout (a multiple of 32)."""
    rows = STAGE_BYTES // (d * es)
    return rows - rows % 32


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _launches(ctx, fn):
    """fn() run with the context's kernel-launch count reset -> launches it made."""
    ctx.reset_stats()
    fn()
    return ctx.stats()["kernel_launches"]


def _assert_f32(got, src):
    """got (a CUDA or host float32 array) is np.asarray(src).astype(np.float32), bit for bit, NaN by isnan."""
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    with np.errstate(over="ignore"):
        want = np.asarray(src).astype(np.float32)
    assert got.dtype == np.float32 and got.shape == want.shape, (got.dtype, got.shape, want.shape)
    nan = np.isnan(want)
    bad = np.isnan(got) != nan
    assert not bad.any(), f"NaN positions differ at {np.argwhere(bad)[:5].tolist()}"
    g, w = got[~nan].view(np.uint32), want[~nan].view(np.uint32)
    if not np.array_equal(g, w):
        i = np.flatnonzero(g != w)[:5]
        raise AssertionError(f"{i.size}+ entries differ, e.g. at {i.tolist()}: got {got[~nan][i]} want {want[~nan][i]} "
                             f"from {np.asarray(src)[~nan][i]}")


def _f64_edges():
    """float64 values at every edge of the conversion to float32."""
    tiny = float(F32.smallest_subnormal)                     # 2^-149
    fmin, fmax = float(F32.tiny), float(F32.max)
    half_ulp_max = 2.0 ** 103                                # half of float32's ulp at FLT_MAX
    e = [
        # round to nearest even at 1: halfway down to even, halfway up to even, just above halfway
        1 + 2.0**-24, 1 + 3 * 2.0**-24, 1 + 2.0**-24 + 2.0**-50, 1 + 2.0**-24 - 2.0**-52,
        # subnormal range: halfway to 0 and to the smallest subnormal, below, between subnormals, the largest one
        tiny / 2, tiny * 1.5, tiny * 0.49, tiny * 2.5, tiny * 3.5, fmin - tiny, fmin - tiny / 2, fmin - tiny * 0.51,
        np.nextafter(fmin, 0.0), fmin, np.nextafter(tiny / 2, 1.0), np.nextafter(tiny / 2, 0.0),
        float(np.finfo(np.float64).smallest_subnormal), float(np.finfo(np.float64).tiny),
        # FLT_MAX neighbours: exact, just below the halfway point to 2^128, the halfway point (-> inf), above
        fmax, fmax + half_ulp_max - 2.0**75, fmax + half_ulp_max, fmax + half_ulp_max * 1.5, np.nextafter(fmax, np.inf),
        float(np.finfo(np.float64).max), 1e39,
        0.0, -0.0, np.inf, -np.inf, np.nan, 16777217.0, 2.0**60 + 2.0**36,
    ]
    e = np.array(e, dtype=np.float64)
    return np.concatenate([e, -e])


def _edges(dt):
    dt = np.dtype(dt)
    if dt == np.float64:
        return _f64_edges()
    if dt == np.float32:
        return np.array([0.0, -0.0, F32.smallest_subnormal, -F32.smallest_subnormal, F32.tiny, F32.max, -F32.max,
                         np.inf, -np.inf, np.nan, 1.5], dtype=np.float32)
    info = np.iinfo(dt)
    e = [info.min, info.max, info.min + 1, info.max - 1, 0, -1, 1]
    if info.bits >= 32:
        # above 2^24 a float32 holds every value only to its ulp: halfway points round to even, others to nearest
        e += [2**24 + 1, 2**24 + 3, 2**25 + 2, 2**25 + 6, 2**31 - 1, -2**31, -(2**24 + 1), 2**31 - 64, 2**31 - 65]
    if info.bits == 64:
        e += [2**53 + 2**29 + 1, 2**53 + 1, 2**62 + 2**38, 2**62 + 2**38 + 1, 2**63 - 2**39, 2**63 - 2**39 - 1,
              -(2**63 - 2**39), 2**40 - 2**16 - 1, -(2**53 + 2**29 + 1)]
    return np.array(e, dtype=dt)


def _values(dt, count, seed):
    """count values of dt: its edges first, then random values over its whole range (float32: random bit patterns,
    subnormals and NaNs among them; float64: random magnitudes across and beyond float32's range)."""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dt)
    if dt == np.float32:
        rest = rng.integers(0, 2**32, size=count, dtype=np.uint64).astype(np.uint32).view(np.float32)
    elif dt == np.float64:
        rest = rng.normal(size=count) * 10.0 ** rng.uniform(-48, 41, size=count)
    else:
        info = np.iinfo(dt)
        rest = rng.integers(info.min, info.max, size=count, dtype=dt, endpoint=True)
    e = _edges(dt)[:count]
    rest[: e.size] = e
    return rest


def _dst(n, d):
    return torch.full((n, d), float(SENTINEL), dtype=torch.float32, device="cuda")


def _assert_rows(dst, row0, src_rows):
    """dst[row0:row0 + n] is src_rows as float32 bits; every other row still holds the sentinel."""
    torch.cuda.synchronize()
    host = dst.cpu().numpy()
    n = src_rows.shape[0]
    _assert_f32(host[row0:row0 + n], src_rows)
    assert (host[:row0] == SENTINEL).all() and (host[row0 + n:] == SENTINEL).all()


# ---- rows -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("n,d,row0", [(1000, 7, 0),     # 16-byte aligned destination, n * d = 7000: vector stores
                                      (333, 5, 0),      # aligned, n * d = 1665: one scalar element after the vectors
                                      (7, 3, 0),        # aligned, n * d = 21: a 1-element tail after 5 vector stores
                                      (2, 3, 0),        # aligned, n * d = 6: a 2-element tail after one vector store
                                      (333, 5, 3),      # row0 * d odd: every store on the scalar branch
                                      (7, 3, 1),        # row0 * d = 3: misaligned, scalar stores only
                                      (1, 1, 2)])
def test_rows_every_type_at_the_conversion_edges(ctx, dt, n, d, row0):
    """Every type at its conversion edges, on both store branches of k_convert_rows.  An aligned destination with a
    count that is not a multiple of 4 ends in a scalar tail; the sentinel rows after the batch catch a 16-byte store
    that runs past it."""
    src = _values(dt, n * d, seed=n + d).reshape(n, d)
    dst = _dst(row0 + n + 2, d)
    assert ctx.ingest_rows(dst, row0, src.reshape(-1), d) == n
    _assert_rows(dst, row0, src)


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.int16], ids=lambda t: np.dtype(t).name)
def test_rows_from_a_sliced_list_array(ctx, dt):
    """Offsets that start past 0: the batch is rows [11, 48) of a list array, whose child buffer holds all 60 rows."""
    d = 6
    full = _values(dt, 60 * d, seed=3)
    lists = pa.ListArray.from_arrays(pa.array(np.arange(61, dtype=np.int32) * d), pa.array(full)).slice(11, 37)
    offsets = lists.offsets.to_numpy()
    assert offsets[0] == 11 * d
    dst = _dst(40, d)
    assert ctx.ingest_rows(dst, 1, lists.values.to_numpy(), d, offsets=offsets) == 37
    _assert_rows(dst, 1, full.reshape(60, d)[11:48])


def test_empty_row_batches_write_nothing(ctx):
    dst = _dst(4, 3)
    assert ctx.ingest_rows(dst, 4, np.zeros(0, np.float64), 3) == 0                  # at the end of dst
    assert ctx.ingest_rows(dst, 1, np.arange(9.0), 3, offsets=np.array([6], np.int32)) == 0   # offsets of no row
    assert ctx.ingest_columns(dst, 2, [np.zeros(0, np.int16)] * 3) == 0
    _assert_rows(dst, 0, np.zeros((0, 3)))


@pytest.mark.parametrize("dt,d,row0", [(np.float64, 3, 0), (np.float64, 3, 1), (np.float32, 5, 0)],
                         ids=["f64", "f64-misaligned", "f32-pageable"])
def test_rows_over_several_staging_slots(ctx, dt, d, row0):
    """A batch of 2.5 slots and a few rows: three chunks, so both slots turn over.  float64 at row0 = 0: every chunk
    starts 16-byte aligned (a slot holds a multiple of 4 elements), the grid-stride loop stores vectors and the last
    chunk ends in a scalar tail; at row0 = 1 every store of every chunk is scalar.  float32 rows are copied through the
    pinned slot and launch no kernel."""
    per = slot_elems(np.dtype(dt).itemsize)
    n = (5 * per // 2) // d + 3
    src = _values(dt, n * d, seed=11).reshape(n, d)
    dst = _dst(row0 + n + 2, d)
    launches = _launches(ctx, lambda: ctx.ingest_rows(dst, row0, src.reshape(-1), d))
    chunks = -(-n * d // per)
    assert chunks == 3 and (n * d - (chunks - 1) * per) % 4 != 0
    assert launches == (0 if dt == np.float32 else chunks)
    _assert_rows(dst, row0, src)


# ---- pinned sources ---------------------------------------------------------------------------------------------------
def test_pinned_float32_tensor(ctx):
    """A page-locked float32 tensor takes the zero-staging copy.  Only its values are checked: a float32 source launches
    no kernel on the staged path either, so no counter tells the two paths apart."""
    n, d = 4097, 9
    src = torch.from_numpy(_values(np.float32, n * d, seed=5).reshape(n, d)).pin_memory()
    dst = _dst(n + 3, d)
    assert _launches(ctx, lambda: ctx.ingest_pinned_tensor(dst, 3, src)) == 0
    _assert_rows(dst, 3, src.numpy())


def test_pinned_float32_rows_with_offsets(ctx):
    """A page-locked child buffer with offsets past 0: the (zero-staging) copy starts at offsets[0].  Only the values
    are checked, as above."""
    d = 4
    buf = torch.from_numpy(_values(np.float32, 300 * d, seed=6)).pin_memory()
    offsets = (np.arange(101, 251, dtype=np.int32) * d)
    dst = _dst(150, d)
    assert ctx.ingest_rows(dst, 1, buf.numpy(), d, offsets=offsets) == 149
    _assert_rows(dst, 1, buf.numpy().reshape(300, d)[101:250])


def test_pinned_float64_rows_over_two_slots(ctx):
    """Page-locked non-float32 rows go to the device staging slot straight from the caller's buffer, chunk by
    chunk."""
    d = 3
    n = (3 * slot_elems(8) // 2) // d + 1
    buf = torch.from_numpy(_values(np.float64, n * d, seed=7)).pin_memory()
    dst = _dst(n + 1, d)
    assert _launches(ctx, lambda: ctx.ingest_rows(dst, 1, buf.numpy(), d)) == 2
    _assert_rows(dst, 1, buf.numpy().reshape(n, d))


# ---- columns ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=lambda t: np.dtype(t).name)
def test_columns_every_type_and_width(ctx, dt):
    """d scalar columns -> row-major rows through the 32 x 32 tile transpose, at widths and row counts on both sides
    of a tile, at a nonzero row0."""
    for d in (1, 31, 32, 33, 100):
        for n in (1, 31, 33, 1000):
            src = _values(dt, n * d, seed=d * n).reshape(d, n)
            dst = _dst(n + 7, d)
            assert ctx.ingest_columns(dst, 5, list(src)) == n
            _assert_rows(dst, 5, src.T)


def test_columns_over_several_staging_chunks(ctx):
    d = 7
    rows = col_chunk(d, 8)
    n = 2 * rows + 1001
    cols = [_values(np.float64, n, seed=20 + c) for c in range(d)]
    dst = _dst(n + 2, d)
    assert _launches(ctx, lambda: ctx.ingest_columns(dst, 2, cols)) == 3
    _assert_rows(dst, 2, np.stack(cols, axis=1))


def test_columns_too_wide_for_a_staging_chunk_are_refused(ctx):
    from spark_rapids_ml_b200._native import B2KError

    d = 2**18 + 1
    assert col_chunk(d, 8) < 32 <= col_chunk(d - 1, 8)
    col = np.zeros(1, np.float64)
    with pytest.raises(B2KError, match="d too large for staging") as e:
        ctx.ingest_columns(torch.empty((1, d), dtype=torch.float32, device="cuda"), 0, [col] * d)
    assert e.value.code == ERR_UNSUPPORTED


# ---- CSR vector rows --------------------------------------------------------------------------------------------------
VECTOR = lambda vt: pa.struct([("type", pa.int8()), ("size", pa.int32()), ("indices", pa.list_(pa.int32())),  # noqa
                               ("values", pa.list_(vt))])


def _vectors(n, d, dt, seed, dense_every=5, empty_every=7, per_row=None):
    """n Spark vector rows of width d as a struct array: every dense_every-th row dense, every empty_every-th row
    sparse with no entries, the rest sparse with up to per_row entries at sorted random columns."""
    rng = np.random.default_rng(seed)
    per_row = per_row or max(1, d // 3)
    types, lens = np.zeros(n, np.int8), np.zeros(n, np.int64)
    idx = []
    for i in range(n):
        if dense_every and i % dense_every == 0:
            types[i], lens[i] = 1, d
            idx.append(np.zeros(0, np.int32))
        elif empty_every and i % empty_every == 0:
            idx.append(np.zeros(0, np.int32))
        else:
            k = int(rng.integers(1, per_row + 1))
            idx.append(np.sort(rng.choice(d, size=k, replace=False)).astype(np.int32))
            lens[i] = k
    vo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    io = np.concatenate([[0], np.cumsum([a.size for a in idx])]).astype(np.int32)
    dense = types == 1
    return pa.StructArray.from_arrays(
        [pa.array(types), pa.array(np.full(n, d, np.int32), mask=dense),
         pa.ListArray.from_arrays(pa.array(io), pa.array(np.concatenate(idx).astype(np.int32)),
                                  mask=pa.array(dense)),
         pa.ListArray.from_arrays(pa.array(vo), pa.array(_values(dt, int(vo[-1]), seed)))],
        fields=list(VECTOR(pa.from_numpy_dtype(np.dtype(dt)))))


def _host_csr(arr, d):
    """The host CSR of a (possibly sliced) vector struct array, values kept in their own dtype."""
    t, _, idx, val = arr.flatten()
    types = t.to_numpy(zero_copy_only=False)
    vo, vv = val.offsets.to_numpy(), val.values.to_numpy()
    io, iv = idx.offsets.to_numpy(), idx.values.to_numpy()
    cols = [np.arange(vo[i + 1] - vo[i], dtype=np.int32) if types[i] == 1 else iv[io[i]:io[i + 1]]
            for i in range(len(arr))]
    indices = np.concatenate(cols) if cols else np.zeros(0, np.int32)
    return sp.csr_matrix((vv[vo[0]:vo[-1]], indices, (vo - vo[0]).astype(np.int64)), shape=(len(arr), d))


def _series(arr):
    return pd.Series(pd.arrays.ArrowExtensionArray(pa.chunked_array([arr])))


def _assert_csr(got, want):
    indptr, indices, values = (x.cpu().numpy() for x in got)
    np.testing.assert_array_equal(indptr, want.indptr)
    np.testing.assert_array_equal(indices, want.indices)
    _assert_f32(values, want.data)


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_csr_rows_dense_sparse_empty_and_sliced(ctx, dt):
    from spark_rapids_ml_b200.utils import DeviceCsrAppender

    d = 37
    full = _vectors(300, d, dt, seed=31)
    batches = [full.slice(0, 100), full.slice(113, 150), full.slice(290, 10)]   # nonzero struct offsets
    app = DeviceCsrAppender(ctx, d)
    for b in batches:
        assert app.append_column(_series(b)) == len(b)
    _assert_csr(app.finish(), sp.vstack([_host_csr(b, d) for b in batches], format="csr"))


def test_csr_many_batches_grow_the_appender(ctx):
    from spark_rapids_ml_b200.utils import DeviceCsrAppender

    d = 64
    batches = [_vectors(int(n), d, np.float64, seed=40 + i, dense_every=3)
               for i, n in enumerate(np.random.default_rng(4).integers(1, 90, size=40))]
    app = DeviceCsrAppender(ctx, d, first_rows=3, first_nnz=5)
    for b in batches:
        app.append_column(_series(b))
    assert app.indptr.shape[0] > 4 and app.values.shape[0] > 5
    _assert_csr(app.finish(), sp.vstack([_host_csr(b, d) for b in batches], format="csr"))


def _csr_chunks(io, vo, es):
    """The library's split of one CSR batch over staging slots: halve the row range until its buffers fit a slot."""
    al = lambda b: (b + 15) // 16 * 16   # noqa: E731
    size = lambda r, r1: (al(r1 - r) + 2 * al(4 * (r1 - r + 1)) + al(4 * int(io[r1] - io[r]))   # noqa: E731
                          + al(es * int(vo[r1] - vo[r])))
    cuts, r, n = [], 0, len(vo) - 1
    while r < n:
        r1 = n
        while r1 > r + 1 and size(r, r1) > STAGE_BYTES:
            r1 = r + (r1 - r) // 2
        cuts.append(r1)
        r = r1
    return cuts


def test_csr_batch_over_several_staging_slots(ctx):
    """About 12 M float64 entries in one batch: the library cuts it into row ranges that fit a slot; indptr must run on
    across every cut."""
    from spark_rapids_ml_b200.utils import DeviceCsrAppender, arrow_vector_column_buffers

    d, n = 4096, 60000
    arr = _vectors(n, d, np.float64, seed=50, dense_every=97, empty_every=11, per_row=380)
    bufs = arrow_vector_column_buffers(_series(arr))
    cuts = _csr_chunks(bufs[2], bufs[4], 8)
    assert len(cuts) >= 3 and bufs[4][-1] > 10_000_000, (cuts, bufs[4][-1])
    app = DeviceCsrAppender(ctx, d)
    assert _launches(ctx, lambda: app.append_column(_series(arr))) == len(cuts)
    want = _host_csr(arr, d)
    _assert_csr(app.finish(), want)
    indptr = app.finish()[0].cpu().numpy()
    for c in cuts:
        assert indptr[c] == want.indptr[c]


def test_csr_dense_row_larger_than_a_slot_is_refused(ctx):
    """A dense float64 row of d values takes 48 bytes of type and offsets beside its values: the widest row that fits a
    slot is ingested, one value more is refused."""
    from spark_rapids_ml_b200._native import B2KError
    from spark_rapids_ml_b200.utils import DeviceCsrAppender

    fits = (STAGE_BYTES - 48) // 8
    for d, ok in ((fits, True), (fits + 1, False)):
        vals = _values(np.float64, d, seed=d)
        arr = pa.StructArray.from_arrays(
            [pa.array([1], pa.int8()), pa.array([None], pa.int32()), pa.array([None], pa.list_(pa.int32())),
             pa.ListArray.from_arrays(pa.array([0, d], pa.int32()), pa.array(vals))], fields=list(VECTOR(pa.float64())))
        app = DeviceCsrAppender(ctx, d, first_rows=1, first_nnz=d)
        if ok:
            app.append_column(_series(arr))
            _assert_csr(app.finish(), _host_csr(arr, d))
        else:
            with pytest.raises(B2KError, match="one row exceeds the staging buffer") as e:
                app.append_column(_series(arr))
            assert e.value.code == ERR_UNSUPPORTED
        del app
        torch.cuda.empty_cache()


# ---- the entry points interleaved on one context -----------------------------------------------------------------------
def test_rows_columns_and_csr_interleaved(ctx):
    """Small f64 rows, i16 columns and f64 CSR batches alternately: each call takes the next staging slot whatever
    layout used it last."""
    from spark_rapids_ml_b200.utils import DeviceCsrAppender

    d = 10
    rows_dst, cols_dst = _dst(3 * 50, d), _dst(3 * 40, d)
    app = DeviceCsrAppender(ctx, d, first_rows=4, first_nnz=8)
    rows, cols, vecs = [], [], []
    for i in range(3):
        rows.append(_values(np.float64, 50 * d, seed=60 + i).reshape(50, d))
        cols.append(_values(np.int16, 40 * d, seed=70 + i).reshape(d, 40))
        vecs.append(_vectors(30, d, np.float64, seed=80 + i))
        ctx.ingest_rows(rows_dst, 50 * i, rows[-1].reshape(-1), d)
        ctx.ingest_columns(cols_dst, 40 * i, list(cols[-1]))
        app.append_column(_series(vecs[-1]))
    _assert_rows(rows_dst, 0, np.concatenate(rows))
    _assert_rows(cols_dst, 0, np.concatenate([c.T for c in cols]))
    _assert_csr(app.finish(), sp.vstack([_host_csr(v, d) for v in vecs], format="csr"))


# ---- the Python layer -------------------------------------------------------------------------------------------------
def test_arrow_list_buffers_of_sliced_and_chunked_columns(ctx):
    from spark_rapids_ml_b200.utils import DeviceRowAppender, arrow_list_column_buffers

    d = 5
    full = _values(np.float64, 400 * d, seed=90)
    lists = pa.ListArray.from_arrays(pa.array(np.arange(401, dtype=np.int32) * d), pa.array(full))
    fixed = pa.FixedSizeListArray.from_arrays(pa.array(full), d)
    cases = [(pd.Series(pd.arrays.ArrowExtensionArray(pa.chunked_array([lists.slice(17, 200)]))), full[17 * d:217 * d]),
             (pd.Series(pd.arrays.ArrowExtensionArray(pa.chunked_array([fixed.slice(33, 150)]))), full[33 * d:183 * d]),
             (pd.Series(pd.arrays.ArrowExtensionArray(pa.chunked_array([lists.slice(0, 90), lists.slice(250, 100),
                                                                        lists.slice(90, 1)]))),
              np.concatenate([full[:90 * d], full[250 * d:350 * d], full[90 * d:91 * d]]))]
    for series, want in cases:
        vals, offsets, n = arrow_list_column_buffers(series, d)
        assert n == want.size // d
        app = DeviceRowAppender(ctx, d, first_capacity=1)
        app.append_values(vals, offsets, n)
        torch.cuda.synchronize()
        _assert_f32(app.finish(), want.reshape(-1, d))


def test_row_appender_concatenates_its_segments(ctx):
    """A small first capacity: the appender opens segments of 1024, 2048, 4096 rows and finish() joins them."""
    from spark_rapids_ml_b200.utils import DeviceRowAppender

    d = 3
    app = DeviceRowAppender(ctx, d, first_capacity=1)
    batches = [_values(dt, 700 * d, seed=100 + i).reshape(700, d)
               for i, dt in enumerate([np.float64, np.int64, np.float32, np.int8, np.float64, np.int32])]
    for b in batches:
        app.append_values(b.reshape(-1), None, b.shape[0])
    assert len(app.segments) == 3 and app.rows == 4200
    torch.cuda.synchronize()
    with np.errstate(over="ignore"):
        want = np.concatenate([b.astype(np.float32) for b in batches])
    _assert_f32(app.finish(), want)


# ---- estimators on mixed-type feature columns -------------------------------------------------------------------------
MIXED = [("a", pa.int64()), ("b", pa.float64()), ("c", pa.int8()), ("d", pa.float32())]


def _mixed_frames(n, seed, wide, parts=2):
    """The same rows twice: as scalar columns of mixed Arrow types, and as one array<double> column.  wide: the
    integer columns span int8 and +-2^24 (the most Arrow's safe cast to float32 in fit accepts) and the double column
    six decades; otherwise all four columns are of the same small scale, so that truncating the double column moves
    rows across cluster boundaries.  Every value is exact in float64."""
    from spark_rapids_ml_b200.sparkshim import LocalSession

    rng = np.random.default_rng(seed)
    lim = (2**24, 128) if wide else (4, 4)
    a = rng.integers(-lim[0], lim[0], size=n)
    b = rng.normal(size=n) * (10.0 ** rng.uniform(-3, 3, size=n) if wide else 2.0)
    c = rng.integers(-lim[1], lim[1], size=n).astype(np.int8)
    dd = rng.normal(size=n).astype(np.float32)
    y = (1e-7 * a + b - 0.03 * c + 2 * dd + rng.normal(size=n)).astype(np.float32)
    cols = [pa.array(v, type=t) for v, (_, t) in zip((a, b, c, dd), MIXED)]
    X = np.stack([np.asarray(v, dtype=np.float64) for v in (a, b, c, dd)], axis=1)
    ses = LocalSession(conf={"spark.sql.execution.arrow.maxRecordsPerBatch": 700})
    mixed = ses.createDataFrame(pa.Table.from_arrays(cols + [pa.array(y)], names=[m for m, _ in MIXED] + ["label"]),
                                num_partitions=parts)
    arr = ses.createDataFrame(pa.Table.from_arrays(
        [pa.ListArray.from_arrays(pa.array(np.arange(n + 1, dtype=np.int32) * 4), pa.array(X.reshape(-1))),
         pa.array(y)], names=["features", "label"]), num_partitions=parts)
    return mixed, arr


def _column_bytes(df, name):
    return np.asarray(df.toPandas()[name].tolist()).tobytes()


def test_linear_regression_on_mixed_feature_types():
    from spark_rapids_ml_b200.evaluation import RegressionEvaluator
    from spark_rapids_ml_b200.regression import LinearRegression
    from spark_rapids_ml_b200.tuning import CrossValidator

    mixed, arr = _mixed_frames(3000, seed=1, wide=True)
    m_mixed = LinearRegression(featuresCol=[m for m, _ in MIXED]).fit(mixed)
    m_arr = LinearRegression(featuresCol="features").fit(arr)
    assert np.asarray(m_mixed.coef_).tobytes() == np.asarray(m_arr.coef_).tobytes()
    assert np.float64(m_mixed.intercept_).tobytes() == np.float64(m_arr.intercept_).tobytes()
    assert _column_bytes(m_mixed.transform(mixed), "prediction") == _column_bytes(m_arr.transform(arr), "prediction")
    metrics = []
    for est, df in ((LinearRegression(featuresCol=[m for m, _ in MIXED]), mixed),
                    (LinearRegression(featuresCol="features"), arr)):
        cv = CrossValidator(estimator=est, estimatorParamMaps=[{est.regParam: 0.0}],
                            evaluator=RegressionEvaluator(metricName="rmse"), numFolds=2, seed=3)
        metrics.append(cv.fit(df).avgMetrics)
    assert np.asarray(metrics[0]).tobytes() == np.asarray(metrics[1]).tobytes(), metrics


def test_kmeans_on_mixed_feature_types():
    from spark_rapids_ml_b200.clustering import KMeans

    mixed, arr = _mixed_frames(2000, seed=2, wide=False)
    # the same initial centres for both fits, injected as cuML's `init` array
    C0 = (np.random.default_rng(5).normal(size=(5, 4)) * [2.0, 2.0, 2.0, 1.0]).astype(np.float32)
    m_mixed = KMeans(k=5, init=C0, maxIter=10, featuresCol=[m for m, _ in MIXED]).fit(mixed)
    m_arr = KMeans(k=5, init=C0, maxIter=10, featuresCol="features").fit(arr)
    assert np.asarray(m_mixed.cluster_centers_).tobytes() == np.asarray(m_arr.cluster_centers_).tobytes()
    assert _column_bytes(m_mixed.transform(mixed), "prediction") == _column_bytes(m_arr.transform(arr), "prediction")
