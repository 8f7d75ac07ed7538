"""Scalar feature columns as they reach b2k_ingest_append, without a GPU.  fit (_features_from_pdf) and transform /
evaluation (_append_transform_features) hand the library d column pointers of one source dtype.  Columns that share a
dtype the library converts must go over unchanged; any other set must arrive as float32, each column converted from
its own type (np.asarray(col).astype(np.float32), the rounding the device applies), never through a common type that
truncates (int64 -> int8, float64 -> int64) or rounds twice (int64 -> float64 -> float32).

A recorder stands in for Context._invoke and reads the columns behind the pointer array while the call is made."""
import ctypes

import numpy as np
import pyarrow as pa
import pytest
import torch

from spark_rapids_ml_b200 import _native
from spark_rapids_ml_b200.core import _append_transform_features, _features_from_pdf
from spark_rapids_ml_b200.sparkshim.sql import _batches_to_pdf_iter
from spark_rapids_ml_b200.utils import DeviceRowAppender

_CODE_DTYPES = {code: dt for dt, code in _native._DTYPE_CODES.items()}
I64_MAX, I64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min

# each mix: (Arrow type, values) per column, four rows.  The large integers round in float32; 2^53 + 2^29 + 1 lies just
# above a float32 halfway point, which float64 rounds it onto, so int64 -> float64 -> float32 gives 2^53, not 2^53 + 2^30
MIXES = {
    "int64,double": [(pa.int64(), [1, 2, 2**53 + 2**29 + 1, I64_MIN]),
                     (pa.float64(), [2.7, -0.5, 1e39, 1e-40])],
    "int8,int64": [(pa.int8(), [1, 2, -128, 127]),
                   (pa.int64(), [300, 70000, 2**24 + 1, I64_MAX])],
    "float32,double": [(pa.float32(), [1.5, -0.0, 3.4e38, 1e-45]),
                       (pa.float64(), [1.0 + 2.0**-24, float("nan"), -float("inf"), 2.0**-150 * 1.5])],
    "bool,int32": [(pa.bool_(), [True, False, True, False]),
                   (pa.int32(), [2**24 + 3, -2**31, 2**31 - 1, 7])],
    "uint16,double": [(pa.uint16(), [0, 1, 65535, 40000]),
                      (pa.float64(), [0.1, -2.5, 65504.0000001, -1e-300])],
}


class _ColumnRecorder:
    """Context._invoke: records the columns of every b2k_ingest_append call of the column layout."""

    def __init__(self):
        self.batches = []

    def __call__(self, fn, *args, after=()):
        assert fn == "b2k_ingest_append" and args[8] == _native.LAYOUT_COLUMNS, (fn, args)
        d, addr, n_b, dt = args[2], args[4], args[6], _CODE_DTYPES[args[7]]
        ptrs = (ctypes.c_void_p * d).from_address(addr)
        self.batches.append([np.frombuffer(ctypes.string_at(p, n_b * dt.itemsize), dtype=dt).copy() for p in ptrs])
        return 0


class _Stream:
    def synchronize(self):
        pass


@pytest.fixture
def ctx(monkeypatch):
    c = _native.Context.__new__(_native.Context)
    c._torch = torch
    c.device = torch.device("cpu")
    c.device_index = 0
    c._h = None
    c._invoke = _ColumnRecorder()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
    return c


def _frame(cols, arrow_backed):
    batch = pa.RecordBatch.from_arrays([pa.array(v, type=t) for t, v in cols], [f"c{i}" for i in range(len(cols))])
    return next(_batches_to_pdf_iter([batch], arrow_backed))


def _assert_bits(got, want):
    """float32 equality bit for bit, NaN positions by isnan."""
    assert got.dtype == np.float32 and got.shape == want.shape
    nan = np.isnan(want)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def _ingest(ctx, path, pdf):
    app = DeviceRowAppender(ctx, pdf.shape[1], first_capacity=1)
    if path == "transform":
        _append_transform_features(app, pdf, pdf.shape[1])
    else:
        _features_from_pdf(pdf, list(pdf.columns), app, None)
    (batch,) = ctx._invoke.batches
    return batch


@pytest.mark.parametrize("arrow_backed", [True, False])
@pytest.mark.parametrize("path", ["transform", "fit"])
@pytest.mark.parametrize("mix", sorted(MIXES))
def test_mixed_columns_reach_the_library_as_their_own_float32(ctx, mix, path, arrow_backed):
    cols = MIXES[mix]
    got = _ingest(ctx, path, _frame(cols, arrow_backed))
    assert len(got) == len(cols)
    for g, (t, v) in zip(got, cols):
        with np.errstate(over="ignore"):
            _assert_bits(g, np.asarray(pa.array(v, type=t).to_numpy(zero_copy_only=False)).astype(np.float32))


@pytest.mark.parametrize("path", ["transform", "fit"])
@pytest.mark.parametrize("t,v", [(pa.int64(), [I64_MIN, 2**53 + 1, -5]), (pa.int8(), [-128, 0, 127]),
                                 (pa.float64(), [1e-40, 2.5, -1e39])])
def test_same_type_columns_go_over_unchanged(ctx, path, t, v):
    """The fast path: one dtype the library converts itself reaches it as is, for the device to convert."""
    got = _ingest(ctx, path, _frame([(t, v), (t, v[::-1])], True))
    want = np.asarray(v, dtype=t.to_pandas_dtype())
    assert got[0].dtype == want.dtype
    np.testing.assert_array_equal(got[0], want)
    np.testing.assert_array_equal(got[1], want[::-1])


@pytest.mark.parametrize("t,v", [(pa.uint8(), [0, 255, 17]), (pa.bool_(), [True, False, True])])
def test_unsigned_and_boolean_columns_alone_arrive_as_float32(ctx, t, v):
    got = _ingest(ctx, "transform", _frame([(t, v), (t, v)], True))
    for g in got:
        _assert_bits(g, np.asarray(v).astype(np.float32))
