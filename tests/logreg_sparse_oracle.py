"""fp64 SciPy restatement of sparse logistic regression (include/b2kmeans.h, b2k_logreg_*_csr): the objective of
tests/logreg_oracle.py on a CSR matrix, sigma over all n rows with the implicit zeros, plus the Spark vector struct
layout the estimator reads (struct<type, size, indices, values>).  Used by the CPU tests, the GPU tests and
bench_logreg_sparse.py."""
from __future__ import annotations

from typing import Any, Dict, Iterable, Optional, Tuple

import numpy as np
import pyarrow as pa
import scipy.sparse as sp

VECTOR_TYPE = pa.struct([("type", pa.int8()), ("size", pa.int32()), ("indices", pa.list_(pa.int32())),
                         ("values", pa.list_(pa.float64()))])
R_BYTES = 256 << 20   # B2K_LOGREG_CSR_R_BYTES: a row chunk's residuals R [rows][kp] fp64 stay under it


def chunk_rows(kp: int) -> int:
    """Rows per row chunk of the CSR passes at kp margins per row (the library's planner, restated)."""
    return max(1, R_BYTES // (8 * kp))


def random_csr(n: int, d: int, per_row: int, seed: int, zipf: float = 0.0) -> sp.csr_matrix:
    """n rows of width d with about per_row float32 entries each (Zipf-skewed column popularity when zipf > 0)."""
    rng = np.random.default_rng(seed)
    lens = rng.poisson(per_row, size=n).clip(0, d)
    rows, cols = [], []
    for i, k in enumerate(lens):
        if zipf > 0:
            c = np.unique(np.minimum(rng.zipf(zipf, size=k) - 1, d - 1))
        else:
            c = rng.choice(d, size=k, replace=False) if k else np.zeros(0, np.int64)
        rows.append(np.full(len(c), i))
        cols.append(np.sort(c))
    r, c = np.concatenate(rows), np.concatenate(cols)
    v = rng.normal(size=r.size).astype(np.float32)
    return sp.csr_matrix((v, (r, c)), shape=(n, d), dtype=np.float32)


def loss_grad(X: sp.csr_matrix, yi: np.ndarray, W: np.ndarray, b: np.ndarray) -> Tuple[float, np.ndarray, np.ndarray]:
    """(1/n) sum l and its gradient (dW [kp, d], db [kp]) at (W, b), as logreg_oracle.loss_grad on X densified."""
    X = sp.csr_matrix(X, dtype=np.float64)
    n = X.shape[0]
    M = np.asarray(X @ np.asarray(W, dtype=np.float64).T) + np.asarray(b, dtype=np.float64)
    kp = M.shape[1]
    if kp == 1:
        m = M[:, 0]
        yy = (yi == 1).astype(np.float64)
        e = np.exp(-np.abs(m))
        loss = np.maximum(m, 0) + np.log1p(e) - yy * m
        R = (np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e)) - yy)[:, None]
    else:
        mx = M.max(axis=1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(M - mx).sum(axis=1))
        rows = np.flatnonzero(yi >= 0)
        loss = lse.copy()
        loss[rows] -= M[rows, yi[rows]]
        R = np.exp(M - lse[:, None])
        R[rows, yi[rows]] -= 1.0
    return float(loss.sum() / n), np.asarray((X.T @ R).T) / n, R.sum(axis=0) / n


def sigma(X: sp.csr_matrix) -> np.ndarray:
    """Sample (n - 1) standard deviations over all rows, implicit zeros included, in the device's stable form:
    sum over the entries of (x - mu)^2 plus (n - nnz) mu^2."""
    X = sp.csc_matrix(X, dtype=np.float64)
    n, d = X.shape
    if n < 2:
        return np.zeros(d)
    mu = np.asarray(X.sum(axis=0)).ravel() / n
    nnz = np.diff(X.indptr)
    dev = X.data - np.repeat(mu, nnz)
    cs = np.concatenate([[0.0], np.cumsum(dev * dev)])
    ss = cs[X.indptr[1:]] - cs[X.indptr[:-1]] + (n - nnz) * mu * mu
    return np.sqrt(np.maximum(ss, 0.0) / (n - 1))


def eval_bound(X: sp.csr_matrix, W: np.ndarray, b: np.ndarray) -> Dict[str, Any]:
    """logreg_oracle.eval_bound restated on a CSR matrix (the same values, without densifying X)."""
    X = sp.csr_matrix(X, dtype=np.float64)
    n, d = X.shape
    u = 2.0 ** -53
    aX = abs(X)
    A = np.asarray(aX @ np.abs(np.asarray(W, dtype=np.float64)).T) + np.abs(b)
    kp = A.shape[1]
    em = (d + 4) * u * A.max(axis=1) + 16 * u
    c = (n + d + 32) * u
    e_r = 2 * kp * em + 16 * u
    loss_b = float((2 * em + c * (1 + A.max(axis=1))).sum() / n)
    colsum = np.asarray(aX.sum(axis=0)).ravel()
    dW_b = np.asarray(aX.T @ e_r).ravel() / n + c * colsum / n
    db_b = float(e_r.sum() / n + c)
    return {"loss": loss_b, "dW": np.tile(dW_b, (kp, 1)), "db": np.full(kp, db_b)}


def vector_array(X: sp.csr_matrix, dense_rows: Iterable[int] = ()) -> pa.StructArray:
    """The rows of X as Spark vectors in their SQL layout: sparse rows (type 0, stored zeros kept) except the rows in
    dense_rows (type 1: size and indices null, all d values)."""
    X = sp.csr_matrix(X)
    n, d = X.shape
    dense = set(int(i) for i in dense_rows)
    out = []
    for i in range(n):
        lo, hi = X.indptr[i], X.indptr[i + 1]
        if i in dense:
            row = np.zeros(d)
            row[X.indices[lo:hi]] = X.data[lo:hi]
            out.append({"type": 1, "size": None, "indices": None, "values": row.tolist()})
        else:
            out.append({"type": 0, "size": d, "indices": X.indices[lo:hi].astype(int).tolist(),
                        "values": X.data[lo:hi].astype(np.float64).tolist()})
    return pa.array(out, type=VECTOR_TYPE)


def vector_frame(X: sp.csr_matrix, y: Optional[np.ndarray] = None, parts: int = 1, dense_rows: Iterable[int] = (),
                 max_records: Optional[int] = None) -> Any:
    """A local frame with a vector struct column "features" (and a float "label" when y is given)."""
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession

    cols, names = [vector_array(X, dense_rows)], ["features"]
    if y is not None:
        cols.append(pa.array(np.asarray(y, dtype=np.float32)))
        names.append("label")
    s = LocalSession()
    if max_records is not None:
        s.conf_map["spark.sql.execution.arrow.maxRecordsPerBatch"] = str(max_records)
    return s.createDataFrame(pa.Table.from_arrays(cols, names=names), num_partitions=parts)
