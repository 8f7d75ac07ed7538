"""fp64 NumPy brute-force k-NN on the float32 rows, and the parity rule a device result must satisfy against it.

Parity rule, per query, with tau = 1e-6 (||q||^2 + max ||x||^2 over the items), the KMeans margin constant:
  - the k reported ids are distinct;
  - reported distances are non-decreasing and each is within 1e-5 relative of the fp64 distance of that item
    (the device reports sqrt of an exact fp32 sum, within (d + 2) 2^-24 relative);
  - the fp64 squared distances of the returned items, sorted, match the oracle's k smallest element-wise within tau;
  - an id may differ from the oracle's at a position only where the oracle distances of the two items are within tau.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np


def knn(items: np.ndarray, queries: np.ndarray, k: int, ids: Optional[np.ndarray] = None, block: int = 256):
    """(squared distances fp64 [nq, k], ids [nq, k]) of the k nearest items, ties broken by the lower global row."""
    X = np.asarray(items, dtype=np.float32).astype(np.float64)
    Q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    ids = np.arange(X.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    xn = (X * X).sum(1)
    D = np.empty((Q.shape[0], k))
    I = np.empty((Q.shape[0], k), dtype=np.int64)
    rows = np.arange(X.shape[0])
    for q0 in range(0, Q.shape[0], block):
        q = Q[q0:q0 + block]
        d2 = ((q[:, None, :] - X[None, :, :]) ** 2).sum(-1) if X.shape[1] <= 8 else \
            np.maximum((q * q).sum(1)[:, None] + xn[None, :] - 2.0 * q @ X.T, 0.0)
        if X.shape[1] > 8:   # exact fp64 differences for the candidates near the cut, so that ties order by row
            m = min(k + 16, X.shape[0])
            part = np.argpartition(d2, m - 1, axis=1)[:, :m]
            for i in range(q.shape[0]):
                cand = part[i]
                ex = ((q[i][None, :] - X[cand]) ** 2).sum(1)
                o = np.lexsort((cand, ex))[:k]
                D[q0 + i] = ex[o]
                I[q0 + i] = ids[cand[o]]
            continue
        for i in range(q.shape[0]):
            o = np.lexsort((rows, d2[i]))[:k]
            D[q0 + i] = d2[i][o]
            I[q0 + i] = ids[o]
    return D, I


def compare(items: np.ndarray, queries: np.ndarray, k: int, dist: np.ndarray, idx: np.ndarray,
            ids: Optional[np.ndarray] = None) -> Dict[str, int]:
    """Counts of queries that break the parity rule (n_outside_margin must be 0)."""
    X = np.asarray(items, dtype=np.float32).astype(np.float64)
    Q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    ids = np.arange(X.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    row_of = {int(v): i for i, v in enumerate(ids)}
    D0, I0 = knn(X, Q, k, ids)
    dist = np.asarray(dist, dtype=np.float64)
    idx = np.asarray(idx, dtype=np.int64)
    xmax = float((X * X).sum(1).max())
    bad = {"n_outside_margin": 0, "n_dup": 0, "n_order": 0, "n_dist": 0, "n_set": 0, "n_index": 0, "n_index_diff": 0}
    for i in range(Q.shape[0]):
        q = Q[i]
        tau = 1e-6 * (float(q @ q) + xmax)
        ok = True
        if len(set(idx[i].tolist())) != k or any(int(v) not in row_of for v in idx[i]):
            bad["n_dup"] += 1
            ok = False
        else:
            r = np.array([row_of[int(v)] for v in idx[i]])
            e = ((q[None, :] - X[r]) ** 2).sum(1)
            if np.any(np.diff(dist[i]) < 0):
                bad["n_order"] += 1
                ok = False
            if np.any(np.abs(dist[i] - np.sqrt(e)) > 1e-5 * np.sqrt(e) + 1e-30):
                bad["n_dist"] += 1
                ok = False
            if np.any(np.abs(np.sort(e) - D0[i]) > tau):
                bad["n_set"] += 1
                ok = False
            diff = idx[i] != I0[i]
            bad["n_index_diff"] += int(diff.sum())
            for p in np.nonzero(diff)[0]:
                ro = row_of[int(I0[i][p])]
                eo = float(((q - X[ro]) ** 2).sum())
                if abs(e[p] - eo) > tau:
                    bad["n_index"] += 1
                    ok = False
                    break
        if not ok:
            bad["n_outside_margin"] += 1
    return bad
