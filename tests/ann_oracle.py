"""fp64 NumPy IVF-Flat: the training-subset rule, the list and probe rules and the search over the probed lists, with the
checks a device result of b2k_ivf_search must pass step by step.

  1. lists:  each item's list is a nearest centre, within the margin TAU_C (||x||^2 + max ||c||^2) of the best: the
     3xTF32 assign pass of the Lloyd kernels works in the unshifted frame;
  2. probes: each query's probe list meets the k-NN parity rule of knn_oracle against the centres;
  3. result: the k-NN parity rule against the exact top-k over the union of the probed lists' items (the device's own
     lists and probes), plus the fill rule for queries that find fewer than k items.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np

import knn_oracle as ko

INT64_MAX = np.iinfo(np.int64).max


def train_mask(n_total: int, f: float) -> np.ndarray:
    """Global row r is a training row when floor((r + 1) f) > floor(r f)."""
    r = np.arange(n_total + 1, dtype=np.float64)
    fl = np.floor(r * f)
    return fl[1:] > fl[:-1]


def assign(items: np.ndarray, centers: np.ndarray) -> np.ndarray:
    """Nearest centre per item, ties to the lowest centre (fp64)."""
    X = np.asarray(items, np.float32).astype(np.float64)
    C = np.asarray(centers, np.float32).astype(np.float64)
    d2 = ((X[:, None, :] - C[None, :, :]) ** 2).sum(-1)
    return d2.argmin(1)


def search(items: np.ndarray, queries: np.ndarray, k: int, lists: np.ndarray, probes: np.ndarray,
           ids: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(squared distances [nq, k] with +inf fill, ids [nq, k] with the fill rule) of the exact search over the items of
    each query's probed lists (probes [nq, p], -1 = none)."""
    X = np.asarray(items, np.float32).astype(np.float64)
    Q = np.asarray(queries, np.float32).astype(np.float64)
    ids = np.arange(X.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    D = np.full((Q.shape[0], k), np.inf)
    I = np.full((Q.shape[0], k), INT64_MAX, dtype=np.int64)
    for i in range(Q.shape[0]):
        if np.isnan(Q[i]).any():
            continue
        rows = np.nonzero(np.isin(lists, probes[i][probes[i] >= 0]))[0]
        if rows.size == 0:
            continue
        e = ((Q[i][None, :] - X[rows]) ** 2).sum(1)
        o = np.lexsort((rows, e))[:k]
        D[i, :o.size] = e[o]
        I[i, :o.size] = ids[rows[o]]
        I[i, o.size:] = I[i, 0]
    return D, I


def ivf(items: np.ndarray, queries: np.ndarray, k: int, centers: np.ndarray, nprobe: int,
        ids: Optional[np.ndarray] = None):
    """Plain fp64 IVF-Flat for given centres: (squared distances, ids, lists, probes)."""
    lists = assign(items, centers)
    p = min(nprobe, centers.shape[0])
    _, probes = ko.knn(centers, queries, p)
    D, I = search(items, queries, k, lists, probes, ids)
    return D, I, lists, probes


def check_lists(items: np.ndarray, centers: np.ndarray, lists: np.ndarray) -> int:
    """Items whose list is farther than the margin from their nearest centre."""
    X = np.asarray(items, np.float32).astype(np.float64)
    C = np.asarray(centers, np.float32).astype(np.float64)
    d2 = ((X[:, None, :] - C[None, :, :]) ** 2).sum(-1)
    # b2k_kmeans_assign screens in the unshifted frame, so its margin scales with the norms, not with the spread
    margin = ko.TAU_C * ((X ** 2).sum(1) + (C ** 2).sum(1).max())
    got = d2[np.arange(X.shape[0]), lists]
    return int(((lists < 0) | (lists >= C.shape[0]) | (got - d2.min(1) > margin)).sum())


def check_probes(centers: np.ndarray, queries: np.ndarray, probes: np.ndarray) -> int:
    p = probes.shape[1]
    C = np.asarray(centers, np.float32).astype(np.float64)
    Q = np.asarray(queries, np.float32).astype(np.float64)
    nan = np.isnan(Q).any(1)   # a NaN query probes nothing
    bad = int((probes[nan] != -1).any(1).sum())
    Q, probes = Q[~nan], probes[~nan]
    # the device orders by fp32 distances, which two nearly equidistant centres may hold in the other order than fp64
    dist = np.sort(np.sqrt(((Q[:, None, :] - C[probes]) ** 2).sum(-1)), axis=1)
    return bad + ko.compare(C, Q, p, dist, probes)["n_outside_margin"]


def check_result(items: np.ndarray, queries: np.ndarray, k: int, lists: np.ndarray, probes: np.ndarray,
                 dist: np.ndarray, idx: np.ndarray, ids: Optional[np.ndarray] = None,
                 squared: bool = False) -> Dict[str, int]:
    """Counts of queries that break the parity rule over their probed items, or the fill rule."""
    X = np.asarray(items, np.float32).astype(np.float64)
    Q = np.asarray(queries, np.float32).astype(np.float64)
    ids = np.arange(X.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    dist = np.asarray(dist, np.float64)
    dist = np.sqrt(dist) if squared else dist
    bad = {"n_outside_margin": 0, "n_fill": 0}
    for i in range(Q.shape[0]):
        rows = np.nonzero(np.isin(lists, probes[i][probes[i] >= 0]))[0] if not np.isnan(Q[i]).any() else \
            np.zeros(0, np.int64)
        found = min(k, rows.size)
        fill_ok = np.all(np.isinf(dist[i, found:])) and \
            np.all(idx[i, found:] == (idx[i, 0] if found > 0 else INT64_MAX))
        if not fill_ok:
            bad["n_fill"] += 1
        if found == 0:
            continue
        res = ko.compare(X[rows], Q[i:i + 1], found, dist[i:i + 1, :found], idx[i:i + 1, :found], ids[rows])
        bad["n_outside_margin"] += res["n_outside_margin"]
    return bad
