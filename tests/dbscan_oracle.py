"""fp64 NumPy oracle of DBSCAN, restating the rule of include/b2kmeans.h (b2k_dbscan_fit) operation for operation.

Adjacency: rows i and j (float32) are adjacent when
  euclidean   sum_f ((double)x_if - (double)x_jf)^2 <= eps^2
  cosine      1 - x_i.x_j / (|x_i| |x_j|) <= eps
with every sum in feature order and every operation rounded once, so the device's fp64 decisions equal these bit for
bit.  Core rows have >= min_samples adjacent rows (themselves included); clusters are the connected components of the
core rows, numbered by their lowest row; a border row takes the cluster of its lowest adjacent core row; the rest is -1.

Also the screen of the wgmma pass restated in NumPy (`screen`) and its error bound (`bound`), for the CPU tests.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24


def _pair_values(Xi: np.ndarray, Xj: np.ndarray, metric: str, ni=None, nj=None) -> np.ndarray:
    """[len(Xi), len(Xj)] fp64 values the rule compares: squared distance (euclidean) or 1 - cos (cosine)."""
    a = Xi.astype(np.float64)
    b = Xj.astype(np.float64)
    acc = np.zeros((a.shape[0], b.shape[0]), dtype=np.float64)
    for f in range(a.shape[1]):   # feature order, no fused multiply-add
        if metric == "euclidean":
            t = a[:, f, None] - b[None, :, f]
            acc += t * t
        else:
            acc += a[:, f, None] * b[None, :, f]
    if metric == "euclidean":
        return acc
    return 1.0 - acc / (ni[:, None] * nj[None, :])


def row_norms(X: np.ndarray) -> np.ndarray:
    a = X.astype(np.float64)
    s = np.zeros(a.shape[0], dtype=np.float64)
    for f in range(a.shape[1]):
        s += a[:, f] * a[:, f]
    return np.sqrt(s)


def adjacency_lists(X: np.ndarray, eps: float, metric: str = "euclidean", chunk: int = 1024):
    """Per row, the sorted array of adjacent rows (itself included)."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    n = X.shape[0]
    thr = eps * eps if metric == "euclidean" else eps
    nrm = row_norms(X) if metric == "cosine" else None
    out = []
    for i0 in range(0, n, chunk):
        i1 = min(n, i0 + chunk)
        parts = [[] for _ in range(i1 - i0)]
        for j0 in range(0, n, chunk):
            j1 = min(n, j0 + chunk)
            v = _pair_values(X[i0:i1], X[j0:j1], metric, None if nrm is None else nrm[i0:i1],
                             None if nrm is None else nrm[j0:j1])
            ii, jj = np.nonzero(v <= thr)
            for r in range(i1 - i0):
                sel = jj[ii == r]
                if sel.size:
                    parts[r].append(sel + j0)
        out.extend(np.concatenate(p) if p else np.zeros(0, dtype=np.int64) for p in parts)
    return out


def dbscan(X: np.ndarray, eps: float, min_samples: int, metric: str = "euclidean"):
    """-> (labels int32 [n], core bool [n], n_clusters)."""
    adj = adjacency_lists(X, eps, metric)
    n = len(adj)
    core = np.array([a.size >= min_samples for a in adj], dtype=bool)
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for i in np.nonzero(core)[0]:
        for j in adj[i]:
            if core[j]:
                a, b = find(i), find(j)
                if a != b:
                    parent[max(a, b)] = min(a, b)
    roots = np.array([find(i) for i in range(n)])
    labels = np.full(n, -1, dtype=np.int32)
    cid = {}
    for i in range(n):   # rows in order: a cluster is numbered when its lowest core row is met
        if core[i]:
            r = roots[i]
            if r not in cid:
                cid[r] = len(cid)
            labels[i] = cid[r]
    for i in np.nonzero(~core)[0]:
        c = [j for j in adj[i] if core[j]]
        if c:
            labels[i] = labels[min(c)]
    return labels, core, len(cid)


# ---- the wgmma screen and its bound (b2k_dbscan.cu, b2k_dbscan_bound) ----
def tf32(v: np.ndarray) -> np.ndarray:
    """rn_tf32_bits: round the float32 bits to 10 explicit mantissa bits (ties away from zero)."""
    b = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def bound_coef(d: int, metric: str, E: float):
    nb = 3.0 * ((d + 7) // 8)
    coef = np.float32((24.0 + 37.0 * (1.0 + nb)) * U * (1.0 + 2.0 ** -10))
    B0 = np.float32((2.01 * U * E + (8.1 * U if metric == "cosine" else 0.0)) * (1.0 + 2.0 ** -10))
    return coef, B0


def shifted(X: np.ndarray, metric: str = "euclidean") -> np.ndarray:
    """The rows the screen sees: x - s (s = row 0), after scaling by 1 / ||x|| for cosine, in fp32."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    if metric == "cosine":
        X = (X.astype(np.float64) / row_norms(X)[:, None]).astype(np.float32)
    return (X - X[0]).astype(np.float32)


def screen(V: np.ndarray, i: np.ndarray, j: np.ndarray, shift: bool = True) -> np.ndarray:
    """S for pairs (i, j) of the shifted rows V: norms rounded once to fp32, the dot product as 3xTF32 (lo.hi + hi.lo +
    hi.hi) summed in fp32 in chunks of 8 features, then fl(fl(n_j - 2 acc) + n_i)."""
    V = np.ascontiguousarray(V, dtype=np.float32)
    nrm = (V.astype(np.float64) ** 2).sum(1).astype(np.float32)
    hi = tf32(V)
    lo = tf32((V - hi).astype(np.float32))
    a_hi, a_lo, b_hi, b_lo = hi[i], lo[i], hi[j], lo[j]
    acc = np.zeros(len(i), dtype=np.float32)
    for k0 in range(0, V.shape[1], 8):
        s = slice(k0, k0 + 8)
        for pa, pb in ((a_lo, b_hi), (a_hi, b_lo), (a_hi, b_hi)):
            blk = (pa[:, s].astype(np.float64) * pb[:, s].astype(np.float64)).sum(1)
            acc = (acc + blk.astype(np.float32)).astype(np.float32)
    t = (nrm[j].astype(np.float64) - 2.0 * acc.astype(np.float64)).astype(np.float32)
    return (t + nrm[i]).astype(np.float32)


def bound(V: np.ndarray, i: np.ndarray, j: np.ndarray, d: int, metric: str, E: float) -> np.ndarray:
    """B' of the kernel for pairs (i, j), as fp32 arithmetic forms it."""
    V = np.ascontiguousarray(V, dtype=np.float32)
    nrm = (V.astype(np.float64) ** 2).sum(1).astype(np.float32)
    coef, B0 = bound_coef(d, metric, E)
    s = (nrm[i] + nrm[j]).astype(np.float32)
    return (coef.astype(np.float64) * s.astype(np.float64) + np.float64(B0)).astype(np.float32)
