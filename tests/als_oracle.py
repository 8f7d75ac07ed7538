"""fp64 NumPy restatement of ALS as include/b2kmeans.h pins it (Spark's pyspark.ml.recommendation.ALS):

- users / items are integral int32 values; users are indexed by their sorted distinct ids, items likewise;
- the start: user factor = rank normals keyed by (seed, raw user id, j) from splitmix64 and Box-Muller, fl32, scaled to
  unit L2 norm in fp32 (Spark draws from XORShiftRandom, so the start differs from Spark's for the same seed);
- each iteration solves the items from the users, then the users from the items.  For destination d over its ratings
  (s, r): explicit A = sum y y^T, b = sum r y, n = #ratings; implicit c1 = alpha |r|, A = Y^T Y + sum c1 y y^T,
  b = sum_{r > 0} (1 + c1) y, n = #{r > 0}; x = (A + reg n I)^-1 b by Cholesky in fp64, stored as fp32;
- the prediction is the fp32 dot product s = fl32(s + fl32(u_j v_j)) in j order; recommendations order by that score
  descending, the lower id first on a tie.
"""
from __future__ import annotations

import numpy as np

M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(z):
    with np.errstate(over="ignore"):
        z = np.asarray(z, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def start(ids, rank, seed):
    """[U, rank] float32 start factors of the users with raw ids `ids` (include/b2kmeans.h)."""
    ids = np.asarray(ids, dtype=np.int64)
    base = splitmix64(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF)) ^ (ids.astype(np.uint32).astype(np.uint64))
    j = np.arange(rank, dtype=np.uint64)
    h = splitmix64(splitmix64(base)[:, None] ^ j[None, :])
    u1 = ((h >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    u2 = (splitmix64(h) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    v = (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)).astype(np.float32)
    nrm = np.sqrt((v.astype(np.float64) ** 2).sum(1))
    return (v.astype(np.float64) / nrm[:, None]).astype(np.float32)


def check_ids(v, col):
    """Spark's integer rule for an id column: the error message of a bad value, or None."""
    v = np.asarray(v, dtype=np.float64)
    bad = ~(np.isfinite(v) & (v >= -2.0 ** 31) & (v <= 2.0 ** 31 - 1) & (v == np.floor(v)))
    if bad.any():
        x = v[np.argmax(bad)]
        return (f"ALS only supports values in Integer range and without fractional part for column {col}. Value "
                f"{_fmt(x)} was either out of Integer range or contained a fractional part that could not be converted.")
    return None


def _fmt(x):
    if np.isnan(x):
        return "NaN"
    return f"{x:.1f}" if x == np.floor(x) and abs(x) < 1e18 else repr(float(x))


def index(users, items):
    uid, du = np.unique(np.asarray(users, dtype=np.int64), return_inverse=True)
    iid, di = np.unique(np.asarray(items, dtype=np.int64), return_inverse=True)
    return uid, iid, du, di


def half_step(dst, src, r, Ys, nd, reg, implicit=False, alpha=1.0):
    """Solve nd destinations from the float32 source table Ys: float32 [nd, rank] and cond(A + reg n I) [nd]."""
    Y = np.asarray(Ys, dtype=np.float64)
    rank = Y.shape[1]
    r = np.asarray(r, dtype=np.float64)
    YtY = Y.T @ Y if implicit else None
    out = np.zeros((nd, rank), dtype=np.float32)
    cond = np.zeros(nd)
    order = np.argsort(dst, kind="stable")
    bounds = np.searchsorted(dst[order], np.arange(nd + 1))
    for d in range(nd):
        sel = order[bounds[d]:bounds[d + 1]]
        ys, rs = Y[src[sel]], r[sel]
        if implicit:
            c1 = alpha * np.abs(rs)
            A = YtY + (ys * c1[:, None]).T @ ys
            b = ((rs > 0) * (1.0 + c1)) @ ys
            n = int((rs > 0).sum())
        else:
            A = ys.T @ ys
            b = rs @ ys
            n = len(rs)
        A = A + reg * n * np.eye(rank)
        L = np.linalg.cholesky(A)   # raises LinAlgError when not positive definite
        out[d] = np.linalg.solve(L.T, np.linalg.solve(L, b)).astype(np.float32)
        cond[d] = np.linalg.cond(A)
    return out, cond


def fit(users, items, ratings, rank, max_iter, reg, implicit=False, alpha=1.0, seed=0, init=None):
    uid, iid, du, di = index(users, items)
    r = np.ones(len(du), dtype=np.float32) if ratings is None else np.asarray(ratings, dtype=np.float32)
    UF = start(uid, rank, seed) if init is None else np.asarray(init, dtype=np.float32)
    IF = np.zeros((len(iid), rank), dtype=np.float32)
    for _ in range(max_iter):
        IF, _ = half_step(di, du, r, UF, len(iid), reg, implicit, alpha)
        UF, _ = half_step(du, di, r, IF, len(uid), reg, implicit, alpha)
    return {"user_ids": uid, "user_factors": UF, "item_ids": iid, "item_factors": IF}


def step_tol(x_ref, cond):
    """Per-entry bound on |x_dev - x_ref| for one half-step from the same fp32 source table: one fp32 rounding of x, plus
    the fp64 solve's error, cond(A) times a few fp64 ulps of the largest entry of x."""
    mx = np.abs(x_ref).max(1, keepdims=True).astype(np.float64)
    return 2.0 ** -23 * np.abs(x_ref) + (64 * 2.0 ** -52 * cond[:, None] + 2.0 ** -24) * mx


def predict(uf, vf):
    """fp32 rank-order dot products of matching rows: s = fl32(s + fl32(u_j v_j))."""
    uf = np.asarray(uf, dtype=np.float32)
    vf = np.asarray(vf, dtype=np.float32)
    s = np.zeros(uf.shape[0], dtype=np.float32)
    for j in range(uf.shape[1]):
        s = (s + (uf[:, j] * vf[:, j]).astype(np.float32)).astype(np.float32)
    return s


def scores(Q, T):
    """[nq, nt] fp32 scores by the prediction's rule."""
    Q = np.asarray(Q, dtype=np.float32)
    T = np.asarray(T, dtype=np.float32)
    s = np.zeros((Q.shape[0], T.shape[0]), dtype=np.float32)
    for j in range(Q.shape[1]):
        s = (s + (Q[:, j:j + 1] * T[None, :, j]).astype(np.float32)).astype(np.float32)
    return s


def recommend(Q, T, n):
    """Top-n target rows per query row: (indices [nq, min(n, nt)], scores), score descending, lower row on a tie."""
    S = scores(Q, T)
    k = min(n, S.shape[1])
    idx = np.zeros((S.shape[0], k), dtype=np.int64)
    for q in range(S.shape[0]):
        order = np.lexsort((np.arange(S.shape[1]), -S[q].astype(np.float64)))
        idx[q] = order[:k]
    return idx, np.take_along_axis(S, idx, 1)
