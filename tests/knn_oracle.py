"""fp64 NumPy brute-force k-NN on the float32 rows, the parity rule a device result must satisfy against it, and a NumPy
restatement of the wgmma pass's screening arithmetic.

Parity rule, per query q, with m the fp64 mean of the items and

    tau = TAU_C (||q - m||^2 + max_x ||x - m||^2):

  - the k reported ids are distinct;
  - reported distances are non-decreasing and each is within 1e-5 relative of the fp64 distance of that item
    (the device reports sqrt of an exact fp32 sum, within (d + 2) 2^-24 relative);
  - the fp64 squared distances of the returned items, sorted, match the oracle's k smallest element-wise within tau;
  - an id may differ from the oracle's at a position only where the oracle distances of the two items are within tau.

Euclidean distance does not change under translation, and neither does tau: it measures the data's spread, not its
distance from the origin.  A tolerance in ||q||^2 + max ||x||^2 grows with the offset and, at an offset of 1e3 and
d = 128, admits almost any k items.

Where TAU_C comes from.  The wgmma pass (k_knn_wg) decides the set of neighbours by a screen formed in the frame of a
shift point s, an item row: a = fl(q - s), b = fl(x - s), sigma(x) = fl(fl(||b||^2) - 2 a.b) with the dot product in
3xTF32, fp32 accumulation and one rounding in the fma.  sigma(x) + ||a||^2 = ||a - b||^2 up to an error e(x), and the k
items of smallest sigma have sorted true squared distances within 2 max e(x) of the true k smallest (an item displaces
a nearer one only if both screens err towards each other).  With u = 2^-24 and |a.b| <= (||a||^2 + ||b||^2) / 2, every
term of e is a multiple of ||a||^2 + ||b||^2:
  - the norm and the fma round once each;
  - the 3xTF32 products drop lo.lo and the residuals of both splits (3 2^-22 |a_f b_f| per feature), and the fp32
    accumulator rounds at every step;
  - fl(x - s) and fl(q - s) round once per component, and are exact where x, q and s lie within a factor 2 of each
    other (Sterbenz), which is the case on data far from the origin.
The worst case of the accumulation grows as d u; its typical size, random-sign roundings, as sqrt(d) u.  Like the
KMeans margin constant, the rule takes the typical size: e(x) / (||a||^2 + ||b||^2) has an RMS of 2u at d = 128 in
screen_emulation (normal data, any offset), and the few items around the k-th, which decide the set, lie within three
RMS: e <= eps (||a||^2 + ||b||^2) with eps = 6u.  The set error is then at most 2 eps (||a||^2 + max ||b||^2).
Because s is an item row, |x - s| <= 2R with R = max |x - m|, and |q - s| <= |q - m| + R, hence
||a||^2 + max ||b||^2 <= (|q - m| + R)^2 + 4R^2 <= (3 + sqrt 5)(||q - m||^2 + R^2) (with (y + z)^2 <= (1 + t) y^2 +
(1 + 1/t) z^2 at the t that equalises 1 + t and 5 + 1/t).  So the set error is at most 12u (3 + sqrt 5) (||q - m||^2 +
R^2) = 3.75e-6 (...), and TAU_C = 4e-6.

screen_emulation() restates the screen, so that the CPU suite can show that the rule tells the shifted screen from the
unshifted one.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

TAU_C = 4e-6


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


def tau(items: np.ndarray, queries: np.ndarray) -> np.ndarray:
    """Per-query tolerance of the parity rule, TAU_C (||q - m||^2 + max ||x - m||^2), m = the fp64 item mean."""
    X = np.asarray(items, dtype=np.float32).astype(np.float64)
    Q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    m = X.mean(0)
    r2 = float(((X - m) ** 2).sum(1).max())
    return TAU_C * (((Q - m) ** 2).sum(1) + r2)


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
    taus = tau(X, Q)
    bad = {"n_outside_margin": 0, "n_dup": 0, "n_order": 0, "n_dist": 0, "n_set": 0, "n_index": 0, "n_index_diff": 0}
    for i in range(Q.shape[0]):
        q = Q[i]
        t = taus[i]
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
            if np.any(np.abs(np.sort(e) - D0[i]) > t):
                bad["n_set"] += 1
                ok = False
            diff = idx[i] != I0[i]
            bad["n_index_diff"] += int(diff.sum())
            for p in np.nonzero(diff)[0]:
                ro = row_of[int(I0[i][p])]
                eo = float(((q - X[ro]) ** 2).sum())
                if abs(e[p] - eo) > t:
                    bad["n_index"] += 1
                    ok = False
                    break
        if not ok:
            bad["n_outside_margin"] += 1
    return bad


def _tf32(a: np.ndarray) -> np.ndarray:
    """rn_tf32_bits: round a float32 to 10 explicit mantissa bits, ties away from zero, kept as a float32."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def screen_emulation(items: np.ndarray, queries: np.ndarray, shift: Optional[np.ndarray] = None) -> np.ndarray:
    """The k_knn_wg screen ||x'||^2 - 2 q'.x' as float32 [nq, n], x' = fl(x - shift), q' = fl(q - shift).

    As the kernel forms it: both sides split into tf32 hi + lo, per feature the products lo.Xhi, hi.Xlo, hi.Xhi (small
    terms first) added to an fp32 accumulator, the norm the fp64 sum of x'^2 rounded once, and one rounding for
    fma(-2, acc, norm).  The order of the fp32 additions inside the tensor core is not modelled: this restates the error
    sizes, not the device's bits.  shift=None screens in the data's own frame."""
    X = np.asarray(items, dtype=np.float32)
    Q = np.asarray(queries, dtype=np.float32)
    if shift is not None:
        s = np.asarray(shift, dtype=np.float32)
        X = X - s
        Q = Q - s
    xh = _tf32(X)
    xl = _tf32(X - xh)
    qh = _tf32(Q)
    ql = _tf32(Q - qh)
    norms = (X.astype(np.float64) ** 2).sum(1).astype(np.float32)
    acc = np.zeros((Q.shape[0], X.shape[0]), np.float32)
    for f in range(X.shape[1]):   # tf32 x tf32 products are exact in fp32; each addition rounds
        acc += np.outer(ql[:, f], xh[:, f])
        acc += np.outer(qh[:, f], xl[:, f])
        acc += np.outer(qh[:, f], xh[:, f])
    return (norms[None, :].astype(np.float64) - 2.0 * acc.astype(np.float64)).astype(np.float32)
