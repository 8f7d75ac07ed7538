"""fp64 NumPy restatement of UMAP as include/b2kmeans.h defines it (McInnes, Healy & Melville 2018): the k-NN graph,
smooth k-NN memberships, the fuzzy set union / intersection, the supervised intersection, the schedule, the negative
draws, the random init and the epoch-synchronous layout.  Written from the published algorithm; the tests feed it the
device's own inputs and compare step by step."""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np

M64 = (1 << 64) - 1
SMOOTH_K_ITERS, SMOOTH_K_TOL, MIN_K_DIST_SCALE = 64, 1e-5, 1e-3


def _mix(z: int) -> int:
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def umap_hash(seed: int, a: int, b: int, c: int) -> int:
    """The counter-based draw of include/b2kmeans.h: splitmix64 finalisers chained over (seed, a, b, c)."""
    return _mix(_mix(_mix(_mix((seed + 0x9E3779B97F4A7C15) & M64) ^ a) ^ b) ^ c)


def unit(h: int) -> float:
    return (h >> 11) * 2.0 ** -53


def knn(X: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """Exact Euclidean k-NN of the rows against themselves in fp64, ties to the lower row."""
    X = X.astype(np.float64)
    d2 = ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)
    idx = np.argsort(d2, axis=1, kind="stable")[:, :k]
    return np.sqrt(np.take_along_axis(d2, idx, 1)), idx


def membership_row(dist: np.ndarray, idx: np.ndarray, self_idx: int, lc: float, mean_floor: float,
                   use_row_mean: bool) -> Tuple[float, float, np.ndarray]:
    dist = np.asarray(dist, dtype=np.float64)
    k = dist.size
    nz = dist[dist > 0.0]
    rho = 0.0
    index = int(math.floor(lc))
    interp = lc - index
    if nz.size >= lc:
        if index > 0:
            rho = nz[index - 1]
            if interp > SMOOTH_K_TOL:
                rho += interp * (nz[index] - nz[index - 1])
        else:
            rho = interp * nz[0]
    elif nz.size > 0:
        rho = float(dist.max())
    target = math.log2(k)
    lo, hi, mid = 0.0, math.inf, 1.0
    for _ in range(SMOOTH_K_ITERS):
        psum = 0.0
        for j in range(k):
            if idx[j] == self_idx:
                continue
            dd = dist[j] - rho
            psum += math.exp(-(dd / mid)) if dd > 0.0 else 1.0
        if abs(psum - target) < SMOOTH_K_TOL:
            break
        if psum > target:
            hi = mid
            mid = (lo + hi) / 2.0
        else:
            lo = mid
            mid = mid * 2.0 if hi == math.inf else (lo + hi) / 2.0
    row_mean = 0.0
    for j in range(k):
        row_mean += dist[j]
    row_mean /= k
    floor_v = MIN_K_DIST_SCALE * (row_mean if (rho > 0.0 or use_row_mean) else mean_floor)
    if mid < floor_v:
        mid = floor_v
    w = np.empty(k)
    for j in range(k):
        dd = dist[j] - rho
        w[j] = 0.0 if idx[j] == self_idx else (1.0 if (dd <= 0.0 or mid == 0.0) else math.exp(-(dd / mid)))
    return float(rho), float(mid), w


def memberships(dist: np.ndarray, idx: np.ndarray, lc: float = 1.0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    dist = np.asarray(dist, dtype=np.float32).astype(np.float64)
    n, k = dist.shape
    mean_all = sum(float(sum(dist[i].tolist())) for i in range(n)) / (n * k)
    rho, sigma, P = np.zeros(n), np.zeros(n), np.zeros((n, k))
    for i in range(n):
        rho[i], sigma[i], P[i] = membership_row(dist[i], idx[i], i, lc, mean_all, False)
    return rho, sigma, P


def symmetrise(rows: np.ndarray, cols: np.ndarray, vals: np.ndarray, n: int, mix: float):
    """W = mix (A + A^T - A o A^T) + (1 - mix) A o A^T of the COO A -> CSR (indptr, indices, weights), zeros dropped."""
    fwd: Dict[Tuple[int, int], float] = {}
    bwd: Dict[Tuple[int, int], float] = {}
    for i, j, v in zip(rows.tolist(), cols.tolist(), vals.tolist()):
        fwd[(i, j)] = v
        bwd[(j, i)] = v
    out = []
    for key in sorted(set(fwd) | set(bwd)):
        a, b = fwd.get(key, 0.0), bwd.get(key, 0.0)
        ab = a * b
        w = mix * (a + b - ab) + (1.0 - mix) * ab
        if w > 0.0:
            out.append((key[0], key[1], w))
    indptr = np.zeros(n + 1, np.int64)
    for i, _, _ in out:
        indptr[i + 1] += 1
    return (np.cumsum(indptr), np.array([o[1] for o in out], np.int32), np.array([o[2] for o in out], np.float64))


def graph(dist: np.ndarray, idx: np.ndarray, lc: float = 1.0, mix: float = 1.0, labels: Optional[np.ndarray] = None):
    n, k = idx.shape
    rho, sigma, P = memberships(dist, idx, lc)
    indptr, indices, w = symmetrise(np.repeat(np.arange(n), k), idx.reshape(-1), P.reshape(-1), n, mix)
    if labels is not None:
        w = w.copy()
        rows = np.repeat(np.arange(n), np.diff(indptr))
        for e in range(w.size):
            li, lj = labels[rows[e]], labels[indices[e]]
            w[e] *= math.exp(-1.0) if (li == -1 or lj == -1) else (math.exp(-5.0) if li != lj else 1.0)
        for i in range(n):
            s = slice(indptr[i], indptr[i + 1])
            w[s] = w[s] / w[s].max()
        indptr, indices, w = symmetrise(rows, indices.astype(np.int64), w, n, 1.0)
    return {"rho": rho, "sigma": sigma, "P": P, "indptr": indptr, "indices": indices, "weights": w}


def schedule(w: np.ndarray, n_epochs: int) -> np.ndarray:
    wmax = float(w.max())
    return np.where(w < wmax / n_epochs, np.inf, wmax / w)


def random_init(n: int, C: int, seed: int) -> np.ndarray:
    Y = np.array([[np.float32(20.0 * unit(umap_hash(seed, 1 << 40, i, c)) - 10.0) for c in range(C)]
                  for i in range(n)], dtype=np.float32)
    return rescale(Y)


def rescale(Y: np.ndarray) -> np.ndarray:
    Y = Y.astype(np.float64)
    lo, hi = Y.min(0), Y.max(0)
    span = hi - lo
    return np.where(span > 0, 10.0 * (Y - lo) / np.where(span > 0, span, 1.0), 0.0).astype(np.float32)


def layout(Y0: np.ndarray, indptr: np.ndarray, indices: np.ndarray, eps: np.ndarray, n_epochs: int, epochs: int,
           a: float, b: float, gamma: float = 1.0, lr: float = 1.0, neg_rate: int = 5, seed: int = 0,
           restart: Optional[Dict[int, np.ndarray]] = None, history: Optional[list] = None) -> np.ndarray:
    """The epoch-synchronous optimize_layout_euclidean (move_other): `epochs` epochs of the n_epochs schedule, every
    update reading the positions of the start of the epoch, positions rounded to fp32 after each epoch.  restart[e]
    replaces the positions at the start of epoch e (the schedule runs on); history collects the positions after each
    epoch."""
    Y = Y0.astype(np.float32).copy()
    n = Y.shape[0]
    rows = np.repeat(np.arange(n), np.diff(indptr))
    nxt = eps.copy()
    epn = eps / neg_rate if neg_rate > 0 else np.full_like(eps, np.inf)
    nxt_neg = epn.copy()
    for e in range(epochs):
        if restart is not None and e in restart:
            Y = np.asarray(restart[e], dtype=np.float32).copy()
        alpha = lr * (1.0 - e / n_epochs)
        Yd = Y.astype(np.float64)
        acc = np.zeros_like(Yd)
        for p in np.nonzero(nxt <= e)[0]:
            i, j = int(rows[p]), int(indices[p])
            diff = Yd[i] - Yd[j]
            d2 = float(diff @ diff)
            ga = (-2.0 * a * b * d2 ** (b - 1.0)) / (a * d2 ** b + 1.0) if d2 > 0 else 0.0
            g = np.clip(ga * diff, -4.0, 4.0)
            acc[i] += g
            acc[j] -= g
            nxt[p] += eps[p]
            nneg = max(0, int((e - nxt_neg[p]) / epn[p]))
            nxt_neg[p] += nneg * epn[p]
            for q in range(nneg):
                kk = umap_hash(seed, e, int(p), q) % n
                if kk == i:
                    continue
                diff = Yd[i] - Yd[kk]
                d2 = float(diff @ diff)
                if d2 > 0:
                    gr = 2.0 * gamma * b / ((0.001 + d2) * (a * d2 ** b + 1.0))
                    acc[i] += np.clip(gr * diff, -4.0, 4.0)
                else:
                    acc[i] += 4.0
        Y = (Yd + alpha * acc).astype(np.float32)
        if history is not None:
            history.append(Y)
    return Y


def transform(X: np.ndarray, emb: np.ndarray, Q: np.ndarray, k: int, n_epochs: int, a: float, b: float,
              gamma: float = 1.0, lr: float = 1.0, neg_rate: int = 5, seed: int = 0, lc: float = 1.0) -> np.ndarray:
    """b2k_umap_transform row by row: exact neighbours among X, memberships with no self edge and the row's own mean as
    the sigma floor, the per-row schedule, the weighted-mean start, then n_epochs epochs moving the query only
    (attraction once per due edge), negatives umap_hash(seed, e, idx_0 n_train + idx_j, q) mod n_train."""
    n = X.shape[0]
    C = emb.shape[1]
    E = emb.astype(np.float64)
    out = np.empty((Q.shape[0], C), np.float32)
    X64 = X.astype(np.float64)
    for r in range(Q.shape[0]):
        q = Q[r].astype(np.float64)
        if not np.all(np.isfinite(q)):
            out[r] = np.nan
            continue
        d = np.sqrt(((X64 - q) ** 2).sum(1))
        nb = np.argsort(d, kind="stable")[:k]
        _, _, w = membership_row(d[nb].astype(np.float32), nb, -1, lc, 0.0, True)
        wmax = w.max()
        eps = np.where(w < wmax / max(n_epochs, 1), np.inf, wmax / w)
        epn = eps / neg_rate if neg_rate > 0 else np.full_like(eps, np.inf)
        nxt, nxt_neg = eps.copy(), epn.copy()
        y = ((w[:, None] * E[nb]).sum(0) / w.sum()).astype(np.float32)
        key0 = int(nb[0]) * n
        for e in range(n_epochs):
            alpha = lr * (1.0 - e / n_epochs)
            yd = y.astype(np.float64)
            acc = np.zeros(C)
            for j in range(k):
                if not nxt[j] <= e:
                    continue
                diff = yd - E[nb[j]]
                d2 = float(diff @ diff)
                ga = (-2.0 * a * b * d2 ** (b - 1.0)) / (a * d2 ** b + 1.0) if d2 > 0 else 0.0
                acc += np.clip(ga * diff, -4.0, 4.0)
                nxt[j] += eps[j]
                nneg = max(0, int((e - nxt_neg[j]) / epn[j]))
                nxt_neg[j] += nneg * epn[j]
                for t in range(nneg):
                    kk = umap_hash(seed, e, key0 + int(nb[j]), t) % n
                    diff = yd - E[kk]
                    d2 = float(diff @ diff)
                    if d2 > 0:
                        acc += np.clip(2.0 * gamma * b / ((0.001 + d2) * (a * d2 ** b + 1.0)) * diff, -4.0, 4.0)
                    else:
                        acc += 4.0
            y = (yd + alpha * acc).astype(np.float32)
        out[r] = y
    return out


def find_ab(spread: float = 1.0, min_dist: float = 0.1) -> Tuple[float, float]:
    """Least-squares fit of 1 / (1 + a x^(2b)) to the min_dist / spread target curve (Gauss-Newton in fp64)."""
    x = np.linspace(0, spread * 3, 300)
    y = np.where(x < min_dist, 1.0, np.exp(-(x - min_dist) / spread))
    a, b = 1.0, 1.0
    for _ in range(200):
        xb = np.where(x > 0, x ** (2 * b), 0.0)
        f = 1.0 / (1.0 + a * xb)
        r = f - y
        lx = np.where(x > 0, np.log(np.where(x > 0, x, 1.0)), 0.0)
        ja = -xb * f * f
        jb = -a * xb * 2 * lx * f * f
        J = np.stack([ja, jb], 1)
        step = np.linalg.lstsq(J, -r, rcond=None)[0]
        a, b = a + step[0], b + step[1]
        if np.abs(step).max() < 1e-14:
            break
    return float(a), float(b)
