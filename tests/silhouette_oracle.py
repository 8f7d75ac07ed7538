"""fp64 NumPy restatement of b2k_silhouette (include/b2kmeans.h): Spark's closed form in a frame shifted by the global
mean, the O(n^2) definition, Spark's expanded form (for the offset cases), and the bound beta of the wgmma pass."""
import numpy as np

U32 = 2.0 ** -24
U64 = 2.0 ** -53


def unit_rows(X, metric):
    """The rows the metric compares, exactly: x (squaredEuclidean) or x / ||x|| (cosine), fp64."""
    y = np.asarray(X, dtype=np.float32).astype(np.float64)
    if metric == "cosine":
        y = y / np.linalg.norm(y, axis=1)[:, None]
    return y


def s_of(a, b):
    """s from the own-cluster and nearest-other mean distances (arrays), arguments clamped at 0."""
    a, b = np.maximum(a, 0.0), np.maximum(b, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(a < b, 1.0 - a / np.where(b > 0, b, 1.0), np.where(a > b, b / np.where(a > 0, a, 1.0) - 1.0, 0.0))


def _parts(X, ids, metric):
    y = unit_rows(X, metric)
    uniq, inv = np.unique(np.asarray(ids, dtype=np.int64), return_inverse=True)
    K = uniq.size
    if K < 2:
        raise ValueError("Number of clusters must be greater than one.")
    N = np.bincount(inv, minlength=K).astype(np.float64)
    m = y.mean(axis=0)
    z = y - m
    mu = np.zeros((K, y.shape[1]))
    np.add.at(mu, inv, z)
    mu /= N[:, None]
    psi = np.zeros(K)
    np.add.at(psi, inv, np.sum((z - mu[inv]) ** 2, axis=1))
    psi /= N
    zn = np.sum(z * z, axis=1)
    mn = np.sum(mu * mu, axis=1)
    D = zn[:, None] + mn[None, :] - 2.0 * (z @ mu.T) + psi[None, :]
    return y, inv, N, D, zn, mn, psi


def _ab(inv, N, D):
    n = D.shape[0]
    own = D[np.arange(n), inv]
    Do = D.copy()
    Do[np.arange(n), inv] = np.inf
    n_own = N[inv]
    a = own * np.where(n_own > 1, n_own / np.maximum(n_own - 1, 1), 0.0)
    return a, Do.min(axis=1), n_own


def closed_form(X, ids, metric="squaredEuclidean"):
    """The metric from D(i, c) = ||y_i - mu_c||^2 + Psi_c in the frame of the global mean (fp64)."""
    _, inv, N, D, *_ = _parts(X, ids, metric)
    a, b, n_own = _ab(inv, N, D)
    return float(np.mean(np.where(n_own > 1, s_of(a, b), 0.0)))


def brute_force(X, ids, metric="squaredEuclidean"):
    """The definition: mean squared distances (or mean 2 (1 - cos)) to every member, O(n^2)."""
    y = unit_rows(X, metric)
    ids = np.asarray(ids, dtype=np.int64)
    uniq, inv = np.unique(ids, return_inverse=True)
    K = uniq.size
    if K < 2:
        raise ValueError("Number of clusters must be greater than one.")
    P = np.sum((y[:, None, :] - y[None, :, :]) ** 2, axis=2)
    N = np.bincount(inv, minlength=K).astype(np.float64)
    D = np.stack([P[:, inv == c].mean(axis=1) for c in range(K)], axis=1)
    a, b, n_own = _ab(inv, N, D)
    return float(np.mean(np.where(n_own > 1, s_of(a, b), 0.0)))


def spark_expanded(X, ids):
    """Spark's SquaredEuclideanSilhouette form: D = ||x||^2 + sum ||y||^2 / N - 2 x.sum y / N, unshifted (fp64)."""
    x = np.asarray(X, dtype=np.float32).astype(np.float64)
    uniq, inv = np.unique(np.asarray(ids, dtype=np.int64), return_inverse=True)
    K = uniq.size
    N = np.bincount(inv, minlength=K).astype(np.float64)
    S = np.zeros((K, x.shape[1]))
    np.add.at(S, inv, x)
    Q = np.bincount(inv, weights=np.sum(x * x, axis=1), minlength=K)
    D = np.sum(x * x, axis=1)[:, None] + (Q / N)[None, :] - 2.0 * (x @ S.T) / N[None, :]
    a, b, n_own = _ab(inv, N, D)
    return float(np.mean(np.where(n_own > 1, s_of(a, b), 0.0)))


def beta(X, ids, metric="squaredEuclidean", nranks=1):
    """The bound of include/b2kmeans.h on |device value - exact value| (wgmma pass; the generic pass is inside it)."""
    y, inv, N, D, zn, mn, psi = _parts(X, ids, metric)
    d = y.shape[1]
    nb = 3.0 * ((d + 7) // 8)
    Qn = np.bincount(inv, weights=np.sum(y * y, axis=1), minlength=N.size) / N
    L = 256.0 + d + N + 8.0 + nranks
    dpsi = (3.0 * L + d + 6.0) * U64 * Qn
    delta = ((31.3 + 36.08 * (1.0 + nb)) * U32 * (zn[:, None] + mn[None, :]) + 2.01 * U32 * psi[None, :] + dpsi[None, :]
             + (8.1 * U32 if metric == "cosine" else 0.0))
    n = D.shape[0]
    a, b, n_own = _ab(inv, N, D)
    da = delta[np.arange(n), inv] * np.where(n_own > 1, n_own / np.maximum(n_own - 1, 1), 0.0)
    do = delta.copy()
    do[np.arange(n), inv] = -np.inf
    db = do.max(axis=1)
    lo = s_of(a + da, b - db)
    hi = s_of(a - da, b + db)
    half = np.where(n_own > 1, (hi - lo) / 2.0, 0.0)
    return float(np.mean(half) + (n + 8) * U64)
