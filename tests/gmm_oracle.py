"""fp64 oracle of the Gaussian mixture semantics pinned in include/b2kmeans.h (b2k_gmm_fit / b2k_gmm_predict)."""
from typing import Tuple

import numpy as np

EPS = 2.220446049250313e-16
_M64 = (1 << 64) - 1


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def init_rows(seed: int, k: int, n_total: int) -> np.ndarray:
    """The global rows of the random start: component i takes rows [5 i, 5 i + 5) of this list."""
    s = int(seed) & _M64
    return np.array([splitmix64(s ^ splitmix64(j)) % n_total for j in range(5 * k)], dtype=np.int64)


def random_init(X: np.ndarray, k: int, seed: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Weights 1/k; per component the mean and the biased per-feature variance (diagonal) of its 5 rows."""
    rows = np.asarray(X, dtype=np.float32).astype(np.float64)[init_rows(seed, k, X.shape[0])].reshape(k, 5, -1)
    mu = rows.mean(axis=1)
    var = ((rows - mu[:, None, :]) ** 2).mean(axis=1)
    return np.full(k, 1.0 / k), mu, np.stack([np.diag(v) for v in var])


def log_pdf(X: np.ndarray, mu: np.ndarray, cov: np.ndarray) -> np.ndarray:
    """Spark's MultivariateGaussian.logpdf with its pseudo-inverse; raises on a covariance with no eigenvalue above
    tol = EPS max(lambda) d."""
    d = mu.shape[0]
    lam, U = np.linalg.eigh((cov + cov.T) / 2)
    tol = EPS * lam.max() * d
    keep = lam > tol
    if not keep.any():
        raise ValueError("covariance has no eigenvalue above the tolerance")
    P = (U[:, keep] / np.sqrt(lam[keep])).T
    q = (((X - mu) @ P.T) ** 2).sum(axis=1)
    return -0.5 * (d * np.log(2 * np.pi) + np.log(lam[keep]).sum()) - 0.5 * q


def e_step(X: np.ndarray, w: np.ndarray, mu: np.ndarray, cov: np.ndarray) -> Tuple[np.ndarray, float, np.ndarray]:
    """(responsibilities [n, k], log-likelihood, first argmax)."""
    X = np.asarray(X, dtype=np.float64)
    p = np.stack([w[j] * np.exp(log_pdf(X, mu[j], cov[j])) + EPS for j in range(len(w))], axis=1)
    s = p.sum(axis=1)
    r = p / s[:, None]
    return r, float(np.log(s).sum()), np.argmax(r, axis=1)


def m_step(X: np.ndarray, r: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    X = np.asarray(X, dtype=np.float64)
    N = r.sum(axis=0)
    mu = (r.T @ X) / N[:, None]
    cov = np.stack([((X - mu[j]) * r[:, j:j + 1]).T @ (X - mu[j]) / N[j] for j in range(r.shape[1])])
    return N / X.shape[0], mu, cov


def fit(X: np.ndarray, w: np.ndarray, mu: np.ndarray, cov: np.ndarray, max_iter: int, tol: float):
    """EM as b2k_gmm_fit runs it: returns (w, mu, cov, log-likelihood of the last E-step, iterations, LL history)."""
    ll, hist, it = -np.inf, [], 0
    while it < max_iter:
        r, new_ll, _ = e_step(X, w, mu, cov)
        llp, ll = ll, new_ll
        hist.append(ll)
        w, mu, cov = m_step(X, r)
        it += 1
        if abs(ll - llp) <= tol:
            break
    return w, mu, cov, ll, it, hist
