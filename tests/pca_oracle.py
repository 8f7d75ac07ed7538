"""fp64 NumPy restatement of the PCA semantics libb2kmeans implements (include/b2kmeans.h, b2k_pca_fit), for the tests
only (the product never imports it):

  mean_ = sum x / n;  cov = (X - mean)^T (X - mean) / (n - 1);  eigenpairs by descending eigenvalue, top k;
  each component signed so that its largest-|value| element (lowest index on a tie) is positive;
  explained_variance_ratio_ = lambda / trace(cov) (0 when the trace is 0);  singular_values_ = sqrt(lambda (n - 1));
  transform(X) = X . components^T (no mean subtracted).
"""
import numpy as np


def sign_fix(components: np.ndarray) -> np.ndarray:
    c = np.array(components, dtype=np.float64, copy=True)
    for i in range(c.shape[0]):
        j = int(np.argmax(np.abs(c[i])))   # first index of the maximum: lowest index wins a tie
        if c[i, j] < 0:
            c[i] = -c[i]
    return c


def covariance(X: np.ndarray) -> np.ndarray:
    X = np.asarray(X, dtype=np.float64)
    Xc = X - X.mean(axis=0)
    return Xc.T @ Xc / (X.shape[0] - 1)


def fit(X: np.ndarray, k: int) -> dict:
    X = np.asarray(X, dtype=np.float64)
    n, d = X.shape
    if not 1 <= k <= d:
        raise ValueError(f"source vector size {d} must be no less than k={k}")
    if n < 2:
        raise ValueError("PCA needs at least 2 rows")
    cov = covariance(X)
    w, V = np.linalg.eigh(cov)
    order = np.argsort(-w, kind="stable")
    lam = np.maximum(w[order[:k]], 0.0)
    comp = sign_fix(V[:, order[:k]].T)
    tr = float(np.trace(cov))
    return {"mean_": X.mean(axis=0), "cov": cov, "eigenvalues": w[order], "components_": comp,
            "explained_variance_ratio_": lam / tr if tr > 0 else np.zeros(k),
            "singular_values_": np.sqrt(lam * (n - 1))}


def transform(X: np.ndarray, components: np.ndarray) -> np.ndarray:
    return np.asarray(X, dtype=np.float64) @ np.asarray(components, dtype=np.float64).T


def relative_gaps(eigenvalues: np.ndarray, k: int) -> np.ndarray:
    """For each of the top k eigenvalues: distance to the nearest other eigenvalue over the largest eigenvalue."""
    w = np.asarray(eigenvalues, dtype=np.float64)
    scale = max(abs(w[0]), 1e-300)
    out = []
    for i in range(k):
        others = np.delete(w, i)
        out.append(np.min(np.abs(others - w[i])) / scale if others.size else np.inf)
    return np.array(out)
