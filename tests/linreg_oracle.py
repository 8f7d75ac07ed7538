"""fp64 NumPy restatement of linear regression as include/b2kmeans.h pins it (b2k_linreg_solve), on the float32 rows and
labels the device sees.

With n rows, mu / muy the means (fp64) and sigma the population standard deviations about the mean:
  centring   fit_intercept: mu, muy; else 0 (the data is scaled, not centred)
  scales     standardization: s_j = sigma_j (1 where sigma_j = 0), s_y = sigma_y; else 1
  problem    z = (x - mu) / s, t = (y - muy) / s_y, lam' = reg / s_y; minimise
             (1/2n) |t - Z v|^2 + lam' (alpha |v|_1 + (1 - alpha)/2 |v|^2)
  result     w = v s_y / s, b = muy - w.mu with an intercept, else 0
A constant label under standardization follows MLlib: w = 0, b = muy (0 without an intercept) when fit_intercept or
muy == 0, else s_y = |muy|.  The closed forms (reg == 0 or alpha == 0) are the minimum-norm solution of the normal
equations (numpy.linalg.lstsq); the elastic net is cyclic coordinate descent run to 1e-15.
"""
import numpy as np


def frame(X, y, fit_intercept=True, standardization=True):
    """-> dict(A = Z^T Z / n, c = Z^T t / n, s, sy, mu, muy, const) of the solver's frame, fp64 from float32 data."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    y = np.asarray(y, dtype=np.float32).astype(np.float64)
    n, d = X.shape
    mu, muy = X.mean(0), y.mean()
    s, sy = np.ones(d), 1.0
    const = False
    if standardization:
        sd = np.sqrt(((X - mu) ** 2).mean(0))
        s = np.where(sd > 0, sd, 1.0)
        sy = float(np.sqrt(((y - muy) ** 2).mean()))
        if sy == 0.0:
            if fit_intercept or muy == 0.0:
                const = True
                sy = 1.0
            else:
                sy = abs(muy)
    cm, cy = (mu, muy) if fit_intercept else (np.zeros(d), 0.0)
    Z = (X - cm) / s
    t = (y - cy) / sy
    return {"A": Z.T @ Z / n, "c": Z.T @ t / n, "s": s, "sy": sy, "mu": mu, "muy": muy, "const": const, "Z": Z, "t": t}


def coordinate_descent(A, c, l1, l2, tol=1e-15, max_iter=100000):
    d = len(c)
    v = np.zeros(d)
    for _ in range(max_iter):
        dmax = 0.0
        for j in range(d):
            if A[j, j] <= 0:
                nv = 0.0
            else:
                r = c[j] - A[j] @ v + A[j, j] * v[j]
                nv = np.sign(r) * max(abs(r) - l1, 0.0) / (A[j, j] + l2)
            dmax = max(dmax, abs(nv - v[j]))
            v[j] = nv
        if dmax <= tol * np.abs(v).max(initial=0.0):
            break
    return v


def fit(X, y, reg=0.0, l1_ratio=0.0, fit_intercept=True, standardization=True):
    """-> (coef [d], intercept, frame) in fp64."""
    f = frame(X, y, fit_intercept, standardization)
    d = f["A"].shape[0]
    if f["const"]:
        return np.zeros(d), (f["muy"] if fit_intercept else 0.0), f
    lam = reg / f["sy"]
    l1, l2 = lam * l1_ratio, lam * (1 - l1_ratio)
    if reg == 0.0 or l1_ratio == 0.0:
        # minimum-norm solution of (Z^T Z / n + l2 I) v = Z^T t / n, through the augmented least-squares problem
        n = f["Z"].shape[0]
        Za = np.vstack([f["Z"] / np.sqrt(n), np.sqrt(l2) * np.eye(d)]) if l2 > 0 else f["Z"] / np.sqrt(n)
        ta = np.concatenate([f["t"] / np.sqrt(n), np.zeros(d)]) if l2 > 0 else f["t"] / np.sqrt(n)
        v = np.linalg.lstsq(Za, ta, rcond=None)[0]
    else:
        v = coordinate_descent(f["A"], f["c"], l1, l2)
    w = v * f["sy"] / f["s"]
    b = f["muy"] - w @ f["mu"] if fit_intercept else 0.0
    return w, float(b), f


def solver_frame_v(coef, f):
    """The solver-frame vector v of coefficients w: v = w s / s_y."""
    return np.asarray(coef) * f["s"] / f["sy"]


def kkt_residual(A, c, v, l1, l2):
    """Largest violation of the elastic-net optimality conditions of (A, c): |c_j - (A v)_j - l2 v_j| <= l1 where
    v_j = 0, and c_j - (A v)_j - l2 v_j = l1 sign(v_j) elsewhere."""
    g = c - A @ v - l2 * v
    viol = np.where(v == 0, np.maximum(np.abs(g) - l1, 0.0), np.abs(g - l1 * np.sign(v)))
    return float(viol.max(initial=0.0))


def moments(X, y):
    """(n, mean [d + 1], centred moments [d + 1, d + 1]) of [X | y] in fp64 — what b2k_linreg_moments returns."""
    V = np.c_[np.asarray(X, np.float32).astype(np.float64), np.asarray(y, np.float32).astype(np.float64)]
    m = V.mean(0)
    C = V - m
    return V.shape[0], m, C.T @ C
