"""fp64 NumPy restatement of the logistic regression semantics in include/b2kmeans.h (b2k_logreg_*), MLlib's objective.

With K' = 1 (binomial) or K (multinomial) margins per row, W [K', d], b [K']:

    minimise (1/n) sum_i l(W x_i + b, y_i) + reg ((1 - a)/2 |V|^2 + a |V|_1),   V = W diag(sigma) (standardization)
                                                                                  or V = W

l is max(m, 0) + log1p(exp(-|m|)) - y m (binomial, y in {0, 1} the class index) or log-sum-exp(m) - m_y (multinomial),
sigma the sample (n - 1) standard deviations of the features; a feature with sigma = 0 has coefficient 0.  The solver
frame is theta = [V (K' x d) | b], W = V / sigma.  Used by the CPU tests (through b2k_logreg_minimize's callback), the
GPU tests, smoke() and bench_logreg.py.
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import numpy as np


def classes_of(y: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(classes, counts, class index of each row)."""
    cls, idx, cnt = np.unique(np.asarray(y, dtype=np.float64), return_inverse=True, return_counts=True)
    return cls, cnt, idx


def sigma(X: np.ndarray) -> np.ndarray:
    X = np.asarray(X, dtype=np.float64)
    return X.std(axis=0, ddof=1) if X.shape[0] > 1 else np.zeros(X.shape[1])


def loss_grad(X: np.ndarray, yi: np.ndarray, W: np.ndarray, b: np.ndarray) -> Tuple[float, np.ndarray, np.ndarray]:
    """(1/n) sum l and its gradient (dW [kp, d], db [kp]) at (W, b); yi are class indices, -1 for a row whose label is
    none of the classes: its one-hot is zero (binomial: a negative row), as b2k_logreg_eval counts it."""
    X = np.asarray(X, dtype=np.float64)
    yi = np.asarray(yi)
    n = X.shape[0]
    M = X @ np.asarray(W, dtype=np.float64).T + np.asarray(b, dtype=np.float64)
    kp = M.shape[1]
    if kp == 1:
        m = M[:, 0]
        yy = (yi == 1).astype(np.float64)
        loss = np.maximum(m, 0) + np.log1p(np.exp(-np.abs(m))) - yy * m
        e = np.exp(-np.abs(m))
        p = np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
        R = (p - yy)[:, None]
    else:
        mx = M.max(axis=1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(M - mx).sum(axis=1))
        rows = np.flatnonzero(yi >= 0)
        loss = lse.copy()
        loss[rows] -= M[rows, yi[rows]]
        R = np.exp(M - lse[:, None])
        R[rows, yi[rows]] -= 1.0
    return float(loss.sum() / n), R.T @ X / n, R.sum(axis=0) / n


class Problem:
    """The solver-frame objective of one fit."""

    def __init__(self, X: np.ndarray, y: np.ndarray, reg: float = 0.0, l1_ratio: float = 0.0,
                 fit_intercept: bool = True, standardization: bool = True, family: str = "auto") -> None:
        self.X = np.asarray(X, dtype=np.float64)
        self.classes, self.counts, self.yi = classes_of(y)
        K = len(self.classes)
        self.multi = family == "multinomial" or (family == "auto" and K > 2)
        self.kp = K if self.multi else 1
        self.d = self.X.shape[1]
        self.fi = fit_intercept
        self.sig = sigma(self.X)
        self.inv = np.where(self.sig > 0, 1.0 / np.where(self.sig > 0, self.sig, 1.0), 0.0)
        self.pen = (self.sig > 0).astype(np.float64) if standardization else self.inv ** 2
        self.reg, self.l1_ratio = float(reg), float(l1_ratio)
        self.l2 = self.reg * (1.0 - self.l1_ratio)
        l1c = self.reg * self.l1_ratio * ((self.sig > 0).astype(np.float64) if standardization else self.inv)
        self.l1 = np.concatenate([np.tile(l1c, self.kp), np.zeros(self.kp if self.fi else 0)])
        self.n_theta = self.kp * self.d + (self.kp if self.fi else 0)

    def split(self, theta: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        nv = self.kp * self.d
        V = np.asarray(theta[:nv]).reshape(self.kp, self.d)
        b = np.asarray(theta[nv:]) if self.fi else np.zeros(self.kp)
        return V, b

    def smooth(self, theta: np.ndarray) -> Tuple[float, np.ndarray]:
        """The smooth part (loss + L2) and its gradient."""
        V, b = self.split(theta)
        loss, gW, gb = loss_grad(self.X, self.yi, V * self.inv, b)
        f = loss + 0.5 * self.l2 * float((self.pen * V * V).sum())
        gV = gW * self.inv + self.l2 * self.pen * V
        g = np.concatenate([gV.ravel(), gb if self.fi else np.zeros(0)])
        return f, g

    def start(self) -> np.ndarray:
        """MLlib's start: zero coefficients, intercepts at the log-odds of the priors."""
        th = np.zeros(self.n_theta)
        if self.fi:
            nv = self.kp * self.d
            if self.multi:
                r = np.log1p(self.counts.astype(np.float64))
                th[nv:] = r - r.mean()
            else:
                th[nv] = np.log(self.counts[1] / self.counts[0])
        return th

    def residual(self, theta: np.ndarray) -> float:
        """Optimality residual: max |grad| on smooth coordinates, |g + w sign(x)| at non-zero L1 coordinates and
        max(|g| - w, 0) at zero ones."""
        _, g = self.smooth(theta)
        w = self.l1
        r = np.where(w == 0, np.abs(g),
                     np.where(theta != 0, np.abs(g + w * np.sign(theta)), np.maximum(np.abs(g) - w, 0.0)))
        return float(r.max())

    def model(self, theta: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """(coef [kp, d], intercept [kp]) as b2k_logreg_fit reports them: W = V / sigma, multinomial centring."""
        V, b = self.split(theta)
        W = V * self.inv
        b = b.copy()
        if self.multi:
            if self.fi:
                b -= b.mean()
            if self.reg == 0.0:
                W = np.where(self.sig > 0, W - W.mean(axis=0, keepdims=True), 0.0)
        return W, b

    def solve_scipy(self, gtol: float = 1e-12, maxiter: int = 20000) -> np.ndarray:
        """The optimum from scipy.optimize: L-BFGS-B on the smooth problem; with an L1 term, on the bound-constrained
        split theta = p - q, p, q >= 0."""
        from scipy.optimize import minimize

        opts = {"gtol": gtol, "ftol": 1e-300, "maxiter": maxiter, "maxcor": 30}
        if not np.any(self.l1 > 0):
            res = minimize(lambda t: self.smooth(t), self.start(), jac=True, method="L-BFGS-B", options=opts)
            return res.x
        m = self.n_theta
        free = self.l1 == 0

        def f2(z: np.ndarray) -> Tuple[float, np.ndarray]:
            p, q = z[:m], z[m:]
            f, g = self.smooth(p - q)
            return f + float(self.l1 @ (p + q)), np.concatenate([g + self.l1, -g + self.l1])

        t0 = self.start()
        z0 = np.concatenate([np.maximum(t0, 0), np.maximum(-t0, 0)])
        bounds = [(None, None) if fr else (0, None) for fr in free] + [(0, 0) if fr else (0, None) for fr in free]
        res = minimize(f2, z0, jac=True, method="L-BFGS-B", bounds=bounds, options=opts)
        return res.x[:m] - res.x[m:]


def predict(X: np.ndarray, W: np.ndarray, b: np.ndarray, classes: np.ndarray) -> Dict[str, np.ndarray]:
    """rawPrediction, probability and prediction as the transform kernel defines them."""
    M = np.asarray(X, dtype=np.float64) @ np.asarray(W, dtype=np.float64).T + np.asarray(b, dtype=np.float64)
    if M.shape[1] == 1:
        m = M[:, 0]
        e = np.exp(-np.abs(m))
        p1 = np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
        return {"raw": np.stack([-m, m], axis=1), "prob": np.stack([1.0 - p1, p1], axis=1),
                "pred": np.asarray(classes, dtype=np.float64)[(m > 0).astype(int)]}
    mx = M.max(axis=1, keepdims=True)
    P = np.exp(M - mx)
    P /= P.sum(axis=1, keepdims=True)
    return {"raw": M, "prob": P, "pred": np.asarray(classes, dtype=np.float64)[M.argmax(axis=1)]}


def eval_bound(X: np.ndarray, W: np.ndarray, b: np.ndarray) -> Dict[str, Any]:
    """Round-off bound of an fp64 evaluation summed over n rows in any fixed order (DESIGN §13.4): with u = 2^-53, a
    margin carries at most (d + 1) u sum |w x| + u |b| error, the residuals and losses a few u on top, and a sum of n
    terms (n + 2) u sum |term|.  Returns the bounds of the loss, of dW and of db as arrays matching their shapes."""
    X = np.asarray(X, dtype=np.float64)
    n, d = X.shape
    u = 2.0 ** -53
    A = np.abs(X) @ np.abs(np.asarray(W, dtype=np.float64)).T + np.abs(b)   # [n, kp] |margin| scale
    kp = A.shape[1]
    em = (d + 4) * u * A.max(axis=1) + 16 * u                                 # per-row margin error (any class)
    c = (n + d + 32) * u
    # residual error of a row <= em (softmax and sigmoid are 1-Lipschitz in each margin up to a factor 2, exp's round-off)
    e_r = 2 * kp * em + 16 * u
    loss_b = float((2 * em + c * (1 + A.max(axis=1))).sum() / n)
    dW_b = (e_r[:, None] * np.abs(X)).sum(axis=0) / n + c * np.abs(X).sum(axis=0) / n
    db_b = float(e_r.sum() / n + c)
    return {"loss": loss_b, "dW": np.tile(dW_b, (kp, 1)), "db": np.full(kp, db_b)}
