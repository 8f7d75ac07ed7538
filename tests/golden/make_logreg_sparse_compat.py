"""Writes logreg_sparse_compat.json: the two sparse datasets of the reference's python/tests/test_logistic_regression.py
(test_compat_sparse_binomial :1591-1612, whose second row is a dense vector among sparse ones, and
test_compat_sparse_multinomial :1643-1664), both fitted with regParam = 0.1, standardization off, with and without an
intercept.  Spark cannot run here, so the answers are the fp64 oracle's optimum (tests/logreg_oracle.py, scipy's
L-BFGS-B to a gradient of 1e-12), reported as b2k_logreg_fit reports a model.
Run: python tests/golden/make_logreg_sparse_compat.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import logreg_oracle as lo  # noqa: E402


def sparse(size, entries):
    return {"type": 0, "size": size, "indices": sorted(entries), "values": [entries[i] for i in sorted(entries)]}


def dense(values):
    return {"type": 1, "size": None, "indices": None, "values": values}


DATASETS = {
    "binomial": ([sparse(3, {2: 1.0}), dense([0.0, 1.0, 0.0]), sparse(3, {0: 1.0}), sparse(3, {0: 2.0, 2: -1.0})],
                 [1.0, 1.0, 0.0, 0.0]),
    "multinomial": ([sparse(3, {2: 1.0}), sparse(3, {1: 1.0}), sparse(3, {0: 1.0}), sparse(3, {0: 2.0, 2: -1.0})],
                    [1.0, 1.0, 0.0, 2.0]),
}


def densify(rows):
    X = np.zeros((len(rows), 3))
    for i, r in enumerate(rows):
        if r["type"] == 1:
            X[i] = r["values"]
        else:
            X[i, r["indices"]] = r["values"]
    return X


cases = []
for name, (rows, y) in DATASETS.items():
    for fi in (True, False):
        p = lo.Problem(densify(rows), np.array(y), reg=0.1, fit_intercept=fi, standardization=False)
        theta = p.solve_scipy()
        assert p.residual(theta) <= 1e-9, p.residual(theta)
        W, b = p.model(theta)
        cases.append({"name": f"{name}_fi{int(fi)}", "rows": rows, "y": y, "regParam": 0.1, "fitIntercept": fi,
                      "standardization": False, "coefficientMatrix": W.tolist(), "interceptVector": b.tolist()})
with open(os.path.join(HERE, "logreg_sparse_compat.json"), "w") as f:
    json.dump({"source": "reference python/tests/test_logistic_regression.py: test_compat_sparse_binomial and "
                         "test_compat_sparse_multinomial; answers from tests/logreg_oracle.py", "cases": cases}, f,
              indent=1)
