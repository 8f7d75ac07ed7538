"""Writes tests/golden/dbscan_known_answers.json: the toy cases of the reference's DBSCAN tests
(python/tests/test_dbscan.py: test_dbscan_basic, test_dbscan_numeric_type) with the labels and core flags that follow
from include/b2kmeans.h's rule, derived by hand below and checked against tests/dbscan_oracle.py.

    python tests/golden/make_dbscan_known_answers.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import dbscan_oracle as do  # noqa: E402

CASES = [
    # four points at eps = 2, min_samples = 2: (0, 0)-(1, 1) at sqrt(2) and (9, 8)-(8, 9) at sqrt(2), 8.5 apart
    {"name": "basic", "X": [[0.0, 0.0], [1.0, 1.0], [9.0, 8.0], [8.0, 9.0]], "eps": 2.0, "min_samples": 2,
     "metric": "euclidean", "labels": [0, 0, 1, 1], "core": [True, True, True, True], "n_clusters": 2},
    # the five integer rows at the defaults (eps = 0.5, min_samples = 5): no two rows within 0.5, every row noise
    {"name": "numeric_type_defaults", "X": [[1, 4, 4, 4, 0], [2, 2, 2, 2, 1], [3, 3, 3, 2, 2], [3, 3, 3, 2, 3],
                                            [5, 2, 1, 3, 4]],
     "eps": 0.5, "min_samples": 5, "metric": "euclidean", "labels": [-1] * 5, "core": [False] * 5, "n_clusters": 0},
]

if __name__ == "__main__":
    import numpy as np

    for c in CASES:
        lab, core, n = do.dbscan(np.array(c["X"], dtype=np.float32), c["eps"], c["min_samples"], c["metric"])
        assert lab.tolist() == c["labels"] and core.tolist() == c["core"] and n == c["n_clusters"], c["name"]
    with open(os.path.join(HERE, "dbscan_known_answers.json"), "w") as f:
        json.dump({"source": "python/tests/test_dbscan.py (test_dbscan_basic, test_dbscan_numeric_type)",
                   "cases": CASES}, f, indent=1)
        f.write("\n")
