"""Writes tests/golden/ann_known_answers.json: known answers of IVF-Flat, TRANSCRIBED (not computed) from the reference
(spark_rapids_ml.knn.ApproximateNearestNeighbors' docstring example, and tests/test_approximate_nearest_neighbors.py
test_return_fewer_k with ivfflat), as this project's semantics give them:

  docstring      six diagonal items, queries (0, 0) and (50, 50), nlist 2, nprobe 1, k 2.  The training subset (rows
                 1, 3, 5) gives either pair of centres {(1, 1), (40, 40)} or {(15.5, 15.5), (50, 50)} from any random
                 init, and both give the reference's answer.
  return_fewer_k four items (0, 0), (0, 0), (2, 2), (2, 2) searched for themselves, nlist 4, nprobe 1, k 4.  The
                 reference trains on any number of rows; here nlist may not exceed the training rows, so the case uses
                 kmeans_trainset_fraction 1.0.  Each duplicate pair forms one list (ties go to the lowest centre) and
                 the other two lists stay empty, so each query finds two items: the reference's "probed" answer.
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
INF = float("inf")

CASES = {
    "docstring": {
        "items": [[0, [0.0, 0.0]], [1, [1.0, 1.0]], [2, [2.0, 2.0]], [3, [30.0, 30.0]], [4, [40.0, 40.0]],
                  [5, [50.0, 50.0]]],
        "queries": [[10, [0.0, 0.0]], [11, [50.0, 50.0]]],
        "k": 2, "algoParams": {"nlist": 2, "nprobe": 1},
        "centers": [[[1.0, 1.0], [40.0, 40.0]], [[15.5, 15.5], [50.0, 50.0]]],
        "indices": [[0, 1], [5, 4]],
        "distances": [[0.0, 1.4142134], [0.0, 14.142137]],
    },
    "return_fewer_k": {
        "items": [[0, [0.0, 0.0]], [1, [0.0, 0.0]], [2, [2.0, 2.0]], [3, [2.0, 2.0]]],
        "queries": [[0, [0.0, 0.0]], [1, [0.0, 0.0]], [2, [2.0, 2.0]], [3, [2.0, 2.0]]],
        "k": 4, "algoParams": {"nlist": 4, "nprobe": 1, "kmeans_trainset_fraction": 1.0},
        "centers": [[[0.0, 0.0], [0.0, 0.0], [2.0, 2.0], [2.0, 2.0]]],
        "indices": [[0, 1, 0, 0], [0, 1, 0, 0], [2, 3, 2, 2], [2, 3, 2, 2]],
        "distances": [[0.0, 0.0, INF, INF], [0.0, 0.0, INF, INF], [0.0, 0.0, INF, INF], [0.0, 0.0, INF, INF]],
    },
}

if __name__ == "__main__":
    with open(os.path.join(HERE, "ann_known_answers.json"), "w") as f:
        json.dump(CASES, f, indent=1)
        f.write("\n")
