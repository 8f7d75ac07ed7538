"""Writes bkm_known_answers.json: bisecting k-means cases whose answers follow by hand from the rules in
include/b2kmeans.h (no solver involved).

- four_points: (0,0), (1,1), (9,8), (8,9), k = 2.  The root centre is (4.5, 4.5); the children start at c -/+ l u with
  u in [0, 1)^2, so the left start has the smaller coordinates and takes (0,0) and (1,1).  One iteration settles the
  children at (0.5, 0.5) and (8.5, 8.5), each of cost 0.5^2 * 4 = 1.0; the training cost is 2.0.
- symmetric: rows symmetric about the origin.  The root centre is 0, so l = 0, both children start at 0, every row
  ties and goes left; the right child is empty and drops out.  With k = 2 one node divides, need reaches 0, and the
  model is the root and its left child (node 2, the only leaf, with every row and the root's cost).
- duplicates: five copies of one row.  The root cost is 0, nothing is divisible, and the root is the only leaf.

    python tests/golden/make_bkm_known_answers.py
"""
import json
import os

CASES = [
    {"name": "four_points", "X": [[0, 0], [1, 1], [9, 8], [8, 9]], "k": 2, "max_iter": 20, "min_divisible": 1.0,
     "node_index": [1, 2, 3], "centers": [[4.5, 4.5], [0.5, 0.5], [8.5, 8.5]], "sizes": [4, 2, 2],
     "costs": [130.0, 1.0, 1.0], "training_cost": 2.0, "cluster_sizes": [2, 2], "labels": [0, 0, 1, 1]},
    {"name": "symmetric", "X": [[1, 2], [-1, -2], [3, -1], [-3, 1]], "k": 2, "max_iter": 5, "min_divisible": 1.0,
     "node_index": [1, 2], "centers": [[0.0, 0.0], [0.0, 0.0]], "sizes": [4, 4], "costs": [30.0, 30.0],
     "training_cost": 30.0, "cluster_sizes": [4], "labels": [0, 0, 0, 0]},
    {"name": "duplicates", "X": [[2, 3]] * 5, "k": 3, "max_iter": 20, "min_divisible": 1.0,
     "node_index": [1], "centers": [[2.0, 3.0]], "sizes": [5], "costs": [0.0], "training_cost": 0.0,
     "cluster_sizes": [5], "labels": [0, 0, 0, 0, 0]},
]

if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "bkm_known_answers.json"), "w") as f:
        json.dump(CASES, f, indent=1)
