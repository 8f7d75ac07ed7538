"""Writes tests/golden/knn_known_answers.json: the known answers of the reference's k-NN toy test, TRANSCRIBED (not
computed) from python/tests/test_nearest_neighbors.py of the reference (func_test_example_no_id, used by test_example
and test_example_with_id).  When the reference sources are present, the literals are first re-checked against them.

  items / queries   the 8 diagonal items and 5 queries with their metadata strings
  k                 topk = 2
  indices           positions into the item list (the test compares against item_ids[...])
  distances         sqrt(2), sqrt(8), sqrt(0.01 + 0.01), sqrt(0.81 + 0.81) as in assert_distances_equal
"""
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/python/tests/test_nearest_neighbors.py"

CASE = {
    "items": [[[1.0, 1.0], "a"], [[2.0, 2.0], "b"], [[3.0, 3.0], "c"], [[4.0, 4.0], "d"], [[5.0, 5.0], "e"],
              [[6.0, 6.0], "f"], [[7.0, 7.0], "g"], [[8.0, 8.0], "h"]],
    "queries": [[[0.0, 0.0], "qa"], [[1.0, 1.0], "qb"], [[4.1, 4.1], "qc"], [[8.0, 8.0], "qd"], [[9.0, 9.0], "qe"]],
    "k": 2,
    "indices": [[0, 1], [0, 1], [3, 4], [7, 6], [7, 6]],
    "distances": [[math.sqrt(2.0), math.sqrt(8.0)], [0.0, math.sqrt(2.0)],
                  [math.sqrt(0.01 + 0.01), math.sqrt(0.81 + 0.81)], [0.0, math.sqrt(2.0)],
                  [math.sqrt(2.0), math.sqrt(8.0)]],
}


def check_transcription() -> None:
    if not os.path.exists(REF):
        print("reference not present; transcription check skipped")
        return
    src = open(REF).read()
    for lit in ['([1.0, 1.0], "a")', '([8.0, 8.0], "h")', '([0.0, 0.0], "qa")', '([4.1, 4.1], "qc")',
                '([9.0, 9.0], "qe")', "topk = 2", "[math.sqrt(2.0), math.sqrt(8.0)]", "[0.0, math.sqrt(2.0)]",
                "[math.sqrt(0.01 + 0.01), math.sqrt(0.81 + 0.81)]", "[item_ids[0], item_ids[1]]",
                "[item_ids[3], item_ids[4]]", "[item_ids[7], item_ids[6]]"]:
        assert lit in src, lit
    print("transcription literals found in", REF)


if __name__ == "__main__":
    check_transcription()
    out = os.path.join(HERE, "knn_known_answers.json")
    with open(out, "w") as f:
        json.dump(CASE, f, indent=1)
        f.write("\n")
    print("wrote", out)
    sys.exit(0)
