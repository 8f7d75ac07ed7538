"""Writes tests/golden/pca_known_answers.json: the known answers of the reference's PCA tests, TRANSCRIBED (not
computed) from python/tests/test_pca.py of the reference (the reference's arithmetic, cuML, is not part of it).  When
the reference sources are present, the literals are first re-checked against them.

  test_fit               test_pca.py:117-147
  test_fit_rectangle     test_pca.py:150-188
  test_pca_basic data    test_pca.py:251
  test_pca_spark_compat  test_pca.py:402-465 (the sparse rows written out densely)

Signs: the reference compares components and transformed rows without sign (array_equal(..., with_sign=False)), so the
fixture marks them "up_to_sign".
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/python/tests/test_pca.py"

CASES = {
    "fit": {"data": [[1.0, 1.0], [2.0, 2.0], [3.0, 3.0]], "k": 1, "mean": [2.0, 2.0],
            "components": [[0.707, 0.707]], "explained_variance_ratio": [1.0], "rel_tol": 1e-3},
    "fit_rectangle": {"data": [[1.0, 1.0], [1.0, 3.0], [5.0, 1.0], [5.0, 3.0]], "k": 2, "mean": [3.0, 2.0],
                      "components": [[1.0, 0.0], [0.0, 1.0]], "explained_variance_ratio": [0.8, 0.2],
                      "rel_tol": 1e-3},
    "pca_basic": {"data": [[1.0, 1.0, 1.0], [1.0, 3.0, 2.0], [5.0, 1.0, 3.9], [5.0, 3.0, 2.9]], "k": 2},
    "spark_compat": {
        "data": [[0.0, 1.0, 0.0, 7.0, 0.0], [2.0, 0.0, 3.0, 4.0, 5.0], [4.0, 0.0, 0.0, 6.0, 7.0],
                 [0.0, 1.0, 0.0, 7.0, 0.0], [2.0, 0.0, 3.0, 4.0, 5.0], [4.0, 0.0, 0.0, 6.0, 7.0]],
        "k": 2,
        "explained_variance_ratio": [0.7943932532230531, 0.20560674677694699],
        # model.pc as a [d][k] matrix: DenseMatrix(5, 2, values, False) is column-major
        "pc_columns": [[-0.4486, 0.133, -0.1252, 0.2165, -0.8477], [-0.2842, -0.0562, 0.7636, -0.5653, -0.1156]],
        "first_transformed_row": [1.6485728230883814, -4.0132827005162985],
        "up_to_sign": True,
    },
}


def check_transcription() -> None:
    if not os.path.exists(REF):
        print("reference not present; transcription check skipped")
        return
    src = open(REF).read()
    for lit in ["[[1.0, 1.0], [2.0, 2.0], [3.0, 3.0]]", "[[1.0, 1.0], [1.0, 3.0], [5.0, 1.0], [5.0, 3.0]]",
                "pytest.approx(0.707, 0.001)", "pytest.approx(0.8, 0.001)", "pytest.approx(0.2, 0.001)",
                "[[1.0, 1.0, 1.0], [1.0, 3.0, 2.0], [5.0, 1.0, 3.9], [5.0, 3.0, 2.9]]",
                "Vectors.sparse(5, [(1, 1.0), (3, 7.0)])", "Vectors.dense([2.0, 0.0, 3.0, 4.0, 5.0])",
                "Vectors.dense([4.0, 0.0, 0.0, 6.0, 7.0])", "[1.6485728230883814, -4.0132827005162985]",
                "[0.7943932532230531, 0.20560674677694699]", "-0.4486", "0.133", "-0.1252", "0.2165", "-0.8477",
                "-0.2842", "-0.0562", "0.7636", "-0.5653", "-0.1156"]:
        assert lit in src, lit
    print("transcription literals found in", REF)


if __name__ == "__main__":
    check_transcription()
    out = os.path.join(HERE, "pca_known_answers.json")
    with open(out, "w") as f:
        json.dump(CASES, f, indent=1)
        f.write("\n")
    print("wrote", out)
    sys.exit(0)
