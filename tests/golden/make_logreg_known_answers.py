"""Writes logreg_known_answers.json: MLlib's published answers for the fixtures of the reference's
python/tests/test_logistic_regression.py, transcribed by hand (test_compat :684-736, test_compat_multinomial :987-999).
test_compat fits regParam = 0.01 (elasticNetParam 0) on 4 rows, with and without an intercept and standardization;
test_compat_multinomial fits regParam = 0.1, elasticNetParam = 0.2, standardization off, family multinomial, on 8 rows;
test_compat_standardization (:1883-1955) fits regParam = 0.01 with standardization on 8000 rows whose first feature is
scaled by 1000 and shifted by 50.  Those rows come from the reference's seeded recipe (python/tests/utils.py:198-220:
make_classification(n_samples=10000, n_features=2, n_classes=2, n_informative=2, n_redundant=0, n_repeated=0,
random_state=0), train_test_split(train_size=0.8, random_state=10), cast to float32) and are stored beside the answers
in logreg_standardization.npz.
Run: python tests/golden/make_logreg_known_answers.py"""
import json
import os

import numpy as np

X4 = [[1.0, 2.0], [1.0, 3.0], [2.0, 1.0], [3.0, 1.0]]
Y4 = [1.0, 1.0, 0.0, 0.0]
X8 = X4 + [[-1.0, -2.0], [-1.0, -3.0], [-2.0, -1.0], [-3.0, -1.0]]
Y8 = Y4 + [3.0, 3.0, 2.0, 2.0]
cases = []
for std, coef, prob in ((True, [-2.48197058, 2.48197058], [0.07713181, 0.92286819]),
                        (False, [-2.42377087, 2.42377087], [0.0814, 0.9186])):
    for fi in (True, False):
        cases.append({"name": f"binomial_std{int(std)}_fi{int(fi)}", "X": X4, "y": Y4, "regParam": 0.01,
                      "elasticNetParam": 0.0, "fitIntercept": fi, "standardization": std, "family": "auto",
                      "coefficientMatrix": [coef], "interceptVector": [0.0], "first_row_probability": prob,
                      "first_row_rawPrediction": [-coef[1], coef[1]],
                      "first_row_prediction": 1.0})
for fi in (True, False):
    cases.append({"name": f"multinomial_fi{int(fi)}", "X": X8, "y": Y8, "regParam": 0.1, "elasticNetParam": 0.2,
                  "fitIntercept": fi, "standardization": False, "family": "multinomial",
                  "coefficientMatrix": [[0.96766883, -0.06190176], [-0.06183558, 0.96774077],
                                        [-0.96773398, 0.06184808], [0.06187553, -0.96768212]],
                  "interceptVector": [1.78813821e-07, 2.82220935e-05, 1.44387586e-05, 4.82081663e-09] if fi else
                  [0.0, 0.0, 0.0, 0.0],
                  "classes": [0.0, 1.0, 2.0, 3.0]})
from sklearn.datasets import make_classification  # noqa: E402
from sklearn.model_selection import train_test_split  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
X, y = make_classification(n_samples=10000, n_features=2, n_classes=2, n_informative=2, n_redundant=0, n_repeated=0,
                           random_state=0)
X_train, _, y_train, _ = train_test_split(X, y, train_size=0.8, random_state=10)
X_train, y_train = X_train.astype(np.float32), y_train.astype(np.float32)
X_train[:, 0] *= 1000   # in float32, as the reference's test does
X_train[:, 0] += 50
np.savez_compressed(os.path.join(HERE, "logreg_standardization.npz"), X=X_train, y=y_train)
for fi, coef, icpt in ((False, [-1.59550205e-04, 1.35555146e00], 0.0),
                       (True, [-1.63432342e-04, 1.35951030e00], -0.05060137)):
    cases.append({"name": f"standardization_fi{int(fi)}", "data": "logreg_standardization.npz", "regParam": 0.01,
                  "elasticNetParam": 0.0, "fitIntercept": fi, "standardization": True, "family": "auto",
                  "coefficientMatrix": [coef], "interceptVector": [icpt]})
with open(os.path.join(HERE, "logreg_known_answers.json"), "w") as f:
    json.dump({"source": "reference python/tests/test_logistic_regression.py (MLlib's answers)", "cases": cases}, f,
              indent=1)
