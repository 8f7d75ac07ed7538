"""Writes linreg_known_answers.json: the data and MLlib's expected answers of the reference's LinearRegression
compatibility test (python/tests/test_linear_model.py:458-562 of NVIDIA/spark-rapids-ml).  The features and labels
reach the estimator as float32 columns there ("c0 float, c1 float, ..., label float")."""
import json
import os

X = [[-0.20515826, 1.4940791], [0.12167501, 0.7610377], [1.4542735, 0.14404356], [-0.85409576, 0.3130677],
     [2.2408931, 0.978738], [-0.1513572, 0.95008844], [-0.9772779, 1.867558], [0.41059852, -0.10321885]]
y = [2.0374513, 22.403986, 139.4456, -76.19584, 225.72075, -0.6784152, -65.54835, 37.30829]
cases = {
    "ols": {"regParam": 0.0, "elasticNetParam": 0.0, "coefficients": [94.46689350900762, 14.33532962562045],
            "intercept": -3.3089753423400734e-07, "intercept_atol": 1e-4, "first_prediction": 2.037452415464224},
    "ridge": {"regParam": 2.0, "elasticNetParam": 0.0, "coefficients": [92.22569365, 12.84336458],
              "intercept": 1.76595778134947},
    "elastic_net": {"regParam": 2.0, "elasticNetParam": 0.5, "coefficients": [91.9070094, 11.23076474],
                    "intercept": 3.138371491598421},
}
out = {"X": X, "y": y, "fitIntercept": True, "standardization": True, "cases": cases}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "linreg_known_answers.json"), "w") as f:
    json.dump(out, f, indent=1)
    f.write("\n")
