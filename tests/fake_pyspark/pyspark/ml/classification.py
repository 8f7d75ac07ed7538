"""Stand-ins for the STOCK pyspark.ml.classification classes (what install.py's proxy must keep returning to pyspark.ml
itself and for names it does not accelerate)."""


class LogisticRegression:
    stock = True


class LogisticRegressionModel:
    stock = True


class RandomForestClassifier:
    stock = True
