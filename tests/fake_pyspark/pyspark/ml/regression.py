"""Stand-ins for the STOCK pyspark.ml.regression classes (what install.py's proxy must keep returning to pyspark.ml
itself and for names it does not accelerate)."""


class LinearRegression:
    stock = True


class LinearRegressionModel:
    stock = True


class RandomForestRegressor:
    stock = True
