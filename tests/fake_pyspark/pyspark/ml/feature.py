"""Stand-ins for the STOCK pyspark.ml.feature classes (what install.py's proxy must keep returning to pyspark.ml itself
and for names it does not accelerate)."""


class PCA:
    stock = True


class PCAModel:
    stock = True


class StandardScaler:
    stock = True
