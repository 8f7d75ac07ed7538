"""MulticlassClassificationEvaluator and RegressionEvaluator: pyspark.ml.evaluation's when pyspark is present, else the
local stand-ins of sparkshim.evaluation (Spark's params, defaults and isLargerBetter(); evaluate() of a local frame in
fp64 on the host).  Both feed the single-pass multi-model evaluation of CrossValidator (tuning.py)."""
from .sparkshim import HAVE_PYSPARK

if HAVE_PYSPARK:
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator, RegressionEvaluator  # noqa: F401
else:
    from .sparkshim.evaluation import MulticlassClassificationEvaluator, RegressionEvaluator  # noqa: F401

__all__ = ["MulticlassClassificationEvaluator", "RegressionEvaluator"]
