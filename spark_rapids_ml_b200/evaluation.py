"""MulticlassClassificationEvaluator, RegressionEvaluator and BinaryClassificationEvaluator: pyspark.ml.evaluation's
when pyspark is present, else the local stand-ins of sparkshim.evaluation (Spark's params, defaults and
isLargerBetter(); evaluate() of a local frame in fp64 on the host).  All three feed the single-pass multi-model
evaluation of CrossValidator (tuning.py)."""
from .sparkshim import HAVE_PYSPARK

if HAVE_PYSPARK:
    from pyspark.ml.evaluation import (  # noqa: F401
        BinaryClassificationEvaluator,
        MulticlassClassificationEvaluator,
        RegressionEvaluator,
    )
else:
    from .sparkshim.evaluation import (  # noqa: F401
        BinaryClassificationEvaluator,
        MulticlassClassificationEvaluator,
        RegressionEvaluator,
    )

__all__ = ["MulticlassClassificationEvaluator", "RegressionEvaluator", "BinaryClassificationEvaluator"]
