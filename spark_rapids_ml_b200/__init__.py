"""spark_rapids_ml_b200 — H100-native (sm_90a) backend for spark-rapids-ml's distributed KMeans.fit() path.

Host side mirrors the reference's operator interface (spark_rapids_ml.clustering.KMeans / KMeansModel,
core._CumlEstimator worker scaffolding, common.cuml_context.CumlContext); the arithmetic is hand-written CUDA
behind the C ABI in include/b2kmeans.h (libb2kmeans.so).  No cuML, no Triton, no CPU fallback.
"""
__version__ = "0.1.0"
