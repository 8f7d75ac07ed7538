"""NumPy oracle of the evaluation accumulators and metrics: straight from Spark's definitions, per label, no merging."""
import numpy as np


def multiclass(y, p, probs, metric, metric_label=0.0, beta=1.0, eps=1e-15):
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    n = y.size
    labels = sorted(set(y.tolist()))

    def tp(c):
        return float(np.sum((y == c) & (p == c)))

    def fp(c):
        return float(np.sum((y != c) & (p == c)))

    def cnt(c):
        return float(np.sum(y == c))

    def prec(c):
        return 0.0 if tp(c) + fp(c) == 0 else tp(c) / (tp(c) + fp(c))

    def rec(c):
        return tp(c) / cnt(c)

    def fm(c, b):
        a, r = prec(c), rec(c)
        return 0.0 if a + r == 0 else (1 + b * b) * a * r / (b * b * a + r)

    def fpr(c):
        return fp(c) / (n - cnt(c)) if n - cnt(c) else float("nan")

    w = {c: cnt(c) / n for c in labels}
    if metric == "accuracy":
        return float(np.mean(y == p))
    if metric == "f1":
        return sum(fm(c, 1.0) * w[c] for c in labels)
    if metric == "weightedFMeasure":
        return sum(fm(c, beta) * w[c] for c in labels)
    if metric == "weightedPrecision":
        return sum(prec(c) * w[c] for c in labels)
    if metric in ("weightedRecall", "weightedTruePositiveRate"):
        return sum(rec(c) * w[c] for c in labels)
    if metric == "weightedFalsePositiveRate":
        return sum(fpr(c) * w[c] for c in labels)
    if metric in ("truePositiveRateByLabel", "recallByLabel"):
        return rec(metric_label)
    if metric == "falsePositiveRateByLabel":
        return fpr(metric_label)
    if metric == "precisionByLabel":
        return prec(metric_label)
    if metric == "fMeasureByLabel":
        return fm(metric_label, beta)
    if metric == "hammingLoss":
        return float(np.mean(y != p))
    if metric == "logLoss":
        P = np.asarray(probs, dtype=np.float64)
        py = np.array([P[i, int(c)] if int(c) < P.shape[1] else 0.0 for i, c in enumerate(y)])
        return float(np.mean(-np.log(np.maximum(py, eps))))
    raise ValueError(metric)


def regression(y, p, metric, through_origin=False):
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    n = y.size
    err = y - p
    if metric == "mse":
        return float(np.mean(err ** 2))
    if metric == "rmse":
        return float(np.sqrt(np.mean(err ** 2)))
    if metric == "mae":
        return float(np.mean(np.abs(err)))
    if metric == "r2":
        den = np.sum(y ** 2) if through_origin else np.sum((y - y.mean()) ** 2)
        return float(1 - np.sum(err ** 2) / den)
    if metric == "var":
        return float(np.sum(p ** 2) / n + y.mean() ** 2 - 2 * y.mean() * p.mean())
    raise ValueError(metric)
