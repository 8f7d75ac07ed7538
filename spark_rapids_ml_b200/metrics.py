"""Multiclass and regression metrics from per-model accumulators, written from Spark's MulticlassMetrics and
RegressionMetrics definitions (unit weights), and the binary metrics (areaUnderROC, areaUnderPR) of Spark's
BinaryClassificationMetrics from scores and labels (binary_metric).

The accumulators are what the device evaluation pass (Context.eval_linear / eval_forest) returns, and what the local
evaluators form from a frame's columns on the host:

  classification  n, label_count [C] (rows per label value), tp [C] (rows predicted right, by label), fp [C] (rows
                  predicted wrong, by predicted value) and loss (sum of -log(max(p_y, eps))).
  regression      reg [3, 5]: for the columns label, label - prediction and prediction, {count, mean, m2n, m2, l1}
                  with m2n the centred sum of squares, m2 the sum of squares and l1 the sum of absolute values.

Accumulators of several partitions or device passes merge in partition order (merge_*).
"""
from __future__ import annotations

import math
from typing import Any, Dict, List, Optional

import numpy as np

MULTICLASS_METRICS = ("f1", "accuracy", "weightedPrecision", "weightedRecall", "weightedTruePositiveRate",
                      "weightedFalsePositiveRate", "weightedFMeasure", "truePositiveRateByLabel",
                      "falsePositiveRateByLabel", "precisionByLabel", "recallByLabel", "fMeasureByLabel", "hammingLoss",
                      "logLoss")
REGRESSION_METRICS = ("rmse", "mse", "r2", "mae", "var")
BINARY_METRICS = ("areaUnderROC", "areaUnderPR")


def _div(a: float, b: float) -> float:
    """a / b with IEEE semantics (Spark's Double division): x / 0 is +-inf, 0 / 0 is NaN."""
    if b == 0:
        return math.nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a)
    return a / b


# ---- classification ----
def class_accumulators(labels: np.ndarray, preds: np.ndarray, probs: Optional[np.ndarray], eps: float) -> Dict[str, Any]:
    """Host accumulators of one model from columns: labels and predictions [n] (integer class values) and the
    probability vectors [n, width] (p_y = probs[row, y], 0 when y >= width) or None."""
    y = np.asarray(labels, dtype=np.float64)
    p = np.asarray(preds, dtype=np.float64)
    for name, v in (("label", y), ("prediction", p)):
        if v.size and (not np.all(np.isfinite(v)) or np.any(v < 0) or np.any(v != np.floor(v))):
            raise ValueError(f"{name} values must be non-negative integers")
    yi, pi = y.astype(np.int64), p.astype(np.int64)
    C = int(max(yi.max(initial=-1), pi.max(initial=-1))) + 1
    lc = np.bincount(yi, minlength=C).astype(np.int64)
    right = yi == pi
    tp = np.bincount(yi[right], minlength=C).astype(np.int64)
    fp = np.bincount(pi[~right], minlength=C).astype(np.int64)
    loss = 0.0
    if probs is not None and y.size:
        P = np.asarray(probs, dtype=np.float64).reshape(y.size, -1)
        inside = yi < P.shape[1]
        py = np.zeros(y.size)
        py[inside] = P[np.nonzero(inside)[0], yi[inside]]
        loss = float(np.sum(-np.log(np.maximum(py, eps))))
    return {"n": int(y.size), "label_count": lc, "tp": tp, "fp": fp, "loss": loss}


def _pad(a: np.ndarray, C: int) -> np.ndarray:
    return np.concatenate([np.asarray(a, dtype=np.int64), np.zeros(C - len(a), dtype=np.int64)])


def merge_class(a: Dict[str, Any], b: Dict[str, Any]) -> Dict[str, Any]:
    """Accumulators of two row sets of one model (a first)."""
    C = max(len(a["label_count"]), len(b["label_count"]))
    return {"n": a["n"] + b["n"], "label_count": _pad(a["label_count"], C) + _pad(b["label_count"], C),
            "tp": _pad(a["tp"], C) + _pad(b["tp"], C), "fp": _pad(a["fp"], C) + _pad(b["fp"], C),
            "loss": a["loss"] + b["loss"]}


def multiclass_metric(acc: Dict[str, Any], metric: str, metric_label: float = 0.0, beta: float = 1.0) -> float:
    """Spark MulticlassMetrics over the labels present (label_count > 0)."""
    n = float(acc["n"])
    lc, tp, fp = (np.asarray(acc[k], dtype=np.int64) for k in ("label_count", "tp", "fp"))
    labels = [int(c) for c in np.nonzero(lc)[0]]

    def tp_of(c: int) -> float:
        return float(tp[c]) if c < len(tp) else 0.0

    def fp_of(c: int) -> float:
        return float(fp[c]) if c < len(fp) else 0.0

    def present(c: float) -> int:
        if c != int(c) or int(c) not in labels:
            raise ValueError(f"metricLabel {c} is not a label of the evaluated rows")
        return int(c)

    def precision(c: int) -> float:
        t, f = tp_of(c), fp_of(c)
        return 0.0 if t + f == 0 else t / (t + f)

    def recall(c: int) -> float:
        return tp_of(c) / float(lc[c])

    def fmeasure(c: int, b: float) -> float:
        p, r = precision(c), recall(c)
        b2 = b * b
        return 0.0 if p + r == 0 else (1 + b2) * p * r / (b2 * p + r)

    def fpr(c: int) -> float:
        return _div(fp_of(c), n - float(lc[c]))

    def weighted(f: Any) -> float:
        return sum(f(c) * float(lc[c]) / n for c in labels)

    if metric not in MULTICLASS_METRICS:
        raise ValueError(f"Unsupported metric name, found {metric}")
    if n == 0:
        return math.nan
    if metric == "f1":
        return weighted(lambda c: fmeasure(c, 1.0))
    if metric == "accuracy":
        return float(tp.sum()) / n
    if metric == "weightedPrecision":
        return weighted(precision)
    if metric in ("weightedRecall", "weightedTruePositiveRate"):
        return weighted(recall)
    if metric == "weightedFalsePositiveRate":
        return weighted(fpr)
    if metric == "weightedFMeasure":
        return weighted(lambda c: fmeasure(c, beta))
    if metric in ("truePositiveRateByLabel", "recallByLabel"):
        return recall(present(metric_label))
    if metric == "falsePositiveRateByLabel":
        return fpr(present(metric_label))
    if metric == "precisionByLabel":
        return precision(present(metric_label))
    if metric == "fMeasureByLabel":
        return fmeasure(present(metric_label), beta)
    if metric == "hammingLoss":
        return float(fp.sum()) / n
    return float(acc["loss"]) / n   # logLoss


# ---- regression ----
def reg_accumulators(labels: np.ndarray, preds: np.ndarray) -> Dict[str, Any]:
    """Host accumulators from columns, two-pass in fp64."""
    y = np.asarray(labels, dtype=np.float64)
    p = np.asarray(preds, dtype=np.float64)
    reg = np.zeros((3, 5))
    for c, v in enumerate((y, y - p, p)):
        if v.size:
            mu = float(np.mean(v))
            reg[c] = (v.size, mu, float(np.sum((v - mu) ** 2)), float(np.sum(v * v)), float(np.sum(np.abs(v))))
    return {"n": int(y.size), "reg": reg}


def chan_merge(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """(count, mean, m2n, m2, l1) of two row sets, a first (Chan et al.)."""
    na, ma, qa = float(a[0]), float(a[1]), float(a[2])
    nb, mb, qb = float(b[0]), float(b[1]), float(b[2])
    if nb == 0:
        return np.array(a, dtype=np.float64)
    if na == 0:
        return np.array(b, dtype=np.float64)
    n = na + nb
    dl = mb - ma
    return np.array([n, ma + dl * (nb / n), qa + qb + dl * dl * (na * nb / n), a[3] + b[3], a[4] + b[4]])


def merge_reg(a: Dict[str, Any], b: Dict[str, Any]) -> Dict[str, Any]:
    return {"n": a["n"] + b["n"], "reg": np.stack([chan_merge(a["reg"][c], b["reg"][c]) for c in range(3)])}


def regression_metric(acc: Dict[str, Any], metric: str, through_origin: bool = False) -> float:
    """Spark RegressionMetrics: SSerr = m2 (label - prediction), SStot = m2n (label), SSy = m2 (label), explained
    variance = (m2 (prediction) + mean(label)^2 n - 2 mean(label) mean(prediction) n) / n."""
    if metric not in REGRESSION_METRICS:
        raise ValueError(f"Unsupported metric name, found {metric}")
    r = np.asarray(acc["reg"], dtype=np.float64)
    n = float(r[0][0])
    if n == 0:
        return math.nan
    sserr = float(r[1][3])
    if metric == "mse":
        return sserr / n
    if metric == "rmse":
        return math.sqrt(sserr / n)
    if metric == "mae":
        return float(r[1][4]) / n
    if metric == "r2":
        return 1.0 - _div(sserr, float(r[0][3]) if through_origin else float(r[0][2]))
    ymean, pmean = float(r[0][1]), float(r[2][1])
    ssreg = float(r[2][3]) + ymean * ymean * n - 2.0 * ymean * pmean * n
    return ssreg / n   # var


def merge_all(accs: List[Dict[str, Any]], classification: bool) -> Dict[str, Any]:
    out = accs[0]
    for a in accs[1:]:
        out = merge_class(out, a) if classification else merge_reg(out, a)
    return out


# ---- binary ----
def _descending_key(scores: np.ndarray) -> np.ndarray:
    """uint64 keys whose ascending order is Java's Double.compare order descending: NaN (one value) first, then +inf
    down to -inf, +0.0 before -0.0."""
    b = np.where(np.isnan(scores), np.uint64(0x7FF8000000000000), np.ascontiguousarray(scores).view(np.uint64))
    neg = (b >> np.uint64(63)) == 1
    asc = np.where(neg, ~b, b | np.uint64(1 << 63))
    return ~asc


def binary_metric(scores: Any, labels: Any, metric: str, num_bins: int) -> float:
    """Spark's BinaryClassificationMetrics(scoreAndLabels, numBins).areaUnderROC / areaUnderPR with unit weights, the
    whole ordered list of distinct scores as one partition (include/b2kmeans.h "binary evaluation" states the rule).
    A row is positive when its label > 0.5."""
    if metric not in BINARY_METRICS:
        raise ValueError(f"Unsupported metric name, found {metric}")
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    pos = np.asarray(labels, dtype=np.float64).reshape(-1) > 0.5
    if s.size == 0:
        raise ValueError("binary metrics need at least one row")
    key = _descending_key(s)
    order = np.argsort(key, kind="stable")
    key, cpos = key[order], np.cumsum(pos[order])
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])   # first row of each distinct score
    g = len(starts) // num_bins if num_bins > 0 else 0
    if g >= 2:
        starts = starts[::g]
    last = np.r_[starts[1:], s.size] - 1                        # last row of each point
    tp = cpos[last].astype(np.float64)
    fp = (last + 1).astype(np.float64) - tp
    P = float(cpos[-1])
    N = float(s.size) - P
    recall = tp / P if P > 0 else np.zeros_like(tp)
    if metric == "areaUnderROC":
        x = np.r_[0.0, fp / N if N > 0 else np.zeros_like(fp), 1.0]
        y = np.r_[0.0, recall, 1.0]
    else:
        with np.errstate(invalid="ignore"):
            precision = np.where(tp + fp == 0, 1.0, tp / (tp + fp))
        x = np.r_[0.0, recall]
        y = np.r_[precision[0], precision]
    return float(np.sum((x[1:] - x[:-1]) * (y[1:] + y[:-1]) / 2.0))
