"""fp64 restatement of Spark's BinaryClassificationEvaluator / BinaryClassificationMetrics (unit weights), written as
plainly as possible, one step per function, for the tests of the binary evaluation.

  score     element 1 of rawPrediction (or the double itself); positive when label > 0.5.
  counts    (positives, negatives) per distinct score, in descending order of Java's Double.compare: NaN (one value)
            above +inf, -0.0 below +0.0.
  bins      numBins > 0 and g = D // numBins >= 2: runs of g consecutive distinct scores merge into one point, the last
            run may be shorter.  The whole ordered list is one partition (Spark groups per partition).
  rates     FPR = FP / N, 0.0 when N == 0; recall = TPR = TP / P, 0.0 when P == 0; precision = TP / (TP + FP), 1.0 when
            TP + FP == 0 (Spark's FalsePositiveRate, Recall, Precision).
  curves    ROC: (0, 0), (FPR, TPR) per point, (1, 1).  PR: (0, precision of the first point), (recall, precision).
  area      trapezoids (x1 - x0) (y1 + y0) / 2 summed in curve order.
"""
import math


def java_key(v):
    """A sort key with Java's Double.compare order."""
    v = float(v)
    if math.isnan(v):
        return (1, 0.0, 0)
    return (0, v, 0 if math.copysign(1.0, v) < 0 else 1)


def score_of(raw):
    if isinstance(raw, (int, float)):
        return float(raw)
    return float(raw[1])


def distinct_counts(scores, labels):
    groups = {}
    for s, y in zip(scores, labels):
        k = java_key(s)
        p, n = groups.get(k, (0, 0))
        groups[k] = (p + 1, n) if y > 0.5 else (p, n + 1)
    return [groups[k] for k in sorted(groups, reverse=True)]


def down_sample(counts, num_bins):
    if num_bins == 0:
        return counts
    g = len(counts) // num_bins
    if g < 2:
        return counts
    out = []
    for i in range(0, len(counts), g):
        run = counts[i:i + g]
        out.append((sum(c[0] for c in run), sum(c[1] for c in run)))
    return out


def confusions(points):
    tp = fp = 0
    out = []
    for p, n in points:
        tp += p
        fp += n
        out.append((tp, fp))
    return out, tp, fp


def roc_curve(scores, labels, num_bins=1000):
    conf, P, N = confusions(down_sample(distinct_counts(scores, labels), num_bins))
    pts = [(0.0, 0.0)]
    for tp, fp in conf:
        pts.append((0.0 if N == 0 else fp / N, 0.0 if P == 0 else tp / P))
    pts.append((1.0, 1.0))
    return pts


def pr_curve(scores, labels, num_bins=1000):
    conf, P, N = confusions(down_sample(distinct_counts(scores, labels), num_bins))
    pts = []
    for tp, fp in conf:
        pts.append((0.0 if P == 0 else tp / P, 1.0 if tp + fp == 0 else tp / (tp + fp)))
    return [(0.0, pts[0][1])] + pts


def area(points):
    total = 0.0
    for (x0, y0), (x1, y1) in zip(points[:-1], points[1:]):
        total += (x1 - x0) * (y1 + y0) / 2.0
    return total


def metric(scores, labels, name="areaUnderROC", num_bins=1000):
    if len(scores) == 0:
        raise ValueError("binary metrics need at least one row")
    if name == "areaUnderROC":
        return area(roc_curve(scores, labels, num_bins))
    if name == "areaUnderPR":
        return area(pr_curve(scores, labels, num_bins))
    raise ValueError(f"Unsupported metric name, found {name}")
