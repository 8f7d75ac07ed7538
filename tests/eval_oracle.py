"""High-precision oracles of the evaluation passes (b2k_eval.cu, b2k_binary.cu), restated from Spark's definitions and
independent of the product's host path (metrics.py):

  linear_margins        margins of float32 rows under fp64 models, in extended precision, with the per-entry bound beta
                        of the device's fp64 FMA chains and the rows whose predicted class that bound does not settle.
  classification_acc    label counts, tp and fp (integers) and the log-loss sum (math.fsum) from explicit predictions.
  regression_acc        per column (label, label - prediction, prediction): count, mean, m2n, m2, l1 (math.fsum).
  binary_counts / area  areaUnderROC / areaUnderPR vectorised: sort on Java's Double.compare key, run starts and
                        cumulative counts, numBins' groups, trapezoids summed by math.fsum.
"""
import math

import numpy as np

U = 2.0 ** -53          # unit round-off of fp64
EXT = np.longdouble     # the oracle's precision for the margins (x86-64: a 64-bit significand)


def _check_extended():
    assert np.finfo(EXT).nmant >= 63, "linear_margins needs an extended-precision numpy.longdouble"


def linear_margins(X, W, b, binomial=False):
    """X [n, d] float32, W [K, d] and b [K] fp64 -> (m [n, K] fp64 margins, beta [n, K], unsettled row indices).

    The device forms each margin as b + (fp64 FMA chains over the features, split over L lanes and added by a butterfly):
    at most d + 1 roundings, each within 2^-53 of the running value, so |device - exact| <= (d + 1) 2^-53 S with
    S = sum_j |x_j w_kj| + |b_k|.  The oracle's own error here is below (d + 1) 2^-64 S, so beta = (d + 1) 2^-52 S bounds
    |device - oracle| with room to spare.  A row is unsettled when its predicted class could differ between the two:
    the top-two margin gap <= 2 max(beta) (softmax), or |m| <= beta (binomial, K = 1)."""
    _check_extended()
    X = np.asarray(X, dtype=np.float32)
    W = np.atleast_2d(np.asarray(W, dtype=np.float64))
    b = np.asarray(b, dtype=np.float64).reshape(-1)
    n, d = X.shape
    Xe, We = X.astype(EXT), W.astype(EXT)
    m = (Xe @ We.T + b.astype(EXT)).astype(np.float64)
    S = np.abs(X.astype(np.float64)) @ np.abs(W).T + np.abs(b)
    beta = (d + 1) * 2.0 ** -52 * S
    if W.shape[0] == 1 or binomial:
        unsettled = np.nonzero(np.abs(m[:, 0]) <= beta[:, 0])[0]
    else:
        top2 = np.sort(m, axis=1)[:, -2:]
        unsettled = np.nonzero(top2[:, 1] - top2[:, 0] <= 2.0 * beta.max(axis=1))[0]
    return m, beta, unsettled


def linear_predictions(m, kind, class_values):
    """(predicted class value [n], the label index -> probability function) of margins m [n, K'] as k_eval_linear's
    finish defines them: binomial class 1 when m > 0, softmax the lowest index of the largest margin."""
    cv = np.asarray(class_values, dtype=np.float64)
    if kind == "logistic":
        mm = m[:, 0].astype(EXT)
        p1 = 1.0 / (1.0 + np.exp(-mm))
        probs = np.stack([1.0 - p1, p1], axis=1)
        return cv[(m[:, 0] > 0.0).astype(np.int64)], probs
    me = m.astype(EXT)
    e = np.exp(me - me.max(axis=1, keepdims=True))
    return cv[np.argmax(m, axis=1)], e / e.sum(axis=1, keepdims=True)


def label_prob(probs, y):
    """p_y per row: the probability vector at index y, 0 when y is beyond the model's classes."""
    yi = np.asarray(y).astype(np.int64)
    K = probs.shape[1]
    inside = yi < K
    out = np.zeros(yi.size, dtype=probs.dtype)
    out[inside] = probs[np.nonzero(inside)[0], yi[inside]]
    return out


def classification_acc(y, pred, py, C, eps=1e-15):
    """Spark's per-label counts from explicit predictions: label_count [C], tp [C] (label c predicted c), fp [C]
    (predicted c, label not c) as int64, and loss = fsum of -log(max(p_y, eps))."""
    yi = np.asarray(y).astype(np.int64)
    pi = np.asarray(pred).astype(np.int64)
    label_count = np.bincount(yi, minlength=C).astype(np.int64)
    tp = np.bincount(yi[yi == pi], minlength=C).astype(np.int64)
    fp = np.bincount(pi[yi != pi], minlength=C).astype(np.int64)
    pe = np.maximum(np.asarray(py, dtype=EXT), EXT(eps))
    loss = math.fsum((-np.log(pe)).astype(np.float64).tolist())
    return {"label_count": label_count, "tp": tp, "fp": fp, "loss": loss}


def _moments(v):
    """count, mean, m2n (centred sum of squares), m2 (sum of squares), l1 of one column, each sum by math.fsum."""
    n = v.size
    if n == 0:
        return [0.0, 0.0, 0.0, 0.0, 0.0]
    mean = math.fsum(v.tolist()) / n
    c = v.astype(EXT) - EXT(mean)
    m2n = math.fsum((c * c).astype(np.float64).tolist())
    ve = v.astype(EXT)
    return [float(n), mean, m2n, math.fsum((ve * ve).astype(np.float64).tolist()), math.fsum(np.abs(v).tolist())]


def regression_acc(y, pred):
    """[3, 5]: columns label, label - prediction, prediction; stats count, mean, m2n, m2, l1.  The label is read as
    float32 (as the device stages it); the residual is the fp64 difference rounded once, as the device forms it."""
    yy = np.asarray(y, dtype=np.float32).astype(np.float64)
    p = np.asarray(pred, dtype=np.float64)
    return np.array([_moments(yy), _moments(yy - p), _moments(p)], dtype=np.float64)


# ---- binary metrics ----
def java_keys(scores):
    """int64 keys whose ascending order is Java's Double.compare: -0.0 below +0.0, every NaN one value above +inf."""
    s = np.asarray(scores, dtype=np.float64).copy()
    s[np.isnan(s)] = np.nan                      # the canonical (positive) NaN
    u = s.view(np.int64)
    return np.where(u < 0, u ^ np.int64(0x7FFFFFFFFFFFFFFF), u)


def binary_counts(scores, labels):
    """(positives, negatives) per distinct score in descending Double.compare order, as int64 arrays."""
    k = java_keys(scores)
    if k.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    pos = np.asarray(labels, dtype=np.float64) > 0.5
    order = np.argsort(k, kind="stable")[::-1]
    ks, ps = k[order], pos[order]
    start = np.ones(ks.size, dtype=bool)
    start[1:] = ks[1:] != ks[:-1]
    ends = np.r_[np.nonzero(start)[0][1:], ks.size] - 1
    cpos = np.cumsum(ps, dtype=np.int64)
    tp_end = cpos[ends]
    rows_end = ends + 1
    p = np.diff(np.r_[0, tp_end])
    return p, np.diff(np.r_[0, rows_end]) - p


def binary_area(p, q, name="areaUnderROC", num_bins=1000):
    """The metric of distinct-score counts (p, q) (binary_counts): numBins' groups of g = D // numBins >= 2 consecutive
    scores (the last group may be shorter), cumulative TP / FP per point, the curve, and the trapezoids by fsum."""
    if p.size == 0:
        raise ValueError("binary metrics need at least one row")
    D = p.size
    g = D // num_bins if num_bins > 0 else 0
    if g < 2:
        g = 1
    tp_all, fp_all = np.cumsum(p), np.cumsum(q)
    last = np.r_[np.arange(g - 1, D - 1, g), D - 1] if g > 1 else np.arange(D)
    last = np.unique(last)
    tp, fp = tp_all[last].astype(np.float64), fp_all[last].astype(np.float64)
    P, N = float(tp_all[-1]), float(fp_all[-1])
    recall = tp / P if P else np.zeros_like(tp)
    if name == "areaUnderROC":
        fpr = fp / N if N else np.zeros_like(fp)
        x, yv = np.r_[0.0, fpr, 1.0], np.r_[0.0, recall, 1.0]
    elif name == "areaUnderPR":
        tot = tp + fp
        with np.errstate(invalid="ignore", divide="ignore"):
            prec = np.where(tot == 0, 1.0, tp / np.where(tot == 0, 1.0, tot))
        x, yv = np.r_[0.0, recall], np.r_[prec[0], prec]
    else:
        raise ValueError(f"Unsupported metric name, found {name}")
    return math.fsum(((x[1:] - x[:-1]) * (yv[1:] + yv[:-1]) / 2.0).tolist())


def binary_metric(scores, labels, name="areaUnderROC", num_bins=1000):
    p, q = binary_counts(scores, labels)
    return binary_area(p, q, name, num_bins)
