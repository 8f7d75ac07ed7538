"""The fp64 oracles of tests/eval_oracle.py pinned without a GPU: the vectorised binary metric against the plain
binary_oracle restatement, the accumulators against tuning_oracle's per-label metrics, and the margins against exact
sums, on random inputs and on hand-made ones (ties, NaN, +-0, +-inf, single-class sets, g = 2 with a short last run)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import binary_oracle
import eval_oracle as eo
import tuning_oracle

NAMES = ("areaUnderROC", "areaUnderPR")


def _close(a, b, rel=1e-12):
    return abs(a - b) <= rel * max(abs(a), abs(b)) or a == b


# ---- binary metric ----
def test_java_keys_order():
    vals = [math.nan, math.inf, 1.5, 0.0, -0.0, -1e-300, -2.0, -math.inf, -math.nan]
    k = eo.java_keys(vals)
    assert k[0] == k[-1]                                 # every NaN is one value
    assert list(np.argsort(-k[:-1].astype(object))) == list(range(len(vals) - 1))   # strictly descending as listed
    assert len(set(k[:-1].tolist())) == len(vals) - 1
    assert [binary_oracle.java_key(v) for v in vals[:-1]] == sorted([binary_oracle.java_key(v) for v in vals[:-1]],
                                                                     reverse=True)


def test_counts_hand_made():
    p, q = eo.binary_counts([0.9, 0.9, 0.5, 0.5, 0.1, math.nan, -0.0, 0.0], [1, 0, 1, 1, 0, 1, 0, 1])
    # NaN, 0.9, 0.5, 0.1, +0.0, -0.0
    assert p.tolist() == [1, 1, 2, 0, 1, 0] and q.tolist() == [0, 1, 0, 1, 0, 1]
    assert binary_oracle.distinct_counts([0.9, 0.9, 0.5, 0.5, 0.1, math.nan, -0.0, 0.0],
                                         [1, 0, 1, 1, 0, 1, 0, 1]) == list(zip(p.tolist(), q.tolist()))


@pytest.mark.parametrize("scores,labels,bins,roc,pr", [
    ([0.9, 0.9, 0.5, 0.5, 0.1], [1, 0, 1, 1, 0], 0, 7 / 12, 7 / 12),
    ([0.3] * 4, [1, 0, 0, 1], 1000, 0.5, 0.5),
    ([5, 4, 3, 2, 1], [1, 0, 1, 0, 0], 2, 2 / 3, 1 / 2),           # g = 2: {5, 4}, {3, 2}, {1} (short last run)
    ([math.nan, 2.0, 1.0, math.nan], [0, 1, 0, 1], 0, 0.625, 0.5 * (0.5 + 0.5) / 2 + 0.5 * (0.5 + 2 / 3) / 2),
    ([-0.0, 0.0], [0, 1], 0, 1.0, 1.0),
    ([math.inf, -math.inf, 0.0], [0, 1, 1], 0, 0.0, None),
    ([3.0, 2.0, 1.0], [0, 0, 0], 0, 0.0, 0.0),
    ([3.0, 2.0, 1.0], [1, 1, 1], 0, 1.0, 1.0),
    ([1.0, 1.0], [0.7, 0.2], 0, 0.5, 0.5),
])
def test_binary_hand_made(scores, labels, bins, roc, pr):
    for name, want in zip(NAMES, (roc, pr)):
        got = eo.binary_metric(scores, labels, name, bins)
        assert got == pytest.approx(binary_oracle.metric(scores, labels, name, bins), rel=1e-15, abs=1e-15)
        if want is not None:
            assert got == pytest.approx(want, abs=1e-15)


def _scores(kind, n, rng):
    if kind == "continuous":
        return rng.normal(size=n)
    if kind == "rounded":
        return np.round(rng.normal(size=n), 3)
    if kind == "two":
        return rng.choice([-0.5, 2.0], size=n)
    if kind == "one":
        return np.full(n, 0.25)
    s = np.round(rng.normal(size=n), 1)          # "edges": NaN, +-inf, +-0 among ties
    s[: n // 10] = np.nan
    s[n // 10: n // 8] = np.inf
    s[n // 8: n // 6] = -np.inf
    s[n // 6: n // 5] = -0.0
    s[n // 5: n // 4] = 0.0
    return rng.permutation(s)


@pytest.mark.parametrize("kind", ["continuous", "rounded", "two", "one", "edges"])
@pytest.mark.parametrize("labels", ["random", "alternating", "one_positive", "one_negative", "all_neg", "all_pos"])
def test_binary_matches_plain_oracle(kind, labels):
    rng = np.random.default_rng(hash((kind, labels)) % 2 ** 32)
    n = 1501
    s = _scores(kind, n, rng)
    y = {"random": rng.integers(0, 2, n), "alternating": np.arange(n) % 2,
         "one_positive": np.eye(1, n, 700)[0], "one_negative": 1 - np.eye(1, n, 3)[0],
         "all_neg": np.zeros(n), "all_pos": np.ones(n)}[labels].astype(np.float64)
    p, q = eo.binary_counts(s, y)
    D = p.size
    for bins in sorted({0, 1, 2, 7, 1000, D // 2, max(D - 1, 0), D + 5}):
        for name in NAMES:
            want = binary_oracle.metric(list(s), list(y), name, bins)
            got = eo.binary_area(p, q, name, bins)
            assert _close(got, want), (kind, labels, bins, name, got, want)


def test_binary_empty_raises():
    with pytest.raises(ValueError, match="at least one row"):
        eo.binary_metric([], [], "areaUnderROC", 0)


# ---- classification accumulators ----
def _metrics_from_acc(acc, n, label):
    """A few of Spark's metrics from the accumulators: accuracy, weighted precision / recall / F1, precisionByLabel."""
    cnt, tp, fp = acc["label_count"], acc["tp"], acc["fp"]
    labels = np.nonzero(cnt)[0]
    prec = {c: (tp[c] / (tp[c] + fp[c]) if tp[c] + fp[c] else 0.0) for c in range(cnt.size)}
    rec = {c: tp[c] / cnt[c] for c in labels}
    f1 = {c: (2 * prec[c] * rec[c] / (prec[c] + rec[c]) if prec[c] + rec[c] else 0.0) for c in labels}
    w = {c: cnt[c] / n for c in labels}
    return {"accuracy": tp.sum() / n, "weightedPrecision": sum(prec[c] * w[c] for c in labels),
            "weightedRecall": sum(rec[c] * w[c] for c in labels), "f1": sum(f1[c] * w[c] for c in labels),
            "precisionByLabel": prec[label], "logLoss": acc["loss"] / n}


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_classification_acc_matches_multiclass(seed):
    rng = np.random.default_rng(seed)
    n, K, C = 2000, 5, 7                       # labels 5 and 6 lie beyond the model's classes: p_y = 0
    y = rng.integers(0, C, n)
    P = rng.dirichlet(np.ones(K), size=n)
    P[:50] = np.eye(K)[rng.integers(0, K, 50)]  # p_y may be exactly 0: the eps clip
    pred = np.argmax(P, axis=1)
    py = eo.label_prob(P, y)
    assert np.all(py[y >= K] == 0.0)
    acc = eo.classification_acc(y, pred, py, C)
    assert acc["label_count"].sum() == n and acc["tp"].sum() + acc["fp"].sum() == n
    got = _metrics_from_acc(acc, n, 1.0)
    for name, v in got.items():
        if name == "precisionByLabel":
            want = tuning_oracle.multiclass(y, pred, P, name, metric_label=1.0)
        else:
            want = tuning_oracle.multiclass(y, pred, P, name)
        assert _close(v, want), (name, v, want)


def test_classification_acc_single_class_and_hand_made():
    acc = eo.classification_acc([0, 0, 0], [0, 0, 0], [1.0, 0.5, 0.0], 2, eps=1e-15)
    assert acc["label_count"].tolist() == [3, 0] and acc["tp"].tolist() == [3, 0] and acc["fp"].tolist() == [0, 0]
    assert acc["loss"] == pytest.approx(math.log(2.0) - math.log(1e-15), rel=1e-15)
    acc = eo.classification_acc([2, 1, 0, 3], [1, 1, 2, 0], [0.2, 0.7, 0.1, 0.0], 4)
    assert acc["tp"].tolist() == [0, 1, 0, 0] and acc["fp"].tolist() == [1, 1, 1, 0]


# ---- regression accumulators ----
@pytest.mark.parametrize("offset,scale", [(0.0, 1.0), (1e6, 1.0), (0.0, 1e-6)])
def test_regression_acc_matches_regression(offset, scale):
    rng = np.random.default_rng(3)
    n = 5000
    y = ((offset + rng.normal(size=n)) * scale).astype(np.float32)
    p = (offset + rng.normal(size=n) * 0.9) * scale
    R = eo.regression_acc(y, p)
    yy = y.astype(np.float64)
    assert R[:, 0].tolist() == [n, n, n]
    mse = R[1, 3] / n
    assert _close(mse, tuning_oracle.regression(yy, p, "mse"), 1e-12)
    assert _close(R[1, 4] / n, tuning_oracle.regression(yy, p, "mae"), 1e-12)
    assert _close(1 - R[1, 3] / R[0, 2], tuning_oracle.regression(yy, p, "r2"), 1e-9)
    assert _close(1 - R[1, 3] / R[0, 3], tuning_oracle.regression(yy, p, "r2", through_origin=True), 1e-12)
    var = R[2, 3] / n + R[0, 1] ** 2 - 2 * R[0, 1] * R[2, 1]
    want = tuning_oracle.regression(yy, p, "var")
    assert abs(var - want) <= 1e-9 * (R[2, 3] / n)   # both cancel sums of squares of size offset^2
    # the moments themselves, exactly in rationals on a short prefix
    v = [Fraction(float(a)) for a in yy[:200]]
    mean = sum(v) / 200
    assert _close(eo.regression_acc(y[:200], p[:200])[0, 1], float(mean), 1e-15)
    assert _close(eo.regression_acc(y[:200], p[:200])[0, 2], float(sum((a - mean) ** 2 for a in v)), 1e-14)


def test_regression_acc_empty_and_constant():
    R = eo.regression_acc(np.full(10, 3.0, np.float32), np.full(10, 3.0))
    assert R[0].tolist() == [10, 3.0, 0.0, 90.0, 30.0] and R[1].tolist() == [10, 0.0, 0.0, 0.0, 0.0]
    assert eo.regression_acc(np.zeros(0, np.float32), np.zeros(0)).tolist() == [[0.0] * 5] * 3


# ---- margins ----
def test_margins_exact_and_bound():
    rng = np.random.default_rng(4)
    n, d, K = 40, 37, 5
    X = (rng.normal(size=(n, d)) * 10.0 ** rng.integers(-3, 4, size=(n, d))).astype(np.float32)
    W, b = rng.normal(size=(K, d)), rng.normal(size=K)
    m, beta, _ = eo.linear_margins(X, W, b)
    for i in range(n):
        for k in range(K):
            exact = sum(Fraction(float(X[i, j])) * Fraction(W[k, j]) for j in range(d)) + Fraction(b[k])
            # the final rounding to fp64 (2^-53 |m|) plus the extended sums: far inside beta / (d + 1)
            assert abs(Fraction(m[i, k]) - exact) <= Fraction(beta[i, k]) / (d + 1)
    # a plain fp64 chain (the device's shape of computation) stays within beta
    plain = np.array([[float(b[k]) + _fma_chain(X[i], W[k]) for k in range(K)] for i in range(n)])
    assert np.all(np.abs(plain - m) <= beta)


def _fma_chain(x, w):
    acc = 0.0
    for a, c in zip(x.astype(np.float64), w):
        acc = acc + a * c
    return acc


def test_margins_unsettled_rows():
    X = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]], dtype=np.float32)
    W = np.array([[1.0, 2.0], [1.0, 0.5], [0.0, 0.0]])
    _, _, un = eo.linear_margins(X, W, np.zeros(3))
    assert un.tolist() == [0]                         # row 0: classes 0 and 1 tie
    _, _, un = eo.linear_margins(X, np.array([[1.0, -1.0]]), np.array([0.0]))
    assert un.tolist() == [2]                         # binomial margin 0
    _, _, un = eo.linear_margins(X, np.array([[1.0, -1.0]]), np.array([1e-300]))
    assert un.tolist() == [2]                         # within beta of 0
    _, _, un = eo.linear_margins(X, np.array([[1.0, -1.0]]), np.array([0.25]))
    assert un.tolist() == []


def test_linear_predictions():
    m = np.array([[0.5, 0.5, -1.0], [-2.0, 0.0, 3.0]])
    pred, P = eo.linear_predictions(m, "softmax", [4.0, 5.0, 9.0])
    assert pred.tolist() == [4.0, 9.0]                # the lowest class of a tie
    assert np.allclose(P.sum(axis=1).astype(np.float64), 1.0, rtol=0, atol=1e-18)
    pred, P = eo.linear_predictions(np.array([[0.0], [1e-300], [-3.0]]), "logistic", [3.0, 7.0])
    assert pred.tolist() == [3.0, 7.0, 3.0]
    assert float(P[2, 1]) == pytest.approx(1 / (1 + math.exp(3.0)), rel=1e-15)
    assert eo.label_prob(P, [0, 1, 7]).astype(np.float64).tolist() == pytest.approx(
        [0.5, 0.5, 0.0], abs=1e-15)
