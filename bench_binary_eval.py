"""Binary evaluation (areaUnderROC) at 10 M x 128 validation rows on one GPU: the score pass (b2k_eval_linear_scores /
b2k_eval_forest_scores) and the curve pass (b2k_eval_binary) against M predict passes plus the host metric, then
_transformEvaluate against M transform() calls plus a host evaluate() on a 1 M-row local frame.

Prints the card's name and power limit, then one JSON line per measurement.  Run: python bench_binary_eval.py [--n N]."""
import argparse
import time

import numpy as np
import torch

from bench_tuning import card, emit, timed
from spark_rapids_ml_b200 import _native, metrics


def host_loop(predict, y_host, M):
    """M predict passes, each copied back and scored by the host metric (what transform() + evaluate() compute)."""
    t0 = time.perf_counter()
    for i in range(M):
        raw = predict(i)
        metrics.binary_metric(raw[:, 1].cpu().numpy(), y_host, "areaUnderROC", 1000)
    return time.perf_counter() - t0


def device_run(ctx, X, y, n, d, name, M, score, predict, y_host):
    scores, pos = ctx.binary_buffers(M, n)
    t_score = timed(lambda: score(scores, pos))
    t_curve = timed(lambda: ctx.eval_binary(scores, pos, 1000, "areaUnderROC"), reps=3)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    score(scores, pos)
    ctx.eval_binary(scores, pos, 1000, "areaUnderROC")
    t_dev = time.perf_counter() - t0
    t_host = host_loop(predict, y_host, M)
    distinct = int(torch.unique(scores[0]).numel())
    emit(workload=name, n=n, d=d, M=M, distinct_scores_model0=distinct, score_pass_s=t_score,
         x_tb_s=n * d * 4 / t_score / 1e12, sort_curve_s=t_curve, device_total_s=t_dev,
         predict_plus_host_metric_s=t_host, speedup=t_host / t_dev)
    del scores, pos


def linear(ctx, X, y, n, d, y_host):
    rng = np.random.default_rng(0)
    for M in (1, 4, 12):
        models = [{"kind": "logistic", "W": rng.normal(scale=0.1, size=(1, d)), "b": rng.normal(size=1),
                   "class_values": np.array([0.0, 1.0])} for _ in range(M)]
        device_run(ctx, X, y, n, d, "binomial logistic", M,
                   lambda s, p: ctx.binary_scores_linear(X, y, models, s, p),
                   lambda i: ctx.logreg_predict(X, models[i]["W"], models[i]["b"], models[i]["class_values"])[0],
                   y_host)


def forests(ctx, X, y, n, d, y_host):
    sub, ys = X[:200_000].contiguous(), y[:200_000].contiguous()
    for depth, label in ((5, "rf 20 trees depth 5"), (2, "rf 20 trees depth 2 (heavily tied)")):
        fs = [ctx.rf_fit(sub, ys, n_trees=20, max_depth=depth, impurity="gini", seed=s) for s in range(4)]
        device_run(ctx, X, y, n, d, label, 4, lambda s, p: ctx.binary_scores_forest(X, y, fs, s, p),
                   lambda i: ctx.rf_predict(X, fs[i], True)[0], y_host)


def end_to_end(d):
    import pandas as pd

    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.evaluation import BinaryClassificationEvaluator
    from spark_rapids_ml_b200.sparkshim import LocalSession

    rng = np.random.default_rng(1)
    n = 1_000_000
    Xh = rng.normal(size=(n, d)).astype(np.float32)
    yh = (Xh @ rng.normal(size=d) + rng.normal(scale=4.0, size=n) > 0).astype(np.float32)
    df = LocalSession().createDataFrame(pd.DataFrame({"features": list(Xh), "label": yh}), num_partitions=2)
    lr = LogisticRegression(maxIter=10)
    grid = [{lr.regParam: r} for r in (0.0, 0.01, 0.1, 1.0)]
    models = [m for _, m in sorted(lr.fitMultiple(df, grid), key=lambda t: t[0])]
    comb = models[0]._combine(models)
    ev = BinaryClassificationEvaluator()
    comb._transformEvaluate(df, ev)   # warm
    t0 = time.perf_counter()
    got = comb._transformEvaluate(df, ev)
    t1 = time.perf_counter()
    want = [ev.evaluate(m.transform(df)) for m in models]
    t2 = time.perf_counter()
    emit(workload="_transformEvaluate 1M x %d, binomial M=4" % d, single_pass_s=t1 - t0, hand_loop_s=t2 - t1,
         speedup=(t2 - t1) / (t1 - t0), max_rel_diff=float(np.max(np.abs(np.subtract(got, want)) / np.abs(want))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_binary_eval.py needs a GPU")
    emit(card=card())
    ctx = _native.Context(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randn(a.n, a.d, device="cuda", generator=g)
    y = (X[:, :8].sum(1) + 2.0 * torch.randn(a.n, device="cuda", generator=g) > 0).float().contiguous()
    y_host = y.cpu().numpy()
    linear(ctx, X, y, a.n, a.d, y_host)
    forests(ctx, X, y, a.n, a.d, y_host)
    del X
    torch.cuda.empty_cache()
    end_to_end(a.d)
    ctx.close()


if __name__ == "__main__":
    main()
