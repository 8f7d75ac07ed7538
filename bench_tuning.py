"""Single-pass multi-model evaluation (b2k_eval_linear / b2k_eval_forest) against M predict passes and an fp64 torch
baseline, at 10 M x 128 validation rows on one GPU, then _transformEvaluate and CrossValidator end to end.

Prints the card's name and power limit, then one JSON line per measurement.  Run: python bench_tuning.py [--n N]."""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from spark_rapids_ml_b200 import _native

FP64_PEAK = 34e12   # H100 SXM non-tensor FP64, data sheet


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / 1e3)
    return best


def emit(**kw):
    print(json.dumps(kw), flush=True)


def linear_workloads(ctx, X, yc, yr, n, d):
    rng = np.random.default_rng(0)
    out = []
    for name, kind, K, M, y in (("binomial M=1", "logistic", 1, 1, yc[2]), ("binomial M=4", "logistic", 1, 4, yc[2]),
                                ("binomial M=12", "logistic", 1, 12, yc[2]), ("multinomial K=10 M=4", "softmax", 10, 4,
                                                                               yc[10]),
                                ("linear regression M=12", "identity", 1, 12, yr)):
        models = []
        for _ in range(M):
            W = rng.normal(scale=0.1, size=(K, d))
            b = rng.normal(size=K)
            md = {"kind": kind, "W": W, "b": b}
            if kind != "identity":
                md["class_values"] = np.arange(2 if K == 1 else K, dtype=np.float64)
            models.append(md)
        t = timed(lambda: ctx.eval_linear(X, y, models))
        if kind == "identity":
            tp = timed(lambda: [ctx.linreg_predict(X, m["W"][0], float(m["b"][0])) for m in models], reps=3)
        else:
            tp = timed(lambda: [ctx.logreg_predict(X, m["W"], m["b"], m["class_values"]) for m in models], reps=3)
        Wt = torch.as_tensor(np.concatenate([m["W"] for m in models]), device=X.device)

        def torch_base():
            S = X.double() @ Wt.T
            if kind == "identity":
                r = y.double()[:, None] - S
                return (r * r).sum(0)
            lab = y.long()
            for i in range(M):
                s = S[:, i * K:(i + 1) * K]
                p = (s[:, 0] > 0).long() if K == 1 else s.argmax(1)
                torch.bincount(lab * 16 + p, minlength=16 * 16)

        tt = timed(torch_base, reps=3)
        flop = M * K * 2 * d * n
        bw = n * d * 4 / t
        rec = dict(workload=name, n=n, d=d, eval_s=t, x_tb_s=bw / 1e12, fp64_tflop_s=flop / t / 1e12,
                   m_predict_s=tp, torch_fp64_s=tt, speedup_vs_predict=tp / t, speedup_vs_torch=tt / t)
        if M * K <= 16:
            rec["aim_2TBs"] = "met" if bw >= 2e12 else "not met"
        if K == 10:
            rec["aim_2x_fp64_bound"] = "met" if t <= 2 * flop / FP64_PEAK else "not met"
        emit(**rec)
        out.append(rec)
    return out


def forest_workload(ctx, X, y, n, d):
    sub = X[: 200_000].contiguous()
    ys = y[: 200_000].contiguous()
    forests = [ctx.rf_fit(sub, ys, n_trees=20, max_depth=5, impurity="gini", seed=s) for s in range(4)]
    t = timed(lambda: ctx.eval_forest(X, y, forests, True))
    tp = timed(lambda: [ctx.rf_predict(X, f, True) for f in forests], reps=3)
    emit(workload="rf classification 20 trees depth 5 M=4", n=n, d=d, eval_s=t, x_tb_s=n * d * 4 / t / 1e12,
         m_predict_s=tp, speedup_vs_predict=tp / t)


def end_to_end(d):
    import pandas as pd

    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.evaluation import MulticlassClassificationEvaluator
    from spark_rapids_ml_b200.sparkshim import LocalSession
    from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder, k_fold

    rng = np.random.default_rng(1)
    n = 1_000_000
    Xh = rng.normal(size=(n, d)).astype(np.float32)
    yh = (Xh @ rng.normal(size=d) > 0).astype(np.float32)
    df = LocalSession().createDataFrame(pd.DataFrame({"features": list(Xh), "label": yh}), num_partitions=2)
    lr = LogisticRegression(maxIter=10)
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.01, 0.1]).addGrid(lr.elasticNetParam, [0.0, 1.0]).build()
    ev = MulticlassClassificationEvaluator(metricName="accuracy")
    models = [m for _, m in sorted(lr.fitMultiple(df, grid), key=lambda t: t[0])]
    comb = models[0]._combine(models)
    t0 = time.perf_counter()
    comb._transformEvaluate(df, ev)
    t1 = time.perf_counter()
    [ev.evaluate(m.transform(df)) for m in models]
    t2 = time.perf_counter()
    emit(workload="_transformEvaluate 1M x %d, M=6" % d, single_pass_s=t1 - t0, hand_loop_s=t2 - t1,
         speedup=(t2 - t1) / (t1 - t0))
    cv = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=1)
    t0 = time.perf_counter()
    cv.fit(df)
    t1 = time.perf_counter()
    for tr, va in k_fold(df, 3, 1, None, 2):
        [ev.evaluate(lr.fit(tr, pm).transform(va)) for pm in grid]
    lr.fit(df, grid[0])
    t2 = time.perf_counter()
    emit(workload="CrossValidator 3 folds x 6 maps, 1M x %d" % d, cv_fit_s=t1 - t0, hand_loop_s=t2 - t1,
         speedup=(t2 - t1) / (t1 - t0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tuning.py needs a GPU")
    print("card:", card(), flush=True)
    ctx = _native.Context(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randn(a.n, a.d, device="cuda", generator=g)
    s = X[:, :8].sum(1)
    yc = {2: (s > 0).float().contiguous(),
          10: torch.clamp(((s + 6) * (10 / 12)).floor(), 0, 9).float().contiguous()}
    yr = (s + torch.randn(a.n, device="cuda", generator=g)).contiguous()
    linear_workloads(ctx, X, yc, yr, a.n, a.d)
    forest_workload(ctx, X, yc[10], a.n, a.d)
    del X
    torch.cuda.empty_cache()
    end_to_end(a.d)
    ctx.close()


if __name__ == "__main__":
    main()
