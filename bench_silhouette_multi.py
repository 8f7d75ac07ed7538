"""Tuning KMeans' k with the silhouette (b2k_silhouette_multi) per GPU, on blobs made as bench.py makes them (256
centres ~ U(-10, 10)^d, unit noise); model m labels a row by its blob index mod K_m:

  a        10 M x 128, M = 12, K = 2 .. 13 (sum 90: one block of 128 means)     wgmma pass
  b        10 M x 128, M = 6, K = 8, 16, 32, 64, 128, 256 (sum 504)              wgmma pass
  generic  12.5 M x 256, M = 4, K = 16, 32, 64, 128                              fp64 SIMT pass
  cv       CrossValidator(KMeans, ClusteringEvaluator) with 3 folds x 6 maps (k = 2 .. 7) on a 1 M x 128 local frame,
           against the hand loop of fit, transform and evaluate per fold and map

For a, b and generic: the per-pass device times of one multi call (CUDA events, option time_kernels: the ids and the
statistics summed over models, the shared silhouette pass(es)), the whole call (host clock around a synchronised call,
median), and the same for M separate b2k_silhouette calls in the same session; for a, also the single-model K = 64
silhouette pass on the same rows.  The aims below were derived from a single-model table, not measured before; each is
reported as met or not met.  Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import time

from bench_silhouette import card

CASES = {"a": (10_000_000, 128, list(range(2, 14))), "b": (10_000_000, 128, [8, 16, 32, 64, 128, 256]),
         "generic": (12_500_000, 256, [16, 32, 64, 128])}


def blobs(torch, n, d, k=256):
    g = torch.Generator(device="cuda").manual_seed(42)
    C = torch.rand((k, d), generator=g, device="cuda") * 20.0 - 10.0
    g = torch.Generator(device="cuda").manual_seed(1234)
    X = torch.empty((n, d), dtype=torch.float32, device="cuda")
    z = torch.empty((n,), dtype=torch.int64, device="cuda")
    for s in range(0, n, 1_000_000):
        e = min(n, s + 1_000_000)
        z[s:e] = torch.randint(0, k, (e - s,), generator=g, device="cuda")
        X[s:e] = C[z[s:e]] + torch.randn((e - s, d), generator=g, device="cuda")
    return X, z


def timed(torch, ctx, fn, steps, warmup):
    """(median wall ms, mean {ids, stats, silhouette} device ms) of fn() over steps, with option time_kernels."""
    ctx.set_option("time_kernels", 1)
    for _ in range(warmup):
        fn()
    walls, ph = [], {"ids": 0.0, "stats": 0.0, "silhouette": 0.0}
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        walls.append((time.perf_counter() - t0) * 1e3)
        st = ctx.stats()
        for key, f in (("ids", "last_finalize_ms"), ("stats", "last_reduce_ms"), ("silhouette", "last_fused_ms")):
            ph[key] += st[f] / steps
    ctx.set_option("time_kernels", 0)
    return sorted(walls)[len(walls) // 2], ph


def run_case(torch, ctx, name, steps, warmup):
    n, d, Ks = CASES[name]
    X, z = blobs(torch, n, d)
    ids = [z % K for K in Ks]
    before = ctx.stats()["fused_tc_launches"] + ctx.stats()["generic_launches"]
    vals = ctx.silhouette_multi(X, ids)
    passes = ctx.stats()["fused_tc_launches"] + ctx.stats()["generic_launches"] - before
    multi_ms, multi_ph = timed(torch, ctx, lambda: ctx.silhouette_multi(X, ids), steps, warmup)
    sep_ph = {"ids": 0.0, "stats": 0.0, "silhouette": 0.0}
    sep_ms = 0.0
    for i in ids:
        ms, ph = timed(torch, ctx, lambda: ctx.silhouette(X, i), steps, warmup)
        sep_ms += ms
        for key in sep_ph:
            sep_ph[key] += ph[key]
    singles = [ctx.silhouette(X, i) for i in ids]
    out = {"case": name, "n": n, "d": d, "Ks": Ks, "passes": passes, "path": ctx.stats()["last_path"],
           "bits_equal_separate": vals == singles,
           "multi": {"call_ms": round(multi_ms, 3), **{k: round(v, 3) for k, v in multi_ph.items()}},
           "separate": {"call_ms": round(sep_ms, 3), **{k: round(v, 3) for k, v in sep_ph.items()}}}
    if name == "a":
        _, ph64 = timed(torch, ctx, lambda: ctx.silhouette(X, z % 64), steps, warmup)
        out["single_K64_silhouette_ms"] = round(ph64["silhouette"], 3)
        out["aims"] = {"shared_pass<=1.25x_K64_pass": multi_ph["silhouette"] <= 1.25 * ph64["silhouette"],
                       "call<=0.5x_separate": multi_ms <= 0.5 * sep_ms}
    if name == "b":
        out["aims"] = {"shared_pass<=25ms": multi_ph["silhouette"] <= 25.0}
    del X, z, ids
    torch.cuda.empty_cache()
    return out


def run_cv(torch):
    import numpy as np
    import pandas as pd

    from spark_rapids_ml_b200.clustering import KMeans
    from spark_rapids_ml_b200.evaluation import ClusteringEvaluator
    from spark_rapids_ml_b200.sparkshim.sql import LocalSession
    from spark_rapids_ml_b200.tuning import CrossValidator, ParamGridBuilder, k_fold

    X, _ = blobs(torch, 1_000_000, 128, k=6)
    Xh = X.cpu().numpy()
    del X
    df = LocalSession().createDataFrame(pd.DataFrame({"features": list(Xh)}), num_partitions=1)
    km = KMeans(seed=1, maxIter=10)
    maps = ParamGridBuilder().addGrid(km.k, list(range(2, 8))).build()
    ev = ClusteringEvaluator()
    cv = CrossValidator(estimator=km, estimatorParamMaps=maps, evaluator=ev, numFolds=3, seed=5)
    cv.fit(df)   # warm-up
    t0 = time.perf_counter()
    model = cv.fit(df)
    cv_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    hand = []
    for train, valid in k_fold(df, 3, 5, None, int(km.num_workers)):
        hand.append([ev.evaluate(km.copy(pm).fit(train).transform(valid)) for pm in maps])
    km.copy(maps[int(np.argmax(np.mean(hand, axis=0)))]).fit(df)   # the refit CrossValidator also does
    hand_s = time.perf_counter() - t0
    return {"case": "cv", "n": 1_000_000, "d": 128, "folds": 3, "maps": 6, "cv_fit_s": round(cv_s, 2),
            "hand_loop_s": round(hand_s, 2), "best_k": model.bestModel.getK(),
            "avgMetrics_equal_hand_loop": model.avgMetrics == [float(v) for v in np.mean(hand, axis=0)]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="a,b,generic,cv")
    args = ap.parse_args()
    import torch

    from spark_rapids_ml_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_silhouette_multi.py needs a CUDA device")
    res = []
    ctx = _native.Context(0)
    for c in args.cases.split(","):
        res.append(run_cv(torch) if c == "cv" else run_case(torch, ctx, c, args.steps, args.warmup))
    ctx.close()
    print(json.dumps({"bench": "silhouette_multi", **card(), "results": res}))


if __name__ == "__main__":
    main()
