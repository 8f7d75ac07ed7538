"""Random-forest benchmark on one GPU: b2k_rf_fit's passes at Spark's defaults (numTrees 20, maxDepth 5, maxBins 32) and
at maxBins 128 on 10 M x 128 rows (binary classification and regression), and one deeper case (1 M x 128, numTrees
100, maxDepth 12).  Seeded synthetic data is generated on the device.  Per case it prints one JSON line:

  card, power limit      nvidia-smi, read in the same run
  phases (ms)            edges (checks, labels, sample, sort, thresholds; host clock), bin pass, histogram passes,
                         their allreduces, split + route (the rest of the fit), device times from option time_kernels
  bin pass TB/s          (n d 4 bytes read + n d bytes written) / bin pass time
  level rates            per level: (row, tree, feature slot) updates with weight > 0 / that level's histogram time
  fit_ms                 the whole fit (host clock, after a warm-up fit of the same shape)
  transform rows/s       k_rf_predict over the training rows
  torch baseline         level 0's histogram by torch scatter_add_ (int64, one tree at a time), same run
  scikit-learn           RandomForest* with the same trees / depth / features on a 1 M-row subsample (CPU, all cores;
                         the core count is printed), held-out accuracy / RMSE beside ours on the same 200 k held-out rows

    python bench_rf.py [--rows N] [--deep-rows N] [--no-sklearn]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

AIMS = {"bin_tbs": 2.5, "level0_ms": 5.0, "default_fit_ms": 100.0}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({e})", "unknown"


def make_data(torch, n, d, regression, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    X = torch.randn((n, d), generator=g, device="cuda", dtype=torch.float32)
    noise = torch.randn((n,), generator=g, device="cuda", dtype=torch.float32)
    if regression:
        y = 2.0 * torch.sin(X[:, 0]) + X[:, 1] ** 2 + 0.3 * noise
    else:
        y = ((X[:, 0] + 0.5 * X[:, 1] * X[:, 2] + 0.3 * noise) > 0).float()
    return X.contiguous(), y.contiguous()


def torch_level0(torch, X, y, forest_args, regression):
    """Level 0's histogram with torch: bins by bucketize against the same thresholds is not available here, so the
    baseline bins by a uniform grid of the same bin count; it times the scatter_add_ of n T k updates."""
    n, d = X.shape
    T, k, B = forest_args["n_trees"], forest_args["features_per_node"], forest_args["max_bins"]
    V = 2
    lo, hi = X.min(0).values, X.max(0).values
    bins = ((X - lo) / (hi - lo + 1e-12) * (B - 1)).round().to(torch.int64)
    lab = y.to(torch.int64).clamp(0, 1) if not regression else torch.zeros(n, dtype=torch.int64, device="cuda")
    H = torch.zeros(T * k * B * V, dtype=torch.int64, device="cuda")
    ones = torch.ones(n * k, dtype=torch.int64, device="cuda")
    feats = [torch.randperm(d, device="cuda")[:k] for _ in range(T)]
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(T):
        sub = bins[:, feats[t]]                                              # [n, k]
        idx = ((t * k + torch.arange(k, device="cuda")[None, :]) * B + sub) * V + lab[:, None]
        H.scatter_add_(0, idx.reshape(-1), ones)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def run_case(torch, ctx, name, n, d, regression, args_fit, sklearn_rows, held_out, do_sklearn):
    from spark_rapids_ml_b200.tree import features_per_node

    X, y = make_data(torch, n + held_out, d, regression, seed=sum(map(ord, name)))
    Xtr, ytr, Xte, yte = X[:n], y[:n], X[n:], y[n:]
    k = features_per_node("auto", d, args_fit["n_trees"], not regression)
    fa = dict(args_fit, features_per_node=k, impurity="variance" if regression else "gini", seed=1)
    ctx.set_option("time_kernels", 0)
    ctx.rf_fit(Xtr, ytr, **fa)                 # warm-up of the same shape
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    forest = ctx.rf_fit(Xtr, ytr, **fa)
    fit_ms = (time.perf_counter() - t0) * 1e3
    ctx.set_option("time_kernels", 1)
    forest_t = ctx.rf_fit(Xtr, ytr, **fa)
    st = ctx.stats()
    ctx.set_option("time_kernels", 0)
    assert st["last_path"] in (1, 2)
    lvl_ms, lvl_up = forest_t["level_ms"], forest_t["level_updates"]
    levels = [{"level": i, "ms": round(float(lvl_ms[i]), 3), "updates": int(lvl_up[i]),
               "G_updates_per_s": round(float(lvl_up[i]) / (lvl_ms[i] * 1e6), 2) if lvl_ms[i] > 0 else None}
              for i in range(len(lvl_ms)) if lvl_up[i] > 0]
    bin_ms = st["last_reduce_ms"]
    split_route = st["last_loop_ms"] - st["last_finalize_ms"] - bin_ms - st["last_fused_ms"] - st["last_allreduce_ms"]
    # transform
    ctx.rf_predict(Xte, forest, not regression)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, _, pred_tr = ctx.rf_predict(Xtr, forest, not regression)
    e1.record()
    torch.cuda.synchronize()
    tr_ms = e0.elapsed_time(e1)
    _, _, pred = ctx.rf_predict(Xte, forest, not regression)
    yt = yte.cpu().numpy()
    pr = pred.cpu().numpy()
    ours = float((pr == yt).mean()) if not regression else float(np.sqrt(((pr - yt) ** 2).mean()))
    res = {"case": name, "rows": n, "d": d, **{k2: v for k2, v in fa.items() if k2 != "seed"},
           "path": "cluster" if st["last_path"] == 2 else "generic", "nodes": int(forest["tree_offsets"][-1]),
           "phases_ms": {"edges": round(st["last_finalize_ms"], 2), "bin": round(bin_ms, 3),
                         "histogram": round(st["last_fused_ms"], 3), "allreduce": round(st["last_allreduce_ms"], 3),
                         "split_route": round(split_route, 2)},
           "bin_TBps": round((n * d * 5) / (bin_ms * 1e9), 3) if bin_ms > 0 else None,
           "levels": levels, "fit_ms": round(fit_ms, 1), "histogram_passes": st["recheck_rows"],
           "transform_rows_per_s": round(n / (tr_ms * 1e-3)), "held_out": "accuracy" if not regression else "rmse",
           "ours_held_out": round(ours, 4)}
    res["torch_scatter_add_level0_ms"] = round(torch_level0(torch, Xtr, ytr, dict(fa, max_bins=fa["max_bins"]),
                                                            regression), 2)
    if do_sklearn:
        from sklearn.ensemble import RandomForestClassifier as SkC, RandomForestRegressor as SkR

        m = min(sklearn_rows, n)
        Xs, ys = Xtr[:m].cpu().numpy(), ytr[:m].cpu().numpy()
        Sk = SkR if regression else SkC
        sk = Sk(n_estimators=fa["n_trees"], max_depth=fa["max_depth"], max_features=k / d, n_jobs=-1, random_state=0)
        t0 = time.perf_counter()
        sk.fit(Xs, ys)
        sk_s = time.perf_counter() - t0
        sp = sk.predict(Xte.cpu().numpy())
        theirs = float((sp == yt).mean()) if not regression else float(np.sqrt(((sp - yt) ** 2).mean()))
        res["sklearn"] = {"rows": m, "cores": os.cpu_count(), "fit_s": round(sk_s, 2),
                          "held_out": round(theirs, 4)}
    del X, y
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--deep-rows", type=int, default=1_000_000)
    ap.add_argument("--held-out", type=int, default=200_000)
    ap.add_argument("--sklearn-rows", type=int, default=1_000_000)
    ap.add_argument("--no-sklearn", action="store_true")
    a = ap.parse_args()
    import torch

    from spark_rapids_ml_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_rf.py needs a CUDA device")
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "cpu_cores": os.cpu_count()}), flush=True)
    out = []
    with _native.Context(0) as ctx:
        for case, n, regression, fit in (
                ("classification_default", a.rows, False, dict(n_trees=20, max_depth=5, max_bins=32)),
                ("classification_bins128", a.rows, False, dict(n_trees=20, max_depth=5, max_bins=128)),
                ("regression_default", a.rows, True, dict(n_trees=20, max_depth=5, max_bins=32)),
                ("regression_bins128", a.rows, True, dict(n_trees=20, max_depth=5, max_bins=128)),
                ("classification_deep", a.deep_rows, False, dict(n_trees=100, max_depth=12, max_bins=32))):
            r = run_case(torch, ctx, case, n, 128, regression, fit, a.sklearn_rows, a.held_out,
                         not a.no_sklearn and case.endswith("default"))
            out.append(r)
            print(json.dumps(r), flush=True)
    d0 = out[0]
    aims = {"bin_pass_ge_2.5TBps": d0["bin_TBps"] is not None and d0["bin_TBps"] >= AIMS["bin_tbs"],
            "level0_le_5ms": d0["levels"][0]["ms"] <= AIMS["level0_ms"],
            "default_fit_le_100ms": d0["fit_ms"] <= AIMS["default_fit_ms"]}
    print(json.dumps({"aims_met": aims}), flush=True)


if __name__ == "__main__":
    main()
