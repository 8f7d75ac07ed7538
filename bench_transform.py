"""Model.transform(df).count() on one GPU for the models with a grouped device transform other than KMeans, whose
transform bench.py times: PCA, linear and logistic regression, the random-forest classifier and regressor, and UMAP.
Each model transforms a LocalSession frame of 10 000-row Arrow batches in pageable host memory: 1 M x 128 float32
rows, and for UMAP 1 M x 64 query rows against a model of bench_umap.py's size (100 k x 64 training rows, a 2-d
embedding).  The models are built from seeded attributes, except the forests, which are fitted on the first 100 k rows.
Prints one JSON line: each model's rows/s, best of --reps after one warm-up transform.  Writes nothing.

  python bench_transform.py [--rows 1000000] [--d 128] [--reps 3]
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


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


def models(X: np.ndarray, y: np.ndarray, rng: np.random.Generator) -> dict:
    from spark_rapids_ml_b200.classification import LogisticRegressionModel, RandomForestClassifier
    from spark_rapids_ml_b200.feature import PCAModel
    from spark_rapids_ml_b200.regression import LinearRegressionModel, RandomForestRegressor
    from spark_rapids_ml_b200.sparkshim import LocalSession

    d = X.shape[1]
    comp = np.linalg.qr(rng.normal(size=(d, 16)))[0].T
    fit_df = LocalSession().from_numpy(X[:100_000], col="features", extra={"label": y[:100_000]})
    pca = PCAModel(mean_=[0.0] * d, components_=comp.tolist(), explained_variance_ratio_=[1 / 16] * 16,
                   singular_values_=[1.0] * 16, n_cols=d, dtype="float32")
    return {
        "pca": pca.setInputCol("features").setOutputCol("pca"),
        "linear_regression": LinearRegressionModel(coef_=rng.normal(size=d).tolist(), intercept_=0.5, n_cols=d,
                                                   dtype="float32"),
        "logistic_regression": LogisticRegressionModel(coef_=[rng.normal(size=d).tolist()], intercept_=[0.1],
                                                       classes_=[0.0, 1.0], n_cols=d, dtype="float32", num_iters=1),
        "rf_classifier": RandomForestClassifier(numTrees=20, maxDepth=5, seed=1, num_workers=1).fit(fit_df),
        "rf_regressor": RandomForestRegressor(numTrees=20, maxDepth=5, seed=1, num_workers=1).fit(fit_df),
    }


def umap_model(rng: np.random.Generator):
    from spark_rapids_ml_b200.umap import UMAPModel

    centres = rng.normal(size=(20, 64)) * 5.0
    raw = (centres[rng.integers(0, 20, 100_000)] + rng.normal(size=(100_000, 64))).astype(np.float32)
    emb = rng.normal(size=(100_000, 2)).astype(np.float32)
    return UMAPModel(embedding_=emb, raw_data_=raw, n_cols=64, dtype="float32").setFeaturesCol("features"), centres


def rate(model, df, reps: int) -> dict:
    import torch

    model.transform(df).count()   # warm-up: module loads, the process's transform context, pinned staging
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = model.transform(df).count()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return {"rows_per_s": n / min(times), "seconds": times, "rows": n}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from spark_rapids_ml_b200.sparkshim import LocalSession

    if not torch.cuda.is_available():
        raise SystemExit("bench_transform.py needs a CUDA device")
    rng = np.random.default_rng(0)
    X = rng.normal(size=(args.rows, args.d)).astype(np.float32)
    y = (X[:, 0] + 0.5 * X[:, 1] > 0).astype(np.float32)
    df = LocalSession().from_numpy(X, col="features")
    out = card()
    out.update({"rows": args.rows, "d": args.d, "batch_rows": LocalSession().max_records_per_batch, "models": {}})
    for name, model in models(X, y, rng).items():
        out["models"][name] = rate(model, df, args.reps)
    del df
    um, centres = umap_model(rng)
    Q = (centres[rng.integers(0, 20, args.rows)] + rng.normal(size=(args.rows, 64))).astype(np.float32)
    out["models"]["umap"] = dict(rate(um, LocalSession().from_numpy(Q, col="features"), args.reps), train_rows=100_000,
                                 d=64)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
