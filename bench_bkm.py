"""Bisecting k-means benchmark: b2k_bkm_fit on a seeded Gaussian mixture at 10 M x 128, k = 16 and 64, maxIter 20, one
GPU.  Prints one JSON record: per level the device time, the rows split and the split pass's bytes/s over those rows
(each level reads them maxIter + 1 times) against the 3.35 TB/s of HBM3 in NVIDIA's H100 SXM data sheet; the split,
reduce, allreduce and host shares of the fit; b2k_kmeans_fit on the same data and k (maxIter 20); predict rows/s; and
the card's name and power limit read in the same run.

    python bench_bkm.py [--n 10000000] [--d 128] [--ks 16,64] [--max-iter 20]
"""
import argparse
import json
import subprocess
import time

import torch

from spark_rapids_ml_b200 import _native

HBM = 3.35e12


def mixture(n, d, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    means = torch.randn(k, d, device="cuda", generator=g) * 4
    z = torch.randint(0, k, (n,), device="cuda", generator=g)
    X = torch.empty(n, d, device="cuda", dtype=torch.float32)
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        X[s:e] = means[z[s:e]] + torch.randn(e - s, d, device="cuda", generator=g)
    return X


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def level_rows(out):
    """Rows of the nodes each level divided (from the tree: a level's dividing nodes are the parents of its nodes)."""
    idx = out["node_index"].tolist()
    size = dict(zip(idx, out["sizes"].tolist()))
    rows = {}
    for i in idx:
        if i > 1 and (i ^ 1 not in size or i % 2 == 0):
            lvl = i.bit_length() - 1
            rows[lvl] = rows.get(lvl, 0) + size[i // 2]
    return [rows.get(lv, 0) for lv in range(1, out["n_levels"] + 1)]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--ks", default="16,64")
    ap.add_argument("--max-iter", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bkm.py needs a GPU")
    ctx = _native.Context(0)
    X = mixture(a.n, a.d, 32, seed=0)
    res = {"bench": "bisecting_kmeans", "n": a.n, "d": a.d, "max_iter": a.max_iter, "card": card(), "runs": []}
    for k in [int(v) for v in a.ks.split(",")]:
        ctx.set_option("time_kernels", 1)
        ctx.bkm_fit(X[: 1 << 16], k, max_iter=2, seed=1)   # warm-up
        out, wall = timed(lambda: ctx.bkm_fit(X, k, max_iter=a.max_iter, seed=1))
        st = ctx.stats()
        ctx.set_option("time_kernels", 0)
        rows = level_rows(out)
        sweep_bytes = [r * a.d * 4 * (a.max_iter + 1) for r in rows]
        split_ms = st["last_fused_ms"]
        ctx.kmeans_fit(X[: 1 << 16], k, max_iter=2, seed=1)   # warm-up
        km, km_wall = timed(lambda: ctx.kmeans_fit(X, k, max_iter=a.max_iter, tol=0.0, seed=1))
        ctx.bkm_predict(X[: 1 << 16], out["node_index"], out["centers"])
        (_, _), p_wall = timed(lambda: ctx.bkm_predict(X, out["node_index"], out["centers"]))
        res["runs"].append({
            "k": k, "leaves": len(out["cluster_sizes"]), "levels": out["n_levels"], "fit_s": wall,
            "level_ms": [round(v, 3) for v in out["level_ms"].tolist()], "level_rows": rows,
            "split_ms": split_ms, "reduce_ms": st["last_reduce_ms"], "allreduce_ms": st["last_allreduce_ms"],
            "host_ms": st["last_finalize_ms"],
            "split_tb_per_s": sum(sweep_bytes) / (split_ms / 1e3) / 1e12,
            "split_share_of_hbm": sum(sweep_bytes) / HBM / (split_ms / 1e3),
            "floor_ms": sum(sweep_bytes) / HBM * 1e3,
            "training_cost": out["training_cost"],
            "kmeans_fit_s": km_wall, "kmeans_iters": int(km.get("n_iter_", 0)),
            "predict_rows_per_s": a.n / p_wall,
        })
    print(json.dumps(res))


if __name__ == "__main__":
    main()
