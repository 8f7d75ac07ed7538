"""UMAP on one GPU: fit of a seeded Gaussian mixture (100 k x 64, n_neighbors 15, 200 epochs) with per-phase device
times, the kNN rate, one layout epoch against the same epoch-synchronous epoch written in torch (index_add_), and the
transform rate.  Prints one JSON line.  Writes nothing."""
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

A, B = 1.5769434603113077, 0.8950608779109733   # min_dist 0.1, spread 1


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


def mixture(n: int, d: int, seed: int):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn(20, d, generator=g, device="cuda") * 5.0
    lab = torch.randint(0, 20, (n,), generator=g, device="cuda")
    return (centres[lab] + torch.randn(n, d, generator=g, device="cuda")).contiguous()


def torch_epoch(Y, rows, cols, eps_due, neg_rate, seed, a=A, b=B):
    """The epoch-synchronous epoch in torch: every due edge attracts both ends, draws neg_rate negatives for its head,
    contributions summed with index_add_."""
    import torch

    n = Y.shape[0]
    r, c = rows[eps_due], cols[eps_due]
    diff = Y[r] - Y[c]
    d2 = (diff * diff).sum(1, keepdim=True)
    ga = torch.where(d2 > 0, -2 * a * b * d2.clamp_min(1e-30) ** (b - 1) / (a * d2 ** b + 1), torch.zeros_like(d2))
    g = (ga * diff).clamp(-4, 4)
    acc = torch.zeros_like(Y)
    acc.index_add_(0, r, g)
    acc.index_add_(0, c, -g)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    head = r.repeat_interleave(neg_rate)
    k = torch.randint(0, n, (head.numel(),), generator=gen, device="cuda")
    diff = Y[head] - Y[k]
    d2 = (diff * diff).sum(1, keepdim=True)
    gr = torch.where(d2 > 0, 2 * b / ((0.001 + d2) * (a * d2 ** b + 1)), torch.zeros_like(d2))
    acc.index_add_(0, head, torch.where(d2 > 0, (gr * diff).clamp(-4, 4), torch.full_like(diff, 4.0)))
    return Y + acc, int(r.numel()) * (1 + neg_rate)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=200)
    ap.add_argument("--transform-rows", type=int, default=10_000_000)
    args = ap.parse_args()
    import torch

    from spark_rapids_ml_b200 import _native

    out = card()
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        X = mixture(args.n, args.d, 0)
        p = _native.umap_params(n_neighbors=15, n_components=2, n_epochs=args.epochs, init="spectral", a=A, b=B,
                                seed=1)
        ctx.umap_fit(X[:5000].contiguous(), _native.umap_params(n_neighbors=15, n_epochs=5, init="random", a=A, b=B))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emb, info = ctx.umap_fit(X, p)
        wall = time.perf_counter() - t0
        st = ctx.stats()
        g = ctx.umap_graph(info)
        eps = g["epochs_per_sample"]
        # attractive samples of the whole layout plus the negatives they draw (rate 5): the schedule's own counts
        fire = np.where(np.isfinite(eps), np.floor(args.epochs / eps), 0.0)
        samples = float(fire.sum() * (1 + 5))
        knn_flop = 2.0 * args.n * args.n * args.d * 3   # 3xTF32
        out.update({
            "fit_s": wall, "knn_ms": st["last_finalize_ms"], "graph_ms": st["last_reduce_ms"],
            "init_ms": st["last_allreduce_ms"], "layout_ms": st["last_fused_ms"], "init_used": info["init_used"],
            "ritz_residual": info["ritz_residual"], "nnz": info["nnz"],
            "knn_tflops": knn_flop / (st["last_finalize_ms"] * 1e-3) / 1e12,
            "layout_epoch_ms": st["last_fused_ms"] / args.epochs,
            "edge_samples_per_s": samples / (st["last_fused_ms"] * 1e-3),
        })
        # the torch epoch over the same graph, every kept edge due (the device's busiest epoch has every edge with
        # epochs_per_sample 1 due; the torch one does more work, so it is the baseline's best case per sample)
        indptr = torch.from_numpy(g["indptr"]).cuda()
        rows = torch.repeat_interleave(torch.arange(args.n, device="cuda"), indptr[1:] - indptr[:-1])
        cols = torch.from_numpy(g["indices"]).cuda().long()
        due = torch.from_numpy(np.isfinite(eps)).cuda()
        Y = emb.clone()
        for _ in range(3):
            torch_epoch(Y, rows, cols, due, 5, 0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        reps = 10
        for r in range(reps):
            _, ns = torch_epoch(Y, rows, cols, due, 5, r)
        e1.record()
        torch.cuda.synchronize()
        t_ms = e0.elapsed_time(e1) / reps
        out.update({"torch_epoch_ms": t_ms, "torch_edge_samples_per_s": ns / (t_ms * 1e-3)})
        # transform
        pt = _native.umap_params(n_neighbors=15, n_components=2, n_epochs=args.epochs // 3, a=A, b=B, seed=1)
        done, chunk, t_tr = 0, 2_000_000, 0.0
        while done < args.transform_rows:
            m = min(chunk, args.transform_rows - done)
            Q = mixture(m, args.d, 100 + done)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.umap_transform(X, emb, Q, pt)
            torch.cuda.synchronize()
            t_tr += time.perf_counter() - t0
            done += m
            del Q
        out.update({"transform_rows": done, "transform_rows_per_s": done / t_tr,
                    "transform_epochs": args.epochs // 3})
    out["layout_speedup_vs_torch_per_sample"] = out["edge_samples_per_s"] / out["torch_edge_samples_per_s"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
