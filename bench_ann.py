"""IVF-Flat (b2k_ivf_search) at BASELINE cfg5's per-GPU shape on one GPU: 1.25 M items x 100 k queries x d = 128,
nlist = 1024, on a 1024-component Gaussian mixture and on plain normal data, for k = 10 and 64 and nprobe in
{1, 5, 20, 50, 200}.

Prints one JSON line.  Per configuration: the device times of each phase (CUDA events, option time_kernels) of one call
after a warm-up call: build (training subset, Lloyd, assign, sort and prep), probe, scan, refine + merge (with the pair
sort and the query gather); queries/s of the whole call; the scan's useful rate, 2 d x (query, probed item) pairs over
the scan time; and recall@k against b2k_knn_search on the same data, whose search time is reported beside it with the
card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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


def data(torch, kind, n, nq, d, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "normal":
        return (torch.randn(n, d, device="cuda", generator=g), torch.randn(nq, d, device="cuda", generator=g))
    mu = torch.randn(1024, d, device="cuda", generator=g) * 3.0
    X = mu[torch.randint(0, 1024, (n,), device="cuda", generator=g)] + torch.randn(n, d, device="cuda", generator=g)
    Q = mu[torch.randint(0, 1024, (nq,), device="cuda", generator=g)] + torch.randn(nq, d, device="cuda", generator=g)
    return X.contiguous(), Q.contiguous()


def recall(torch, idx, ex, k):
    hit = 0
    for q0 in range(0, idx.shape[0], 4096):
        a, b = idx[q0:q0 + 4096], ex[q0:q0 + 4096]
        hit += int((a[:, :, None] == b[:, None, :]).any(-1).sum())
    return hit / (idx.shape[0] * k)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1_250_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--k", type=int, nargs="+", default=[10, 64])
    ap.add_argument("--nprobe", type=int, nargs="+", default=[1, 5, 20, 50, 200])
    ap.add_argument("--data", nargs="+", default=["mixture", "normal"])
    args = ap.parse_args()
    import torch

    from spark_rapids_ml_b200 import _native

    out = {"shape": [args.items, args.queries, args.d], "nlist": args.nlist, **card(), "runs": []}
    with _native.Context(0) as ctx:
        for kind in args.data:
            X, Q = data(torch, kind, args.items, args.queries, args.d)
            for k in args.k:
                ctx.set_option("time_kernels", 1)
                ctx.knn_search(X, Q, k)
                _, ex = ctx.knn_search(X, Q, k)
                exact_ms = ctx.stats()["last_fused_ms"]
                for nprobe in args.nprobe:
                    ctx.ivf_search(X, Q, k, args.nlist, nprobe)
                    torch.cuda.synchronize()
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    ev[0].record()
                    _, idx, _, lists, _ = ctx.ivf_search(X, Q, k, args.nlist, nprobe, return_lists=True)
                    ev[1].record()
                    torch.cuda.synchronize()
                    st = ctx.stats()
                    sizes = torch.bincount(lists.long(), minlength=args.nlist).double()
                    scanned = float(sizes.mean()) * args.queries * min(nprobe, args.nlist)   # expected pairs
                    out["runs"].append({
                        "data": kind, "k": k, "nprobe": nprobe, "call_ms": ev[0].elapsed_time(ev[1]),
                        "build_ms": st["last_finalize_ms"], "probe_ms": st["last_probe_ms"],
                        "scan_ms": st["last_fused_ms"], "refine_merge_ms": st["last_reduce_ms"],
                        "queries_per_s": args.queries / (ev[0].elapsed_time(ev[1]) / 1e3),
                        "scan_useful_tflops": 2.0 * args.d * scanned / (st["last_fused_ms"] / 1e3) / 1e12
                        if st["last_fused_ms"] > 0 else None,
                        "items_scanned_share": scanned / (args.queries * args.items),
                        "recall": recall(torch, idx, ex, k), "exact_search_ms": exact_ms,
                        "path": st["last_path"]})
                ctx.set_option("time_kernels", 0)
            del X, Q
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
